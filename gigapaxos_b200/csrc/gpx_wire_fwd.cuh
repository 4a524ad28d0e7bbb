/*
 * gpx_wire_fwd.cuh -- client requests forwarded between nodes, on the device.  With the coordinators spread over the
 * members (PISM.roundRobinCoordinator :2251-2256), most requests enter at a node that does not coordinate their group,
 * and that node forwards them to the coordinator (PISM.handleProposal :854-885):
 *   k_wire_fwd    the sending side (gpx_wire_encode_forwards_device): the requests gpx_propose_device gave
 *                 GPX_RS_FORWARD become REQUEST packets addressed to the ballot's coordinator, cut as the RequestBatcher
 *                 cuts them.  One thread per run of a gid's requests, as in k_propose.  The walk of a run (fwd_run) is
 *                 shared with the JSON sweep (gpx_wire_json_enc.cuh, k_json_enc_fwd), which sends the same cuts.
 *   k_json_req    the receiving side for a Java peer (gpx_wire_decode_json_requests_device): under load a Java node
 *                 sends its forwards as JSON members of BATCHED_PAXOS_PACKETs (PaxosPacketBatcher.process :270-277),
 *                 which gpx_wire_decode_json_device lists as GPX_WS_UNHANDLED; the REQUEST members among them become
 *                 proposals, as k_wire_req_decode makes them of the byte form.  One thread per member.
 *   k_json_client the same decoder over a client's own packets (gpx_wire_decode_client_requests_device): a gigapaxos
 *                 client sends each RequestPacket as a bare JSON object (PaxosClientAsync.sendRequest :165-172) with
 *                 no "CA", so the client address comes from the receiver's stamp or the connection.  One thread per
 *                 packet.
 * Both are scalar, like the kernels they sit beside, so tests/emu compiles this file for the host.
 */
#pragma once
#include <type_traits>

#include "gpx_wire_json.cuh"

/* ---- forwarded REQUEST packets (gpx_wire_encode_forwards_device) -------------------------------------------------- */
struct WireFwdArgs {
  const gpx_request_rec* reqs;   /* [n] grouped by gid, as gpx_propose_device took them */
  const gpx_wire_req_meta* meta; /* [n] */
  const int32_t* status;         /* [n] gpx_propose_device's */
  const uint8_t* payload;        /* the request arena: bodies at reqs[q].payload_off */
  const int32_t* down;           /* [n_down] the nodes the host takes for down (PaxosManager.isNodeUp) */
  uint32_t n, n_down;
  uint8_t* rstatus;              /* [n] GPX_WE_* */
  uint32_t* cnt;                 /* [2][n] pass 0, per request that starts a packet: packet bytes, 1 */
  const uint32_t* off;           /* [2][n] their exclusive prefix sums */
  uint8_t* out;
  gpx_wire_ref* refs;
  int emit;
};

/* request q is forwarded: propose_run gave it GPX_RS_FORWARD (a wrapped slot may equal that code: the caller's route
 * says which), and it is not broadcasted (a broadcasted request reached every replica already, :854) */
__device__ __forceinline__ bool fwd_request(const WireFwdArgs& A, uint32_t q) {
  return A.status[q] == GPX_RS_FORWARD && !(A.meta[q].flags & GPX_RM_BROADCASTED);
}

/* request k heads a cut: its end, the consecutive forwarded requests after it that batch_end lets into its packet */
__device__ __forceinline__ uint32_t fwd_cut_end(const DevState& S, const WireFwdArgs& A, uint32_t k, uint32_t gid) {
  const uint32_t b = batch_end(S, A.reqs, A.n, k, gid);
  uint32_t e = k + 1;
  while (e < b && fwd_request(A, e)) e++;
  return e;
}

/* the forward count the outer request of a cut headed by k carries: forwardCount++ (setForwarderID :437-441, Java int) */
__device__ __forceinline__ int32_t fwd_count(const WireFwdArgs& A, uint32_t k) {
  return (int32_t)((uint32_t)A.meta[k].forward_count + 1u);
}

/* the run of gid's requests that starts at request i, walked as PISM.handleProposal forwards it.  The run is routed as
 * propose_run routes it, from its first request's entry lane; its forwarded requests are cut with batch_end.
 * skip(k) is called for every request that is not forwarded, cut(k, b, st, dst, di) once per cut [k, b) with its
 * status and its destination node dst, member index di of the group's member set (valid when st is GPX_WE_SENT). */
template <typename Skip, typename Cut>
__device__ __forceinline__ void fwd_run(const DevState& S, const WireNames& W, const WireFwdArgs& A, uint32_t i,
                                        Skip&& skip, Cut&& cut) {
  const uint32_t gid = A.reqs[i].gid;
  uint32_t run_end = i + 1;
  while (run_end < A.n && A.reqs[run_end].gid == gid) run_end++;
  uint32_t meta = 0;
  int clane = -1;
  int32_t bcoord = 0;
  const bool routed = propose_route(S, gid, (A.reqs[i].flags >> 8) & 0xfu, &meta, &clane, &bcoord) == GPX_RS_FORWARD;
  /* the destination: the ballot's coordinator, or the member after it when the host takes it for down
   * (getNextCoordinator :2232-2241); the host runs for coordinator instead when that is a local node (:869) or the
   * coordinator is not a member */
  uint8_t run_st = GPX_WE_SENT;
  int32_t dst = bcoord;
  uint32_t di = 0xffu;
  if (routed) {
    const MsetInfo* ms = &S.msets[meta & 0xffffu];
    const uint32_t R = (meta >> 16) & 0xffu;
    di = wire_member_idx(ms, R, bcoord);
    if (di == 0xffu) {
      run_st = GPX_WE_ELECT;
    } else {
      for (uint32_t d = 0; d < A.n_down; d++)
        if (A.down[d] == bcoord) {
          di = (di + 1u) % R;
          break;
        }
      dst = ms->nodes[di];
      if (ms->lane_of_idx[di] != 0xffu) run_st = GPX_WE_ELECT;
    }
  }
  const bool named = routed && W.slot != nullptr && W.slot[gid] != GPX_NAME_NONE;
  uint32_t k = i;
  while (k < run_end) {
    if (!routed || !fwd_request(A, k)) {
      skip(k);
      k++;
      continue;
    }
    const uint32_t b = fwd_cut_end(S, A, k, gid);
    uint8_t st = run_st;
    if (st == GPX_WE_SENT && fwd_count(A, k) > 3) st = GPX_WE_ELECT; /* isPingPonging :508 */
    if (st == GPX_WE_SENT && !named) st = GPX_WE_NO_NAME;
    cut(k, b, st, dst, di);
    k = b;
  }
}

/* the REQUEST packet of the cut [k, b) at o, byte-identical to gpx_wire_encode_request: the outer request is the
 * cut's first with forwardCount + 1, the others its `batched`.  Returns its bytes. */
__device__ __forceinline__ uint32_t fwd_packet(uint8_t* o, const WireNames& W, const WireFwdArgs& A, uint32_t gid,
                                               uint32_t k, uint32_t b) {
  WireAccArgs X;
  X.head = nullptr;
  X.reqs = A.reqs;
  X.meta = A.meta;
  X.n_reqs = A.n;
  X.payload = A.payload;
  const uint32_t len = ww_requests(o, GPX_PT_REQUEST, W, gid, X, k, b - k);
  ww_i32(o + 13u + W.name[(size_t)gid * GPX_NAME_BYTES] + 34u, fwd_count(A, k)); /* the outer request's forwardCount */
  return len;
}

/* one thread per request; the first request of a gid's run walks the run (fwd_run), each cut one REQUEST packet.
 * Pass 0 writes rstatus and the packet sizes, pass 1 the packets and their refs at the scanned offsets. */
__global__ void k_wire_fwd(const __grid_constant__ DevState S, const __grid_constant__ WireNames W,
                           const __grid_constant__ WireFwdArgs A) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= A.n) return;
  const uint32_t gid = A.reqs[i].gid;
  if (i > 0 && A.reqs[i - 1].gid == gid) return;
  fwd_run(
      S, W, A, i,
      [&](uint32_t k) {
        if (!A.emit) {
          A.rstatus[k] = GPX_WE_VOID;
          A.cnt[k] = A.cnt[A.n + k] = 0;
        }
      },
      [&](uint32_t k, uint32_t b, uint8_t st, int32_t dst, uint32_t) {
        if (!A.emit) {
          for (uint32_t q = k; q < b; q++) {
            A.rstatus[q] = st;
            A.cnt[q] = A.cnt[A.n + q] = 0;
          }
          if (st == GPX_WE_SENT) {
            A.cnt[k] = wire_requests_bytes(W, gid, A.reqs, k, b - k);
            A.cnt[A.n + k] = 1;
          }
        } else if (st == GPX_WE_SENT) {
          gpx_wire_ref r;
          r.off = A.off[k];
          r.len = fwd_packet(A.out + A.off[k], W, A, gid, k, b);
          r.gid = gid;
          r.node = dst;
          A.refs[A.off[A.n + k]] = r;
        }
      });
}

/* ---- REQUEST members of a Java peer's BATCHED_PAXOS_PACKETs (gpx_wire_decode_json_requests_device) ---------------- */
/* the keys of RequestPacket(net.minidev.json.JSONObject) :584-649 / toJSONSmartImpl :697-742 and PaxosPacket's */
enum { JQ_TYPE, JQ_PT, JQ_ID, JQ_V, JQ_QID, JQ_QV, JQ_ET, JQ_E, JQ_NFWDS, JQ_STOP, JQ_QF, JQ_BC, JQ_CA, JQ_LA, JQ_BATCH,
       JQ_RV, JQ_DIG, JQ_N };
__device__ __forceinline__ int json_req_key(const JStr& s) {
  if (s.wide) return -1;
  switch (s.len) {
    case 1:
      if (s.head == 'V') return JQ_V;
      if (s.head == 'E') return JQ_E;
      return -1;
    case 2:
      if (s.head == JK('P', 'T', 0, 0, 0)) return JQ_PT;
      if (s.head == JK('I', 'D', 0, 0, 0)) return JQ_ID;
      if (s.head == JK('Q', 'V', 0, 0, 0)) return JQ_QV;
      if (s.head == JK('E', 'T', 0, 0, 0)) return JQ_ET;
      if (s.head == JK('Q', 'F', 0, 0, 0)) return JQ_QF;
      if (s.head == JK('B', 'C', 0, 0, 0)) return JQ_BC;
      if (s.head == JK('C', 'A', 0, 0, 0)) return JQ_CA;
      if (s.head == JK('L', 'A', 0, 0, 0)) return JQ_LA;
      if (s.head == JK('R', 'V', 0, 0, 0)) return JQ_RV;
      return -1;
    case 3:
      if (s.head == JK('Q', 'I', 'D', 0, 0)) return JQ_QID;
      if (s.head == JK('D', 'I', 'G', 0, 0)) return JQ_DIG;
      return -1;
    case 4:
      if (s.head == JK('t', 'y', 'p', 'e', 0)) return JQ_TYPE;
      if (s.head == JK('S', 'T', 'O', 'P', 0)) return JQ_STOP;
      return -1;
    case 5:
      if (s.head == JK('N', 'F', 'W', 'D', 'S')) return JQ_NFWDS;
      if (s.head == JK('B', 'A', 'T', 'C', 'H')) return JQ_BATCH;
      return -1;
    default: return -1;
  }
}
struct JsonReqKeys {
  enum { N = JQ_N, PP = -2 };
  __device__ __forceinline__ static int id(const JStr& s, const JRd&, uint32_t) { return json_req_key(s); }
};
/* ... and the receiver's stamps of a packet that came in over a socket (MessageExtractor.stampAddressIntoJSONObject
 * :348-376): the connection's remote and local address, read where "CA" / "LA" are absent (RequestPacket(JSONObject)
 * :530-536, JSONNIOTransport.getSenderAddress / getReceiverAddress).  A client's own request carries no "CA". */
enum { JQ_SNDR = JQ_N, JQ_RCVR, JQ_CN };
struct JsonClientKeys {
  enum { N = JQ_CN, PP = -2 };
  __device__ __forceinline__ static int id(const JStr& s, const JRd& J, uint32_t at) {
    if (s.len != 13u || s.wide) return json_req_key(s);
    if (s.head == JK8('_', 'S', 'N', 'D', 'R', '_', 'A', 'D') && json_key_rest(J, at, s, "DRESS", 5)) return JQ_SNDR;
    if (s.head == JK8('_', 'R', 'C', 'V', 'R', '_', 'A', 'D') && json_key_rest(J, at, s, "DRESS", 5)) return JQ_RCVR;
    return -1;
  }
};
/* a request object's address keys: a stamp stands in for an absent "CA" / "LA", as the reference reads it */
template <class Keys>
__device__ __forceinline__ void json_req_stamps(uint32_t* pos) {
  if constexpr (Keys::N > JQ_N) {
    if (!pos[JQ_CA]) pos[JQ_CA] = pos[JQ_SNDR];
    if (!pos[JQ_LA]) pos[JQ_LA] = pos[JQ_RCVR];
  }
}

/* the fields of one request object */
struct JsonReq {
  int64_t qid, et;
  int32_t e, nfwds;
  uint32_t qv_at, qv_len; /* QV's opening quote, its characters */
  bool stop, qf, bc;
  uint8_t ca_ip[4], la_ip[4];
  uint16_t ca_port, la_port;
};

/* an optional bool at `at`: false when present and not true / false */
__device__ __forceinline__ bool json_get_bool(const JRd& J0, uint32_t at, bool* v) {
  JRd J = J0;
  *v = false;
  if (!json_at(J, at)) return true;
  if (jr_peek(J) == 't') return *v = jr_word(J, "true", 4);
  return jr_word(J, "false", 5);
}
/* an optional address string at `at` (false: not a string).  *lit: it is [anything/]a.b.c.d:port with a port of
 * 1-65535 -- Util.getInetSocketAddressFromString :278-287 (everything up to the last '/' dropped) for a literal IPv4
 * address.  Anything else (a hostname wants a lookup; leading zeros, a line terminator, which the reference's ".*"
 * does not cross, or extra ':' parts) is left to the host. */
__device__ __forceinline__ bool json_get_addr(const JRd& J0, uint32_t at, bool* lit, uint8_t* ip, uint16_t* port) {
  JRd J = J0;
  *lit = true;
  if (!json_at(J, at)) return true;
  if (!jr_eat(J, '"')) return false;
  uint32_t part = 0, val = 0, nd = 0;
  bool bad = false, host = false;
  for (;;) {
    uint32_t u = 0;
    const int r = jr_unit(J, &u);
    if (r < 0) return false;
    if (r == 1) break;
    if (u == '\n' || u == '\r' || u == 0x85u || u > 0xffu) host = true;
    if (u == '/') {
      part = val = nd = 0;
      bad = false;
    } else if (bad) {
    } else if (u >= '0' && u <= '9') {
      if (part < 4 && nd == 1 && val == 0) bad = true; /* a leading zero in an octet */
      val = val * 10u + (u - '0');
      if (++nd > 5 || (part < 4 && val > 255u)) bad = true;
    } else if (u == '.' && part < 3 && nd > 0) {
      ip[part++] = (uint8_t)val;
      val = nd = 0;
    } else if (u == ':' && part == 3 && nd > 0) {
      ip[3] = (uint8_t)val;
      part = 4;
      val = nd = 0;
    } else {
      bad = true;
    }
  }
  *lit = !host && !bad && part == 4 && nd > 0 && val >= 1u && val <= 65535u;
  *port = *lit ? (uint16_t)val : (uint16_t)0;
  if (!*lit) ip[0] = ip[1] = ip[2] = ip[3] = 0;
  return true;
}
/* the request fields of an object whose keys are at pos: GPX_WS_OK, GPX_WS_MALFORMED (a schema failure) or
 * GPX_WS_UNHANDLED (RV or DIG present, a QV character above U+00FF, an address the host decides) */
__device__ __forceinline__ int32_t json_req_fields(const JRd& J0, const uint32_t* pos, JsonReq& f) {
  memset(&f, 0, sizeof f);
  JRd J = J0;
  bool ok = json_at(J, pos[JQ_QID]);
  if (ok) {
    f.qid = jr_i64(J);
    ok = J.ok;
  }
  J = J0;
  if (ok && (ok = json_at(J, pos[JQ_ET]))) {
    f.et = jr_i64(J);
    ok = J.ok;
  }
  ok = ok && json_get_i32(J0, pos[JQ_E], &f.e);
  ok = ok && (!pos[JQ_NFWDS] || json_get_i32(J0, pos[JQ_NFWDS], &f.nfwds));
  ok = ok && json_get_bool(J0, pos[JQ_STOP], &f.stop) && json_get_bool(J0, pos[JQ_QF], &f.qf) &&
       json_get_bool(J0, pos[JQ_BC], &f.bc);
  bool wide = false, ca = true, la = true;
  J = J0;
  if (ok && (ok = json_at(J, pos[JQ_QV]) && jr_peek(J) == '"')) {
    f.qv_at = J.n;
    const JStr s = jr_string(J);
    ok = J.ok;
    f.qv_len = s.len;
    wide = s.wide;
  }
  ok = ok && json_get_addr(J0, pos[JQ_CA], &ca, f.ca_ip, &f.ca_port) &&
       json_get_addr(J0, pos[JQ_LA], &la, f.la_ip, &f.la_port);
  if (!ok) return GPX_WS_MALFORMED;
  if (pos[JQ_RV] || pos[JQ_DIG] || wide || !ca || !la) return GPX_WS_UNHANDLED;
  return GPX_WS_OK;
}

struct WireJsonReqArgs {
  const uint8_t* bytes;
  const gpx_wire_ref* pkts;
  const gpx_wire_member* mem;
  uint64_t n_bytes;
  uint32_t n_pkts;
  uint32_t n;          /* members */
  long long now_ms;
  int32_t* status;     /* [n] */
  uint32_t* cnt;       /* [WQ_NCNT][n]: pass 0 writes the member's requests and payload bytes (each value padded to 16) */
  const uint32_t* off; /* [WQ_NCNT][n]: pass 1 reads their exclusive prefix sums */
  /* pass 1: requests and meta staged in member order, the sort keys (gids) beside them; the payload is the output */
  gpx_request_rec* req;
  gpx_wire_req_meta* meta;
  uint32_t* key;
  uint8_t* payload;
  int emit;
};

/* a client's own packets (gpx_wire_decode_client_requests_device): the members are the whole packets, peers[k] the
 * transport address of packet k's connection (nullptr: none) */
static_assert(sizeof(gpx_wire_peer) == 16, "gpx_wire_peer is 16 bytes");
struct WireClientReqArgs : WireJsonReqArgs {
  const gpx_wire_peer* peers;
};

/* the first byte after leading whitespace opens a JSON object (a byteified packet's first byte is its type) */
__device__ __forceinline__ bool json_object_at(JRd J) {
  jr_ws(J);
  return jr_peek(J) == '{';
}

/* an outer request with neither "CA" nor a stamp takes the connection's address, "LA" the local one; an unknown port
 * (0) leaves the request to the host.  Entries of its BATCH take none: each is read from its own object (:541-552). */
__device__ __forceinline__ int32_t json_req_peer(const gpx_wire_peer* peers, uint32_t k, const uint32_t* pos,
                                                 JsonReq& f, int32_t st) {
  if (!peers || st == GPX_WS_MALFORMED) return st;
  const gpx_wire_peer p = peers[k];
  if (!pos[JQ_CA]) {
    if (!p.sender_port) return GPX_WS_UNHANDLED;
    for (int b = 0; b < 4; b++) f.ca_ip[b] = p.sender_ip[b];
    f.ca_port = p.sender_port;
  }
  if (!pos[JQ_LA]) {
    if (!p.receiver_port) return GPX_WS_UNHANDLED;
    for (int b = 0; b < 4; b++) f.la_ip[b] = p.receiver_ip[b];
    f.la_port = p.receiver_port;
  }
  return st;
}

/* one request with its value unescaped: k_wire_req_decode's record (wire_put_request) for the same RequestPacket */
__device__ __forceinline__ void json_put_request(const WireJsonReqArgs& A, WireReqTo& t, const JRd& J0,
                                                 const JsonReq& f) {
  gpx_wire_req_meta m;
  memset(&m, 0, sizeof m);
  for (int b = 0; b < 4; b++) {
    m.client_ip[b] = f.ca_ip[b];
    m.listen_ip[b] = f.la_ip[b];
  }
  m.client_port = f.ca_port;
  m.listen_port = f.la_port;
  m.forward_count = f.nfwds;
  m.entry_time = f.et;
  m.flags = (f.qf ? GPX_RM_RETURN_VALUE : 0u) | (f.bc ? GPX_RM_BROADCASTED : 0u);
  uint8_t* d = wire_put_request(A, t, f.qid, f.stop, f.e, f.qv_len, m);
  JRd Q = J0;
  Q.n = f.qv_at + 1u;
  for (uint32_t b = 0; b < f.qv_len; b++) { /* one thread copies the whole value, however long */
    uint32_t u = 0;
    jr_unit(Q, &u);
    d[b] = (uint8_t)u;
  }
}

/* one member (k_json_req: a member listed GPX_WS_UNHANDLED; k_json_client: a whole packet, Client).  Pass 0
 * (emit == 0): a REQUEST object (PT 1) is parsed and validated with its BATCH, its name, version and receiving node
 * looked up: its status and output sizes; every other member's status is copied.  Pass 1 parses the OK members again
 * and writes their requests, meta and values at the scanned offsets.  A client's packet is decoded when it is an
 * object: anything else, and JSON of another type, is the host's (GPX_WS_UNHANDLED); its addresses fall back to the
 * stamps and then to the connection (json_req_peer). */
template <bool Client, typename Args>
__device__ __forceinline__ void json_req_run(const DevState& S, const WireNames& W, const Args& A, uint32_t i,
                                             const gpx_wire_member mb) {
  using Keys = typename std::conditional<Client, JsonClientKeys, JsonReqKeys>::type;
  if (A.emit && (A.status[i] != GPX_WS_OK || mb.status != GPX_WS_UNHANDLED)) return; /* a copied OK has no request */
  int32_t st = mb.status;
  uint32_t nreq = 0, pay = 0, gid = GPX_NAME_NONE, lane = 0;
  int32_t node = 0;
  JRd J;
  J.b = A.bytes;
  J.n = mb.off;
  J.end = mb.off + mb.len;
  J.ok = true;
  uint32_t pos[Keys::N], ppc = GPX_JSON_NONE;
  JsonReq f;
  if (st == GPX_WS_UNHANDLED) {
    int32_t type = 0, pt = 0, ver = 0;
    if ((uint64_t)mb.off + mb.len > A.n_bytes || mb.pkt >= A.n_pkts) {
      st = GPX_WS_MALFORMED;
    } else if (Client && !json_object_at(J)) {
      /* the byte form, or no JSON object: the host's */
    } else {
      json_keys_t<Keys>(J, pos, nullptr, &ppc);
      jr_ws(J);
      if (!J.ok || J.n != J.end || !json_get_i32(J, pos[JQ_TYPE], &type))
        st = GPX_WS_MALFORMED;
      else if (Client && type != GPX_PT_PAXOS_PACKET) /* a client's other JSON */
        st = GPX_WS_UNHANDLED;
      else if (type != GPX_PT_PAXOS_PACKET || !json_get_i32(J, pos[JQ_PT], &pt))
        st = GPX_WS_MALFORMED;
      else if (pt != GPX_PT_REQUEST)
        st = GPX_WS_UNHANDLED;
      else
        st = pos[JQ_ID] && J.b[pos[JQ_ID]] == '"' && json_get_i32(J, pos[JQ_V], &ver) ? GPX_WS_OK : GPX_WS_MALFORMED;
    }
    if (st == GPX_WS_OK) {
      json_req_stamps<Keys>(pos);
      st = json_req_fields(J, pos, f);
      if constexpr (Client) st = json_req_peer(A.peers, i, pos, f, st);
      nreq = 1;
      pay = (f.qv_len + 15u) & ~15u;
      if (st != GPX_WS_MALFORMED && pos[JQ_BATCH]) { /* one level of latched requests (RequestBatcher) */
        JRd B = J;
        B.n = pos[JQ_BATCH];
        bool ok = jr_eat(B, '[');
        jr_ws(B);
        if (ok && jr_peek(B) == ']') {
        } else {
          while (ok) {
            uint32_t sp[Keys::N];
            json_keys_t<Keys>(B, sp, nullptr, &ppc);
            ok = B.ok && !sp[JQ_BATCH];
            if (!ok) break;
            JsonReq g;
            json_req_stamps<Keys>(sp);
            const int32_t s = json_req_fields(B, sp, g);
            if (s == GPX_WS_MALFORMED) {
              ok = false;
              break;
            }
            if (s == GPX_WS_UNHANDLED) st = GPX_WS_UNHANDLED; /* the request goes to the host whole */
            nreq++;
            pay += (g.qv_len + 15u) & ~15u;
            jr_ws(B);
            if (jr_peek(B) == ',') {
              B.n++;
              continue;
            }
            ok = jr_eat(B, ']');
            break;
          }
        }
        if (!ok) st = GPX_WS_MALFORMED;
      }
    }
    GroupCtx g;
    if (st == GPX_WS_OK) {
      JRd I = J;
      I.n = pos[JQ_ID];
      const JStr id = jr_string(I);
      gid = json_id_gid(W, J, pos[JQ_ID], id);
      st = wire_group(S, W, gid, ver, g);
    }
    if (st == GPX_WS_OK) {
      node = A.pkts[mb.pkt].node;
      st = wire_recv_lane(S, g, node, lane);
    }
  }
  if (!A.emit) {
    A.status[i] = st;
    A.cnt[i] = st == GPX_WS_OK ? nreq : 0u;
    A.cnt[A.n + i] = st == GPX_WS_OK ? pay : 0u;
    return;
  }
  WireReqTo t = {A.off[i], A.off[A.n + i], gid, i, lane, node};
  json_put_request(A, t, J, f);
  if (!pos[JQ_BATCH]) return;
  JRd B = J;
  B.n = pos[JQ_BATCH] + 1u;
  jr_ws(B);
  if (jr_peek(B) == ']') return;
  for (;;) {
    uint32_t sp[Keys::N];
    json_keys_t<Keys>(B, sp, nullptr, &ppc);
    JsonReq g;
    json_req_stamps<Keys>(sp);
    json_req_fields(B, sp, g);
    json_put_request(A, t, B, g);
    jr_ws(B);
    if (jr_peek(B) != ',') return;
    B.n++;
  }
}

/* one thread per member of gpx_wire_decode_json_requests_device */
__global__ void k_json_req(const __grid_constant__ DevState S, const __grid_constant__ WireNames W,
                           const __grid_constant__ WireJsonReqArgs A) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= A.n) return;
  json_req_run<false>(S, W, A, i, A.mem[i]);
}

/* one thread per packet of gpx_wire_decode_client_requests_device: the packet is the member */
__global__ void k_json_client(const __grid_constant__ DevState S, const __grid_constant__ WireNames W,
                              const __grid_constant__ WireClientReqArgs A) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= A.n) return;
  const gpx_wire_ref r = A.pkts[i];
  json_req_run<true>(S, W, A, i, gpx_wire_member{i, r.off, r.len, GPX_WS_UNHANDLED});
}
