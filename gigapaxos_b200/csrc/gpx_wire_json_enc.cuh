/*
 * gpx_wire_json_enc.cuh -- the sending side of the JSON form (gpx_wire_encode_json_sweep_device, and
 * gpx_wire_encode_json_device, the sweep without forwards): a node's reply and decision records, and the requests it
 * forwards, become what a loaded Java node sends, BATCHED_PAXOS_PACKET wrappers (type 37) of BatchedAcceptReply (34),
 * BatchedCommit (35) and REQUEST (1) objects, one wrapper per recipient set and cut, every NACK as a bare ACCEPT_REPLY
 * (8) and every forward of several requests as a lone REQUEST packet in the byte form.  The rules are in
 * include/gpx.h; the objects are byte-identical to gigapaxos_b200/packets_json.py's.
 *
 * The records are classified and sorted as the byte encoders do it (k_wire_enc_keys_*, then a stable sort of the keys),
 * so a member is a run of wire_run, with wire_slots_each's slots.  Then:
 *   k_json_enc_nacks    one thread per reply: routes a NACK as wire_reply_route routes a positive reply, sizes its
 *                       bare packet.
 *   k_json_enc_fwd      one thread per run of a gid's requests (gpx_wire_fwd.cuh's fwd_run, as k_wire_fwd walks it):
 *                       each request's status; a cut of one request becomes a member, any other cut (and a member too
 *                       large to wrap) a lone REQUEST packet, sized here.
 *   k_json_enc_members  one thread per member candidate (sorted reply positions, then sorted decision positions, then
 *                       requests): the run or forward it starts, its sending lane, its recipient set and its object's
 *                       size (nothing written); the first candidate of each (lane, recipient set) by atomicMin.
 *   k_json_enc_keys     the wrapper sort key (lane, first candidate of the member's set) per candidate.
 *   (a stable radix sort by that key; candidates are in sweep order already, so the order is (lane, first, position))
 *   k_json_enc_vals     the member sizes + 1 in sorted order, for a scan by key: each member's start in its group's
 *                       comma-joined stream.
 *   k_json_enc_cut      one thread per sorted member: does it open or close a wrapper (the cut rule), its bytes in the
 *                       output (object, separator or wrapper head, wrapper tail) and its wrapper's refs.
 *   k_json_enc_emit_nacks, k_json_enc_emit_fwd, k_json_enc_emit   write the packets at the scanned offsets (bare
 *                       NACKs, then lone REQUEST packets, then wrappers); the member that opens a wrapper writes its
 *                       head and notes where it starts, the one that closes it writes its tail.
 *   k_json_enc_refs     the member that closes a wrapper indexes it once per recipient node.
 * Every kernel is scalar and byte-addressed, so tests/emu compiles this file for the host.
 */
#pragma once
#include "gpx_wire_fwd.cuh" /* fwd_run: the forwards are k_wire_fwd's */

#include <algorithm>
#include <map>
#include <vector>

#define GPX_JSON_ENC_NONE 0xffffffffu
#define GPX_JSON_ENC_NOKEY 0xffffffffffffffffull

/* {"type":90,"PT":37,"V":-1,"PP":[ and ]} */
#define GPX_JSON_WRAP_HEAD "{\"type\":90,\"PT\":37,\"V\":-1,\"PP\":["
static_assert(sizeof(GPX_JSON_WRAP_HEAD) - 1 + 2 == GPX_JSON_WRAP_OVERHEAD, "wrapper head and tail");

/* the distinct recipient sets, built on the host from the member-set table (json_sets in gpx_wire_host.inc) */
struct JsonSets {
  const uint32_t* of_mset; /* [GPX_MAX_MSETS] set of the member nodes no local lane serves */
  const uint32_t* one;     /* [GPX_MAX_MSETS][GPX_MAX_GROUP_SIZE] set {nodes[i]} */
  const int32_t* nodes;    /* [n][GPX_MAX_GROUP_SIZE] each set's nodes, ascending */
  const uint32_t* count;   /* [n] */
  uint32_t n;
};

/* the host's side of JsonSets: interned member sets never change, so the table grows with the member-set table
 * (grow covers the sets interned since the last call); at most GPX_MAX_MSETS x (GPX_MAX_GROUP_SIZE + 1) sets */
struct JsonSetTable {
  std::vector<uint32_t> of_mset, one, count;
  std::vector<int32_t> nodes;
  std::map<std::vector<int32_t>, uint32_t> ids;
  size_t msets = 0; /* member sets covered */
  uint32_t id(std::vector<int32_t> v) {
    std::sort(v.begin(), v.end());
    const auto it = ids.find(v);
    if (it != ids.end()) return it->second;
    const uint32_t k = (uint32_t)count.size();
    ids.emplace(v, k);
    count.push_back((uint32_t)v.size());
    v.resize(GPX_MAX_GROUP_SIZE, INT32_MIN);
    nodes.insert(nodes.end(), v.begin(), v.end());
    return k;
  }
  void grow(const MsetInfo* ms, size_t n) {
    of_mset.resize(n, GPX_JSON_ENC_NONE);
    one.resize(n * GPX_MAX_GROUP_SIZE, GPX_JSON_ENC_NONE);
    for (; msets < n; msets++) {
      const MsetInfo& m = ms[msets];
      std::vector<int32_t> remote;
      for (uint32_t i = 0; i < m.R && i < GPX_MAX_GROUP_SIZE; i++) {
        one[msets * GPX_MAX_GROUP_SIZE + i] = id({m.nodes[i]});
        if (m.lane_of_idx[i] == 0xffu) remote.push_back(m.nodes[i]);
      }
      of_mset[msets] = id(remote);
    }
  }
};

enum { JE_BYTES = 0, JE_REFS = 1, JE_OPENS = 2, JE_BIG = 3, JE_NCNT = 4 };

struct WireJsonEncArgs {
  WireEncodeArgs R, D; /* replies and decisions: records, rstatus, keys and their stable order (perm, skey) */
  JsonSets Z;
  uint32_t n;          /* member candidates: the R.n sorted reply positions, the D.n sorted decision positions, then
                        * the F.n requests */
  uint32_t L;
  uint32_t T;          /* cut width: wrap_bytes - GPX_JSON_WRAP_OVERHEAD - GPX_JSON_MAX_MEMBER */
  uint32_t* first;     /* [L][Z.n] the lowest candidate of each (lane, recipient set) */
  uint32_t* mset;      /* [n] recipient set of the member candidate c starts, GPX_JSON_ENC_NONE if it starts none */
  uint8_t* mlane;      /* [n] its sending lane */
  uint32_t* msize;     /* [n] its object's bytes */
  unsigned long long* key;         /* [n] (lane << 32 | first), GPX_JSON_ENC_NOKEY for no member */
  const unsigned long long* skey;  /* [n] the keys in stable order */
  const uint32_t* order;           /* [n] the candidate at sorted position j */
  uint32_t* val;       /* [n] msize + 1 in sorted order (0: no member) */
  const uint32_t* start; /* [n] exclusive sums of val within each key: the member's start in its group's stream */
  uint32_t* cnt;       /* [JE_NCNT][n] per sorted position: output bytes, refs, wrappers opened, oversized members */
  const uint32_t* off; /* [JE_NCNT][n] their exclusive prefix sums */
  uint32_t* ncnt;      /* [2][R.n] per reply: bare NACK bytes, NACK packets */
  const uint32_t* noff;
  uint32_t nack_bytes, n_nacks; /* the totals of ncnt: the lone REQUEST packets follow the bare NACKs */
  uint2* wbeg;         /* [n] per wrapper: its offset in out, its first ref */
  uint8_t* out;
  gpx_wire_ref* refs;
  /* the forwards (F.n == 0, as a zeroed struct has it: none).  Candidate R.n + D.n + q is request q.  F.rstatus gets
   * the statuses; F.cnt / F.off are [2][F.n] rows per request that heads a lone packet: its bytes, 1 */
  WireFwdArgs F;
  uint8_t* fmem;       /* [F.n] request q heads a cut of one request that is written as a member */
  uint8_t* flane;      /* [F.n] at the head of a GPX_WE_SENT cut: its sending lane (the run's entry lane) */
  uint8_t* fdi;        /* [F.n] and its destination's member index */
  uint32_t lone_bytes, n_lone; /* the totals of F.cnt: the wrappers follow the lone REQUEST packets */
};

/* ---- JSON text, or only its length (p == nullptr) ------------------------------------------------------------------- */
struct JsonW {
  uint8_t* p;
  uint32_t n;
};
__device__ __forceinline__ void jw_c(JsonW& w, uint32_t c) {
  if (w.p) w.p[w.n] = (uint8_t)c;
  w.n++;
}
__device__ __forceinline__ void jw_s(JsonW& w, const char* s) {
  for (; *s; s++) jw_c(w, (uint8_t)*s);
}
/* json.dumps of an int: decimal, '-' when negative */
__device__ __forceinline__ void jw_i64(JsonW& w, int64_t v) {
  uint64_t u = v < 0 ? 0ull - (uint64_t)v : (uint64_t)v;
  if (v < 0) jw_c(w, '-');
  uint32_t d = 1;
  for (uint64_t t = u; t >= 10u; t /= 10u) d++;
  if (w.p)
    for (uint32_t k = d; k-- > 0; u /= 10u) w.p[w.n + k] = (uint8_t)('0' + u % 10u);
  w.n += d;
}
/* n ISO-8859-1 bytes as json.dumps writes the string: \" \\ \b \f \n \r \t, every other byte below 0x20 or from
 * 0x7f up as \u00xx (lowercase hex), the rest as it is */
__device__ __forceinline__ void jw_str(JsonW& w, const uint8_t* m, uint32_t n) {
  jw_c(w, '"');
  for (uint32_t i = 0; i < n; i++) {
    const uint32_t c = m[i];
    const uint32_t e = c == '"' ? '"' : c == '\\' ? '\\' : c == 8 ? 'b' : c == 12 ? 'f' : c == 10 ? 'n'
                     : c == 13 ? 'r' : c == 9 ? 't' : 0u;
    if (e) {
      jw_c(w, '\\');
      jw_c(w, e);
    } else if (c < 0x20u || c >= 0x7fu) {
      jw_s(w, "\\u00");
      jw_c(w, "0123456789abcdef"[c >> 4]);
      jw_c(w, "0123456789abcdef"[c & 15u]);
    } else {
      jw_c(w, c);
    }
  }
  jw_c(w, '"');
}
/* a group's paxosID */
__device__ __forceinline__ void jw_name(JsonW& w, const WireNames& W, uint32_t gid) {
  const uint8_t* m = W.name + (size_t)gid * GPX_NAME_BYTES;
  jw_str(w, m + 1, m[0]);
}
/* PaxosPacket.toJSONObject :478-494: {"type":90,"PT":pt,"ID":name,"V":version */
__device__ __forceinline__ void jw_head(JsonW& w, const WireNames& W, int32_t pt, uint32_t gid) {
  jw_s(w, "{\"type\":90,\"PT\":");
  jw_i64(w, pt);
  jw_s(w, ",\"ID\":");
  jw_name(w, W, gid);
  jw_s(w, ",\"V\":");
  jw_i64(w, W.version[gid]);
}
__device__ __forceinline__ void jw_ballot(JsonW& w, int32_t bnum, int32_t bcoord) {
  jw_s(w, ",\"B\":\"");
  jw_i64(w, bnum);
  jw_c(w, ':');
  jw_i64(w, bcoord);
  jw_c(w, '"');
}
/* accept_reply_json's object up to QID (AcceptReplyPacket.toJSONSmartImpl :214-224), from reply x of a live group */
__device__ __forceinline__ void jw_reply(JsonW& w, const DevState& S, const WireNames& W, int32_t pt,
                                         const gpx_accept_reply_rec& x) {
  jw_head(w, W, pt, x.gid);
  jw_s(w, ",\"SNDR\":");
  jw_i64(w, group_ctx(S, x.gid).ms->nodes[GPX_WHO_ACC(x.who)]);
  jw_ballot(w, x.bnum, x.bcoord);
  jw_s(w, ",\"S\":");
  jw_i64(w, x.slot);
  jw_s(w, ",\"CP_S\":");
  jw_i64(w, x.max_cp);
  jw_s(w, ",\"QID\":");
  jw_i64(w, x.req_id);
}

/* ,"CA":"/a.b.c.d:port" -- InetSocketAddress.toString() of a literal address */
__device__ __forceinline__ void jw_addr(JsonW& w, const char* key, const uint8_t* ip, uint16_t port) {
  jw_s(w, key);
  for (int j = 0; j < 4; j++) {
    jw_c(w, j ? '.' : '/');
    jw_i64(w, ip[j]);
  }
  jw_c(w, ':');
  jw_i64(w, port);
  jw_c(w, '"');
}
/* request q forwarded alone as a JSON member: request_json (RequestPacket.toJSONSmartImpl :697-742) with forwardCount +
 * 1.  A forwarded request carries no response, no digest and no batched requests, and is not broadcasted. */
__device__ __forceinline__ void jw_request(JsonW& w, const WireNames& W, const WireFwdArgs& F, uint32_t q) {
  const gpx_request_rec rq = F.reqs[q];
  const gpx_wire_req_meta m = F.meta[q];
  jw_head(w, W, GPX_PT_REQUEST, rq.gid);
  jw_s(w, ",\"QID\":");
  jw_i64(w, rq.req_id);
  jw_s(w, ",\"QV\":");
  jw_str(w, F.payload + rq.payload_off, rq.payload_len);
  jw_s(w, ",\"ET\":");
  jw_i64(w, m.entry_time);
  const int32_t fc = fwd_count(F, q);
  if (fc > 0) {
    jw_s(w, ",\"NFWDS\":");
    jw_i64(w, fc);
  }
  if (rq.flags & GPX_F_STOP) jw_s(w, ",\"STOP\":true");
  jw_s(w, ",\"E\":");
  jw_i64(w, rq.entry_node);
  if (m.client_port) jw_addr(w, ",\"CA\":\"", m.client_ip, m.client_port);
  if (m.listen_port) jw_addr(w, ",\"LA\":\"", m.listen_ip, m.listen_port);
  if (m.flags & GPX_RM_RETURN_VALUE) jw_s(w, ",\"QF\":true");
  jw_c(w, '}');
}
/* request q fits in a member: at most 6 bytes per value byte and 2 KiB for the rest (a name of at most 127 bytes,
 * escaped, the keys, numbers and addresses) -- else its exact size */
__device__ __forceinline__ bool jw_request_fits(const WireNames& W, const WireFwdArgs& F, uint32_t q) {
  if (6ull * F.reqs[q].payload_len + 2048u <= GPX_JSON_MAX_MEMBER) return true;
  JsonW w = {nullptr, 0};
  jw_request(w, W, F, q);
  return w.n <= GPX_JSON_MAX_MEMBER;
}

/* the member object of candidate c, which starts a run or a forward: a BatchedAcceptReply
 * (batched_accept_reply_json), a BatchedCommit (batched_commit_json) or a REQUEST (request_json) */
__device__ __forceinline__ void jw_member(JsonW& w, const DevState& S, const WireNames& W, const WireJsonEncArgs& A,
                                          uint32_t c) {
  uint32_t end = 0;
  if (c >= A.R.n + A.D.n) {
    jw_request(w, W, A.F, c - A.R.n - A.D.n);
    return;
  }
  if (c < A.R.n) {
    wire_run<gpx_accept_reply_rec>(A.R, c, end);
    const gpx_accept_reply_rec* recs = reinterpret_cast<const gpx_accept_reply_rec*>(A.R.recs);
    jw_reply(w, S, W, GPX_PT_BATCHED_ACCEPT_REPLY, recs[A.R.perm[c]]);
    jw_s(w, ",\"SLOTS\":[");
    wire_slots_each<gpx_accept_reply_rec>(A.R, c, end, [&](uint32_t k, int32_t s, uint32_t bi) {
      if (k) jw_c(w, ',');
      jw_i64(w, s);
      jw_c(w, ',');
      jw_i64(w, recs[A.R.perm[bi]].req_id);
    });
    jw_s(w, "]}");
    return;
  }
  const uint32_t q = c - A.R.n;
  wire_run<gpx_decision_rec>(A.D, q, end);
  const gpx_decision_rec d = reinterpret_cast<const gpx_decision_rec*>(A.D.recs)[A.D.perm[q]];
  const GroupCtx g = group_ctx(S, d.gid);
  jw_head(w, W, GPX_PT_BATCHED_COMMIT, d.gid);
  jw_ballot(w, d.bnum, d.bcoord);
  jw_s(w, ",\"GC_S\":");
  jw_i64(w, wire_run_median(A.D, q, end));
  jw_s(w, ",\"GROUP\":[");
  for (uint32_t m = 0; m < g.R; m++) {
    if (m) jw_c(w, ',');
    jw_i64(w, g.ms->nodes[m]);
  }
  jw_s(w, "],\"SLOTS\":[");
  wire_slots_each<gpx_decision_rec>(A.D, q, end, [&](uint32_t k, int32_t s, uint32_t) {
    if (k) jw_c(w, ',');
    jw_i64(w, s);
  });
  jw_s(w, "]}");
}

/* ---- kernels ------------------------------------------------------------------------------------------------------ */
/* one thread per reply (after k_wire_enc_keys_replies): a NACK whose destination no local lane serves stays
 * GPX_WE_NACK and is written alone; otherwise it is routed as a positive reply would be */
__global__ void k_json_enc_nacks(const __grid_constant__ DevState S, const __grid_constant__ WireNames W,
                                 const __grid_constant__ WireJsonEncArgs A) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= A.R.n) return;
  uint32_t bytes = 0;
  if (A.R.rstatus[i] == GPX_WE_NACK) {
    const gpx_accept_reply_rec x = reinterpret_cast<const gpx_accept_reply_rec*>(A.R.recs)[i];
    const uint8_t st = wire_reply_route(S, W, x, group_ctx(S, x.gid));
    if (st == GPX_WE_SENT) {
      JsonW w = {nullptr, 0};
      jw_reply(w, S, W, GPX_PT_ACCEPT_REPLY, x);
      bytes = w.n + 1u; /* and '}' */
    } else {
      A.R.rstatus[i] = st;
    }
  }
  A.ncnt[i] = bytes;
  A.ncnt[A.R.n + i] = bytes ? 1u : 0u;
}

/* the lane a commit is sent from: the lane serving its ballot coordinator, else the group's lowest local lane (lane 0
 * when it has none) */
__device__ __forceinline__ uint32_t json_commit_lane(const GroupCtx& g, int32_t bcoord) {
  const uint8_t idx = wire_member_idx(g.ms, g.R, bcoord);
  if (idx != 0xffu && g.ms->lane_of_idx[idx] != 0xffu) return g.ms->lane_of_idx[idx];
  for (uint32_t l = 0; l < GPX_MAX_LANES; l++)
    if (g.ms->lane_mask & (1u << l)) return l;
  return 0;
}

/* one thread per request; the first of a gid's run walks it as k_wire_fwd does, with its statuses.  A GPX_WE_SENT cut
 * of one request whose object fits GPX_JSON_MAX_MEMBER is a member sent from the run's entry lane; every other
 * GPX_WE_SENT cut is a lone REQUEST packet, sized in F.cnt as k_wire_fwd sizes it. */
__global__ void k_json_enc_fwd(const __grid_constant__ DevState S, const __grid_constant__ WireNames W,
                               const __grid_constant__ WireJsonEncArgs A) {
  const WireFwdArgs& F = A.F;
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= F.n) return;
  const uint32_t gid = F.reqs[i].gid;
  if (i > 0 && F.reqs[i - 1].gid == gid) return;
  const uint8_t lane = (uint8_t)((F.reqs[i].flags >> 8) & 0xfu);
  fwd_run(
      S, W, F, i,
      [&](uint32_t k) {
        F.rstatus[k] = GPX_WE_VOID;
        A.fmem[k] = 0;
        F.cnt[k] = F.cnt[F.n + k] = 0;
      },
      [&](uint32_t k, uint32_t b, uint8_t st, int32_t, uint32_t di) {
        for (uint32_t q = k; q < b; q++) {
          F.rstatus[q] = st;
          A.fmem[q] = 0;
          F.cnt[q] = F.cnt[F.n + q] = 0;
        }
        if (st != GPX_WE_SENT) return;
        A.flane[k] = lane;
        A.fdi[k] = (uint8_t)di;
        if (b - k == 1 && jw_request_fits(W, F, k)) {
          A.fmem[k] = 1;
        } else {
          F.cnt[k] = wire_requests_bytes(W, gid, F.reqs, k, b - k);
          F.cnt[F.n + k] = 1;
        }
      });
}

/* one thread per member candidate: the run or forward it starts (if any), its lane, recipient set and size */
__global__ void k_json_enc_members(const __grid_constant__ DevState S, const __grid_constant__ WireNames W,
                                   const __grid_constant__ WireJsonEncArgs A) {
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= A.n) return;
  uint32_t end = 0, set = GPX_JSON_ENC_NONE, lane = 0;
  if (c < A.R.n) {
    if (wire_run<gpx_accept_reply_rec>(A.R, c, end)) {
      const uint32_t i = A.R.perm[c];
      const gpx_accept_reply_rec x = reinterpret_cast<const gpx_accept_reply_rec*>(A.R.recs)[i];
      lane = i % A.R.n_lanes;
      set = A.Z.one[(S.grp_meta[x.gid] & 0xffffu) * GPX_MAX_GROUP_SIZE + GPX_WHO_DST(x.who)];
    }
  } else if (c < A.R.n + A.D.n) {
    if (wire_run<gpx_decision_rec>(A.D, c - A.R.n, end)) {
      const gpx_decision_rec d = reinterpret_cast<const gpx_decision_rec*>(A.D.recs)[A.D.perm[c - A.R.n]];
      lane = json_commit_lane(group_ctx(S, d.gid), d.bcoord);
      set = A.Z.of_mset[S.grp_meta[d.gid] & 0xffffu];
    }
  } else if (A.fmem[c - A.R.n - A.D.n]) {
    const uint32_t q = c - A.R.n - A.D.n;
    lane = A.flane[q];
    set = A.Z.one[(S.grp_meta[A.F.reqs[q].gid] & 0xffffu) * GPX_MAX_GROUP_SIZE + A.fdi[q]];
  }
  A.mset[c] = set;
  A.mlane[c] = (uint8_t)lane;
  uint32_t bytes = 0;
  if (set != GPX_JSON_ENC_NONE) {
    JsonW w = {nullptr, 0};
    jw_member(w, S, W, A, c);
    bytes = w.n;
    atomicMin(&A.first[lane * A.Z.n + set], c);
  }
  A.msize[c] = bytes;
}

/* one thread per candidate: the wrapper sort key */
__global__ void k_json_enc_keys(const __grid_constant__ WireJsonEncArgs A) {
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= A.n) return;
  const uint32_t set = A.mset[c];
  A.key[c] = set == GPX_JSON_ENC_NONE ? GPX_JSON_ENC_NOKEY
                                      : (unsigned long long)A.mlane[c] << 32 | A.first[A.mlane[c] * A.Z.n + set];
}

/* one thread per sorted position: the value the scan by key sums */
__global__ void k_json_enc_vals(const __grid_constant__ WireJsonEncArgs A) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= A.n) return;
  A.val[j] = A.skey[j] == GPX_JSON_ENC_NOKEY ? 0u : A.msize[A.order[j]] + 1u;
}

/* sorted position j holds a member: does it open / close a wrapper?  Member j opens one iff it is the first of its
 * group or floor(start / T) changes; it closes one iff the next member opens one or there is none in the group. */
__device__ __forceinline__ bool json_cut(const WireJsonEncArgs& A, uint32_t j, bool& opens, bool& closes) {
  const unsigned long long k = A.skey[j];
  if (k == GPX_JSON_ENC_NOKEY) return false;
  const uint32_t w = A.start[j] / A.T;
  opens = j == 0 || A.skey[j - 1] != k || A.start[j - 1] / A.T != w;
  closes = j + 1 == A.n || A.skey[j + 1] != k || A.start[j + 1] / A.T != w;
  return true;
}

/* one thread per sorted position: its output bytes, refs, wrappers opened and whether the member is too large */
__global__ void k_json_enc_cut(const __grid_constant__ WireJsonEncArgs A) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= A.n) return;
  bool opens = false, closes = false;
  uint32_t c[JE_NCNT] = {0, 0, 0, 0};
  if (json_cut(A, j, opens, closes)) {
    const uint32_t s = A.val[j] - 1u;
    c[JE_BYTES] = s + (opens ? sizeof(GPX_JSON_WRAP_HEAD) - 1u : 1u) + (closes ? 2u : 0u);
    c[JE_REFS] = opens ? A.Z.count[A.mset[A.order[j]]] : 0u;
    c[JE_OPENS] = opens ? 1u : 0u;
    c[JE_BIG] = s > GPX_JSON_MAX_MEMBER ? 1u : 0u;
  }
  for (int r = 0; r < JE_NCNT; r++) A.cnt[(size_t)r * A.n + j] = c[r];
}

/* one thread per reply: a bare ACCEPT_REPLY (accept_reply_json) for each NACK, in record order */
__global__ void k_json_enc_emit_nacks(const __grid_constant__ DevState S, const __grid_constant__ WireNames W,
                                      const __grid_constant__ WireJsonEncArgs A) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= A.R.n || !A.ncnt[A.R.n + i]) return;
  const gpx_accept_reply_rec x = reinterpret_cast<const gpx_accept_reply_rec*>(A.R.recs)[i];
  JsonW w = {A.out + A.noff[i], 0};
  jw_reply(w, S, W, GPX_PT_ACCEPT_REPLY, x);
  jw_c(w, '}');
  gpx_wire_ref r;
  r.off = A.noff[i];
  r.len = w.n;
  r.gid = x.gid;
  r.node = group_ctx(S, x.gid).ms->nodes[GPX_WHO_DST(x.who)];
  A.refs[A.noff[A.R.n + i]] = r;
}

/* one thread per request: the lone REQUEST packet it heads (fwd_packet), after the bare NACKs, in request order; its ref
 * as k_wire_fwd writes it */
__global__ void k_json_enc_emit_fwd(const __grid_constant__ DevState S, const __grid_constant__ WireNames W,
                                    const __grid_constant__ WireJsonEncArgs A) {
  const WireFwdArgs& F = A.F;
  const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= F.n || !F.cnt[F.n + q]) return;
  const uint32_t gid = F.reqs[q].gid, at = A.nack_bytes + F.off[q];
  gpx_wire_ref r;
  r.off = at;
  r.len = fwd_packet(A.out + at, W, F, gid, q, fwd_cut_end(S, F, q, gid));
  r.gid = gid;
  r.node = S.msets[S.grp_meta[gid] & 0xffffu].nodes[A.fdi[q]];
  A.refs[A.n_nacks + F.off[F.n + q]] = r;
}

/* one thread per sorted position: the member's separator (or its wrapper's head), object and its wrapper's tail */
__global__ void k_json_enc_emit(const __grid_constant__ DevState S, const __grid_constant__ WireNames W,
                                const __grid_constant__ WireJsonEncArgs A) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= A.n) return;
  bool opens = false, closes = false;
  if (!json_cut(A, j, opens, closes)) return;
  const uint32_t at = A.nack_bytes + A.lone_bytes + A.off[(size_t)JE_BYTES * A.n + j];
  JsonW w = {A.out + at, 0};
  if (opens) {
    jw_s(w, GPX_JSON_WRAP_HEAD);
    A.wbeg[A.off[(size_t)JE_OPENS * A.n + j]] =
        make_uint2(at, A.n_nacks + A.n_lone + A.off[(size_t)JE_REFS * A.n + j]);
  } else {
    jw_c(w, ',');
  }
  jw_member(w, S, W, A, A.order[j]);
  if (closes) jw_s(w, "]}");
}

/* one thread per sorted position: the member that closes a wrapper indexes it once per recipient node, ascending; gid =
 * the sending lane */
__global__ void k_json_enc_refs(const __grid_constant__ WireJsonEncArgs A) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= A.n) return;
  bool opens = false, closes = false;
  if (!json_cut(A, j, opens, closes) || !closes) return;
  const uint32_t wi = A.off[(size_t)JE_OPENS * A.n + j] + (opens ? 1u : 0u) - 1u;
  const uint2 b = A.wbeg[wi];
  const uint32_t end =
      A.nack_bytes + A.lone_bytes + A.off[(size_t)JE_BYTES * A.n + j] + A.cnt[(size_t)JE_BYTES * A.n + j];
  const uint32_t c = A.order[j], set = A.mset[c];
  for (uint32_t k = 0; k < A.Z.count[set]; k++) {
    gpx_wire_ref r;
    r.off = b.x;
    r.len = end - b.x;
    r.gid = A.mlane[c];
    r.node = A.Z.nodes[(size_t)set * GPX_MAX_GROUP_SIZE + k];
    A.refs[b.y + k] = r;
  }
}
