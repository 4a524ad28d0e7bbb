/*
 * gpx_wire_json.cuh -- the JSON form of the phase-2 replies and commits on the device (gpx_wire_decode_json_device).
 * A loaded Java peer sends its BatchedAcceptReplies and BatchedCommits as members of a BATCHED_PAXOS_PACKET (type 37,
 * PaxosPacketBatcher.process :270-277, BatchedPaxosPacket.toJSONSmartImpl :87-99) of up to 4 MiB, and its NACKs as
 * singleton ACCEPT_REPLYs (type 8); the schema and the strictness rules are in include/gpx.h.
 *
 * A wrapper is split in parallel, never by one thread walking its bytes:
 *   k_json_pre     one thread per packet: JSON or not, its number of chunks (GPX_JSON_CHUNK bytes aligned to arena
 *                  offsets).
 *   k_json_sum     one thread per chunk: for each of the three lexer states a chunk may start in (outside a string,
 *                  inside one, just after a backslash in one) the state it ends in, its bracket depth delta and the
 *                  lowest depth it reaches.  These summaries compose (JsonCompose), so an exclusive scan by packet
 *                  gives every chunk its true start state and depth.
 *   k_json_struct  one thread per chunk: marks structural errors (a negative depth, an unterminated string, a non-zero
 *                  final depth) and counts, then writes, two kinds of events: a bracket that opens depth 3 (a member
 *                  candidate: an object in the wrapper's PP array) and a bracket that closes to depth 1.
 *   k_json_packet  one thread per packet: the top-level keys; the PP array is jumped over with the depth-1 closes,
 *                  and its member candidates are a binary search in the depth-3 opens.
 *   k_json_member  one thread per member: parses and validates its object, checks the separators up to the next
 *                  member (so the PP array is validated in parallel), looks the name up, writes its status and record
 *                  counts; pass 1 writes its records.
 *   k_json_fix     drops the members of packets a member found malformed.
 * The scans between the launches, the stable radix sort by gid and the gather (k_wire_gather) are gpx_wire_seq.h's
 * wire_decode_json, run with CUB on the device and with the standard library in tests/emu.  Every kernel is scalar, with byte
 * loads only, so the emulation compiles this file for the host with any chunk size.
 */
#pragma once
#include "gpx_wire_dev.cuh"

#ifndef GPX_JSON_CHUNK
#define GPX_JSON_CHUNK 64u
#endif
/* {"type":90,"PT":37,"V":0} (a nested wrapper needs no ID; every other member also has "ID":"" at least): no member
 * with its required keys is shorter, so a PP holding more members than its length / this is malformed */
#define GPX_JSON_MIN_MEMBER 25u
#define GPX_JSON_MAX_SKIP_DEPTH 64u
#define GPX_JSON_NONE 0xffffffffu

/* lexer states */
enum { JS_OUT = 0, JS_IN = 1, JS_ESC = 2 };

/* a chunk's effect for each start state: end state (2 bits per start state), depth delta, lowest running depth */
struct JsonSum {
  int32_t delta[3];
  int32_t mind[3];
  uint32_t end;
};
__host__ __device__ __forceinline__ JsonSum json_identity() {
  JsonSum s;
  for (int k = 0; k < 3; k++) {
    s.delta[k] = 0;
    s.mind[k] = 0;
  }
  s.end = JS_OUT | (JS_IN << 2) | (JS_ESC << 4);
  return s;
}
/* a, then b */
struct JsonCompose {
  __host__ __device__ __forceinline__ JsonSum operator()(const JsonSum& a, const JsonSum& b) const {
    JsonSum r;
    r.end = 0;
    for (uint32_t k = 0; k < 3; k++) {
      const uint32_t m = (a.end >> (2 * k)) & 3u;
      r.end |= ((b.end >> (2 * m)) & 3u) << (2 * k);
      r.delta[k] = a.delta[k] + b.delta[m];
      const int32_t t = a.delta[k] + b.mind[m];
      r.mind[k] = a.mind[k] < t ? a.mind[k] : t;
    }
    return r;
  }
};

__device__ __forceinline__ uint32_t json_lex(uint32_t s, uint32_t c) {
  if (s == JS_ESC) return JS_IN;
  if (s == JS_IN) return c == '\\' ? JS_ESC : c == '"' ? JS_OUT : JS_IN;
  return c == '"' ? JS_IN : JS_OUT;
}
__device__ __forceinline__ int32_t json_bracket(uint32_t c) { /* +1 open, -1 close, 0 other (outside strings) */
  return (c == '{' || c == '[') ? 1 : (c == '}' || c == ']') ? -1 : 0;
}

struct WireJsonArgs {
  const uint8_t* bytes;
  const gpx_wire_ref* pkts;
  uint64_t n_bytes;
  uint32_t n;
  int32_t* status;      /* [n] */
  uint32_t* pcnt;       /* [2][n] chunks (k_json_pre), members (k_json_packet) */
  uint32_t* poff;       /* [2][n] their exclusive prefix sums */
  uint32_t* bad;        /* [n] structure or schema failure */
  uint32_t* pp;         /* [3][n] wrappers: first candidate (index into ev_open), PP's '[' and ']' positions */
  uint32_t cap_items;   /* chunks processed: those past it are never read (the call refuses such a batch) */
  uint32_t* ikey;       /* [cap_items] packet of the chunk (GPX_JSON_NONE past the count) */
  JsonSum* isum;        /* [cap_items] */
  JsonSum* ipre;        /* [cap_items] exclusive prefix by packet */
  uint32_t* ecnt;       /* [2][cap_items] depth-3 opens, depth-1 closes */
  uint32_t* eoff;       /* [2][cap_items] */
  uint32_t* ev_open;    /* positions (arena offsets) */
  uint32_t* ev_close;
  uint32_t cap_mem;     /* member slots */
  gpx_wire_member* mem; /* [cap_mem] members in packet order */
  uint32_t* mcnt;       /* [3][cap_mem] listed, replies, decisions */
  uint32_t* moff;       /* [3][cap_mem] */
  /* pass 1 */
  gpx_wire_member* mem_out;
  gpx_accept_reply_rec* rep;
  gpx_decision_rec* dec;
  uint32_t* rep_key;
  uint32_t* dec_key;
  int emit;
};

__device__ __forceinline__ bool json_ws(uint32_t c) { return c == ' ' || c == '\t' || c == '\n' || c == '\r'; }

/* chunks of packet [off, off + len) */
__device__ __forceinline__ uint32_t json_chunks(uint32_t off, uint32_t len) {
  return len ? (off + len - 1) / GPX_JSON_CHUNK - off / GPX_JSON_CHUNK + 1u : 0u;
}
/* the last index k of sorted off[0..n) with off[k] <= i */
__device__ __forceinline__ uint32_t json_upper(const uint32_t* off, uint32_t n, uint32_t i) {
  uint32_t lo = 0, hi = n;
  while (lo < hi) {
    const uint32_t m = (lo + hi) >> 1;
    if (off[m] <= i) lo = m + 1;
    else hi = m;
  }
  return lo - 1u;
}
/* the first index in [lo, hi) of sorted v with v[i] > x */
__device__ __forceinline__ uint32_t json_first_above(const uint32_t* v, uint32_t lo, uint32_t hi, uint32_t x) {
  while (lo < hi) {
    const uint32_t m = (lo + hi) >> 1;
    if (v[m] <= x) lo = m + 1;
    else hi = m;
  }
  return lo;
}

/* one thread per packet: status (GPX_WS_OK for JSON, pending its parse) and its chunks */
__global__ void k_json_pre(const __grid_constant__ WireJsonArgs A) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= A.n) return;
  const gpx_wire_ref r = A.pkts[k];
  int32_t st = GPX_WS_UNHANDLED;
  if ((uint64_t)r.off + r.len > A.n_bytes) {
    st = GPX_WS_MALFORMED;
  } else {
    uint32_t i = 0;
    while (i < r.len && json_ws(A.bytes[r.off + i])) i++;
    if (i < r.len && A.bytes[r.off + i] == '{') st = GPX_WS_OK;
  }
  A.status[k] = st;
  A.pcnt[k] = st == GPX_WS_OK ? json_chunks(r.off, r.len) : 0u;
  A.pcnt[A.n + k] = 0;
  A.bad[k] = 0;
  A.pp[k] = 0;
  A.pp[A.n + k] = GPX_JSON_NONE; /* not a wrapper */
  A.pp[2 * A.n + k] = GPX_JSON_NONE;
}

/* chunk i: its packet and byte range; false past the device count of chunks */
__device__ __forceinline__ bool json_item(const WireJsonArgs& A, uint32_t i, uint32_t& k, uint32_t& a, uint32_t& b,
                                          bool& last) {
  const uint32_t total = A.poff[A.n - 1] + A.pcnt[A.n - 1];
  if (i >= total) return false;
  k = json_upper(A.poff, A.n, i);
  const gpx_wire_ref r = A.pkts[k];
  const uint32_t j = i - A.poff[k];
  const uint32_t c = r.off / GPX_JSON_CHUNK + j;
  a = c * GPX_JSON_CHUNK > r.off ? c * GPX_JSON_CHUNK : r.off;
  const uint32_t ce = (c + 1u) * GPX_JSON_CHUNK, pe = r.off + r.len;
  b = ce < pe ? ce : pe;
  last = j + 1u == A.pcnt[k];
  return true;
}

/* one thread per chunk slot (cap_items of them): the chunk's summary and its scan key */
__global__ void k_json_sum(const __grid_constant__ WireJsonArgs A) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= A.cap_items) return;
  uint32_t k, a, b;
  bool last;
  if (!json_item(A, i, k, a, b, last)) {
    A.ikey[i] = GPX_JSON_NONE;
    A.isum[i] = json_identity();
    return;
  }
  uint32_t s[3] = {JS_OUT, JS_IN, JS_ESC};
  int32_t d[3] = {0, 0, 0}, m[3] = {0, 0, 0};
  for (uint32_t p = a; p < b; p++) {
    const uint32_t c = A.bytes[p];
    for (int q = 0; q < 3; q++) {
      if (s[q] == JS_OUT) {
        d[q] += json_bracket(c);
        m[q] = d[q] < m[q] ? d[q] : m[q];
      }
      s[q] = json_lex(s[q], c);
    }
  }
  JsonSum r;
  r.end = s[0] | (s[1] << 2) | (s[2] << 4);
  for (int q = 0; q < 3; q++) {
    r.delta[q] = d[q];
    r.mind[q] = m[q];
  }
  A.ikey[i] = k;
  A.isum[i] = r;
}

/* one thread per chunk slot, with its start state and depth from the scan: structural errors, then the events (pass 0
 * counts them, pass 1 writes them at the scanned offsets) */
__global__ void k_json_struct(const __grid_constant__ WireJsonArgs A) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= A.cap_items) return;
  uint32_t k, a, b;
  bool last;
  if (!json_item(A, i, k, a, b, last)) {
    if (!A.emit) A.ecnt[i] = A.ecnt[A.cap_items + i] = 0;
    return;
  }
  const JsonSum pre = A.ipre[i];
  uint32_t s = pre.end & 3u;
  int32_t d = pre.delta[0];
  uint32_t n3 = 0, n1 = 0, o3 = 0, o1 = 0;
  if (A.emit) {
    o3 = A.eoff[i];
    o1 = A.eoff[A.cap_items + i];
  }
  bool neg = d < 0;
  for (uint32_t p = a; p < b; p++) {
    const uint32_t c = A.bytes[p];
    if (s == JS_OUT) {
      const int32_t t = json_bracket(c);
      d += t;
      if (d < 0) neg = true;
      if (t > 0 && d == 3) {
        if (A.emit) A.ev_open[o3 + n3] = p;
        n3++;
      } else if (t < 0 && d == 1) {
        if (A.emit) A.ev_close[o1 + n1] = p;
        n1++;
      }
    }
    s = json_lex(s, c);
  }
  if (A.emit) return;
  A.ecnt[i] = n3;
  A.ecnt[A.cap_items + i] = n1;
  if (neg || (last && (s != JS_OUT || d != 0))) A.bad[k] = 1u;
}

/* ---- the serial parser of one object (a packet's top level, or a member) ------------------------------------------ */
struct JRd {
  const uint8_t* b; /* the arena; positions are arena offsets */
  uint32_t n, end;
  bool ok;
};
__device__ __forceinline__ void jr_ws(JRd& J) {
  while (J.n < J.end && json_ws(J.b[J.n])) J.n++;
}
__device__ __forceinline__ uint32_t jr_peek(const JRd& J) { return J.n < J.end ? J.b[J.n] : 0u; }
__device__ __forceinline__ bool jr_eat(JRd& J, uint32_t c) {
  if (J.ok && J.n < J.end && J.b[J.n] == c) {
    J.n++;
    return true;
  }
  J.ok = false;
  return false;
}
__device__ __forceinline__ int32_t json_hex(uint32_t c) {
  if (c >= '0' && c <= '9') return (int32_t)(c - '0');
  if (c >= 'a' && c <= 'f') return (int32_t)(c - 'a' + 10);
  if (c >= 'A' && c <= 'F') return (int32_t)(c - 'A' + 10);
  return -1;
}
/* inside a string: 0 and the next character in *u, 1 at the closing quote (consumed), -1 on an error (J.ok false) */
__device__ __forceinline__ int jr_unit(JRd& J, uint32_t* u) {
  if (!J.ok || J.n >= J.end) {
    J.ok = false;
    return -1;
  }
  uint32_t c = J.b[J.n++];
  if (c == '"') return 1;
  if (c < 0x20u) { /* a raw control character */
    J.ok = false;
    return -1;
  }
  if (c != '\\') {
    *u = c; /* 0x80-0xff: ISO-8859-1 */
    return 0;
  }
  if (J.n >= J.end) {
    J.ok = false;
    return -1;
  }
  c = J.b[J.n++];
  switch (c) {
    case '"': case '\\': case '/': *u = c; return 0;
    case 'b': *u = 8; return 0;
    case 'f': *u = 12; return 0;
    case 'n': *u = 10; return 0;
    case 'r': *u = 13; return 0;
    case 't': *u = 9; return 0;
    case 'u': {
      if (J.end - J.n < 4) break;
      uint32_t v = 0;
      for (int q = 0; q < 4; q++) {
        const int32_t h = json_hex(J.b[J.n + q]);
        if (h < 0) {
          J.ok = false;
          return -1;
        }
        v = (v << 4) | (uint32_t)h;
      }
      J.n += 4;
      *u = v;
      return 0;
    }
    default: break;
  }
  J.ok = false;
  return -1;
}
/* a string at J.n: its characters' count, whether one is above U+00FF, the first 8 packed (for key names) */
struct JStr {
  uint32_t len;
  bool wide, esc;
  uint64_t head;
};
__device__ __forceinline__ JStr jr_string(JRd& J) {
  JStr s;
  s.len = 0;
  s.wide = s.esc = false;
  s.head = 0;
  if (!jr_eat(J, '"')) return s;
  for (;;) {
    uint32_t u = 0;
    const uint32_t at = J.n;
    const int r = jr_unit(J, &u);
    if (r != 0) break;
    if (J.n - at > 1) s.esc = true;
    if (u > 0xffu) s.wide = true;
    if (s.len < 8) s.head |= (uint64_t)(u & 0xffu) << (8 * s.len);
    s.len++;
  }
  return s;
}
/* a JSON integer (no fraction, exponent, leading zero or '+') within [lo, hi] */
__device__ __forceinline__ int64_t jr_int(JRd& J, int64_t lo, int64_t hi) {
  const bool neg = jr_peek(J) == '-';
  if (neg) J.n++;
  const uint32_t c0 = jr_peek(J);
  if (c0 < '0' || c0 > '9') {
    J.ok = false;
    return 0;
  }
  uint64_t mag = 0;
  uint32_t nd = 0;
  while (J.n < J.end && J.b[J.n] >= '0' && J.b[J.n] <= '9') {
    const uint32_t dgt = J.b[J.n] - '0';
    if (mag > (0x8000000000000000ull - dgt) / 10u) J.ok = false; /* beyond 2^63 */
    else mag = mag * 10u + dgt;
    J.n++;
    nd++;
  }
  if (c0 == '0' && nd > 1) J.ok = false;
  const uint32_t c = jr_peek(J);
  if (c == '.' || c == 'e' || c == 'E') J.ok = false;
  if (!J.ok) return 0;
  if (!neg && mag > (uint64_t)hi) J.ok = false;
  if (neg && mag > (uint64_t)(-(lo + 1)) + 1u) J.ok = false;
  if (!J.ok) return 0;
  return neg ? (int64_t)(0ull - mag) : (int64_t)mag;
}
__device__ __forceinline__ int32_t jr_i32(JRd& J) { return (int32_t)jr_int(J, INT32_MIN, INT32_MAX); }
__device__ __forceinline__ int64_t jr_i64(JRd& J) { return jr_int(J, INT64_MIN, INT64_MAX); }

/* any JSON number (the value of a key that is skipped) */
__device__ __forceinline__ void jr_number(JRd& J) {
  if (jr_peek(J) == '-') J.n++;
  const uint32_t c0 = jr_peek(J);
  if (c0 < '0' || c0 > '9') {
    J.ok = false;
    return;
  }
  J.n++;
  if (c0 != '0')
    while (jr_peek(J) >= '0' && jr_peek(J) <= '9') J.n++;
  if (jr_peek(J) == '.') {
    J.n++;
    if (jr_peek(J) < '0' || jr_peek(J) > '9') J.ok = false;
    while (jr_peek(J) >= '0' && jr_peek(J) <= '9') J.n++;
  }
  if (jr_peek(J) == 'e' || jr_peek(J) == 'E') {
    J.n++;
    if (jr_peek(J) == '+' || jr_peek(J) == '-') J.n++;
    if (jr_peek(J) < '0' || jr_peek(J) > '9') J.ok = false;
    while (jr_peek(J) >= '0' && jr_peek(J) <= '9') J.n++;
  }
}
__device__ __forceinline__ bool jr_word(JRd& J, const char* w, uint32_t n) {
  if (J.end - J.n < n) return J.ok = false;
  for (uint32_t q = 0; q < n; q++)
    if (J.b[J.n + q] != (uint8_t)w[q]) return J.ok = false;
  J.n += n;
  return true;
}
/* one scalar value */
__device__ __forceinline__ void jr_scalar(JRd& J) {
  const uint32_t c = jr_peek(J);
  if (c == '"') jr_string(J);
  else if (c == 't') jr_word(J, "true", 4);
  else if (c == 'f') jr_word(J, "false", 5);
  else if (c == 'n') jr_word(J, "null", 4);
  else jr_number(J);
}
/* skips one value, validating it; nesting deeper than GPX_JSON_MAX_SKIP_DEPTH inside it is malformed */
__device__ void jr_skip(JRd& J) {
  uint64_t obj = 0; /* bit d: container d is an object */
  uint32_t d = 0;
  bool want_key = false;
  while (J.ok) {
    jr_ws(J);
    if (want_key) {
      jr_string(J);
      jr_ws(J);
      jr_eat(J, ':');
      jr_ws(J);
      want_key = false;
    }
    const uint32_t c = jr_peek(J);
    if (c == '{' || c == '[') {
      J.n++;
      jr_ws(J);
      if (jr_peek(J) == (c == '{' ? '}' : ']')) {
        J.n++;
      } else {
        if (d >= GPX_JSON_MAX_SKIP_DEPTH) {
          J.ok = false;
          return;
        }
        obj = c == '{' ? (obj | (1ull << d)) : (obj & ~(1ull << d));
        d++;
        want_key = c == '{';
        continue;
      }
    } else {
      jr_scalar(J);
    }
    /* after a value: close containers or move to the next element */
    for (;;) {
      if (!J.ok || d == 0) return;
      jr_ws(J);
      const bool is_obj = (obj >> (d - 1)) & 1u;
      const uint32_t e = jr_peek(J);
      if (e == ',') {
        J.n++;
        want_key = is_obj;
        break;
      }
      if (e == (is_obj ? '}' : ']')) {
        J.n++;
        d--;
        continue;
      }
      J.ok = false;
      return;
    }
  }
}

/* the keys the schema knows, as up to 8 ISO-8859-1 characters packed little-endian */
#define JK(a, b, c, d, e) ((uint64_t)(a) | ((uint64_t)(b) << 8) | ((uint64_t)(c) << 16) | ((uint64_t)(d) << 24) | ((uint64_t)(e) << 32))
#define JK8(a, b, c, d, e, f, g, h) (JK(a, b, c, d, e) | ((uint64_t)(f) << 40) | ((uint64_t)(g) << 48) | ((uint64_t)(h) << 56))
enum { JK_TYPE, JK_PT, JK_ID, JK_V, JK_SNDR, JK_B, JK_S, JK_CP_S, JK_QID, JK_NACK, JK_SLOTS, JK_GC_S, JK_GROUP, JK_PP, JK_N };
__device__ __forceinline__ int json_key(const JStr& s) {
  if (s.wide) return -1;
  switch (s.len) {
    case 1:
      if (s.head == 'V') return JK_V;
      if (s.head == 'B') return JK_B;
      if (s.head == 'S') return JK_S;
      return -1;
    case 2:
      if (s.head == JK('P', 'T', 0, 0, 0)) return JK_PT;
      if (s.head == JK('I', 'D', 0, 0, 0)) return JK_ID;
      if (s.head == JK('P', 'P', 0, 0, 0)) return JK_PP;
      return -1;
    case 3: return s.head == JK('Q', 'I', 'D', 0, 0) ? JK_QID : -1;
    case 4:
      if (s.head == JK('t', 'y', 'p', 'e', 0)) return JK_TYPE;
      if (s.head == JK('S', 'N', 'D', 'R', 0)) return JK_SNDR;
      if (s.head == JK('C', 'P', '_', 'S', 0)) return JK_CP_S;
      if (s.head == JK('N', 'A', 'C', 'K', 0)) return JK_NACK;
      if (s.head == JK('G', 'C', '_', 'S', 0)) return JK_GC_S;
      return -1;
    case 5:
      if (s.head == JK('S', 'L', 'O', 'T', 'S')) return JK_SLOTS;
      if (s.head == JK('G', 'R', 'O', 'U', 'P')) return JK_GROUP;
      return -1;
    default: return -1;
  }
}

/* the key table of the packets and members above: json_key, JK_N of them, JK_PP the array a top level jumps over.
 * A table's id() sees the key's JStr, and the reader and the key's opening quote for a key longer than JStr.head. */
struct JsonPktKeys {
  enum { N = JK_N, PP = JK_PP };
  __device__ __forceinline__ static int id(const JStr& s, const JRd&, uint32_t) { return json_key(s); }
};
/* the key string at `at` (JStr s) goes on after its first 8 characters with the n characters of rest */
__device__ __forceinline__ bool json_key_rest(const JRd& J0, uint32_t at, const JStr& s, const char* rest, uint32_t n) {
  if (s.len != 8u + n) return false;
  JRd J = J0;
  J.n = at + 1u;
  for (uint32_t q = 0; q < s.len; q++) {
    uint32_t u = 0;
    if (jr_unit(J, &u) != 0 || (q >= 8u && u != (uint8_t)rest[q - 8u])) return false;
  }
  return true;
}

/* the PP jump of a packet's top level: PP's '[' at p closes at the first depth-1 close after p */
struct JsonJump {
  const uint32_t* close;
  uint32_t lo, hi;
};
/* phase 1 of an object at J.n: every key's value is validated (the PP array of a top level only by its members'
 * threads: jumped over) and the last position of each known key's value kept (0 = absent: a value is never at
 * arena offset 0).  pp_close: the ']' of the jumped PP.  Keys: the key table (JsonPktKeys, or a table without a PP
 * whose PP is -2, which no key has). */
template <typename Keys>
__device__ __forceinline__ void json_keys_t(JRd& J, uint32_t* pos, const JsonJump* jump, uint32_t* pp_close) {
  constexpr int JK_N = Keys::N, JK_PP = Keys::PP;
  for (int q = 0; q < JK_N; q++) pos[q] = 0;
  jr_ws(J);
  jr_eat(J, '{');
  jr_ws(J);
  if (jr_peek(J) == '}') {
    J.n++;
    return;
  }
  while (J.ok) {
    jr_ws(J);
    const uint32_t kat = J.n;
    const JStr key = jr_string(J);
    jr_ws(J);
    jr_eat(J, ':');
    jr_ws(J);
    if (!J.ok) return;
    const int kid = Keys::id(key, J, kat);
    if (kid == JK_PP && *pp_close != GPX_JSON_NONE) { /* a duplicated PP: validate the jumped one, the last counts */
      JRd V = J;
      V.n = pos[JK_PP];
      jr_skip(V);
      if (!V.ok || V.n != *pp_close + 1u) {
        J.ok = false;
        return;
      }
      *pp_close = GPX_JSON_NONE;
    }
    if (kid >= 0) pos[kid] = J.n;
    if (kid == JK_PP && jump && jr_peek(J) == '[') {
      const uint32_t c = json_first_above(jump->close, jump->lo, jump->hi, J.n);
      if (c >= jump->hi || J.b[jump->close[c]] != ']') {
        J.ok = false;
        return;
      }
      *pp_close = jump->close[c];
      J.n = *pp_close + 1u;
    } else {
      jr_skip(J);
    }
    jr_ws(J);
    if (jr_peek(J) == ',') {
      J.n++;
      continue;
    }
    jr_eat(J, '}');
    return;
  }
}
__device__ __forceinline__ void json_keys(JRd& J, uint32_t* pos, const JsonJump* jump, uint32_t* pp_close) {
  json_keys_t<JsonPktKeys>(J, pos, jump, pp_close);
}
__device__ __forceinline__ bool json_at(JRd& J, uint32_t at) {
  if (!at) return false;
  J.n = at;
  return true;
}
/* a required int32 at pos (false: absent or not an int32) */
__device__ __forceinline__ bool json_get_i32(const JRd& J0, uint32_t at, int32_t* v) {
  JRd J = J0;
  if (!json_at(J, at)) return false;
  *v = jr_i32(J);
  return J.ok;
}
/* "<int32>:<int32>", an optional '-' before each */
__device__ __forceinline__ bool json_get_ballot(const JRd& J0, uint32_t at, int32_t* bnum, int32_t* bcoord) {
  JRd J = J0;
  if (!json_at(J, at) || !jr_eat(J, '"')) return false;
  int32_t out[2] = {0, 0};
  for (int part = 0; part < 2; part++) {
    uint32_t u = 0;
    int r = jr_unit(J, &u);
    const bool neg = r == 0 && u == '-';
    if (neg) r = jr_unit(J, &u);
    uint64_t mag = 0;
    uint32_t nd = 0;
    bool lead0 = false;
    while (r == 0 && u >= '0' && u <= '9') {
      if (nd == 0) lead0 = u == '0';
      mag = mag * 10u + (u - '0');
      if (mag > 0x80000000ull) return false;
      nd++;
      r = jr_unit(J, &u);
    }
    if (nd == 0 || (lead0 && nd > 1)) return false;
    if ((!neg && mag > 0x7fffffffull)) return false;
    out[part] = neg ? (int32_t)(0u - (uint32_t)mag) : (int32_t)mag;
    if (part == 0 && !(r == 0 && u == ':')) return false;
    if (part == 1 && r != 1) return false;
  }
  *bnum = out[0];
  *bcoord = out[1];
  return J.ok;
}
/* an array of integers at pos: its length; int32 everywhere, or (pairs) int32 at even and int64 at odd indices.
 * With out != nullptr, element j is handed to out->put(j, value). */
struct JsonNoSink {
  __device__ __forceinline__ void put(uint32_t, int64_t) {}
};
template <typename Sink>
__device__ __forceinline__ bool json_get_ints(const JRd& J0, uint32_t at, bool pairs, uint32_t* count, Sink* out) {
  JRd J = J0;
  if (!json_at(J, at) || !jr_eat(J, '[')) return false;
  uint32_t j = 0;
  jr_ws(J);
  if (jr_peek(J) == ']') {
    *count = 0;
    return true;
  }
  while (J.ok) {
    jr_ws(J);
    const int64_t v = (pairs && (j & 1u)) ? jr_i64(J) : (int64_t)jr_i32(J);
    if (!J.ok) return false;
    if (out) out->put(j, v);
    j++;
    jr_ws(J);
    if (jr_peek(J) == ',') {
      J.n++;
      continue;
    }
    if (!jr_eat(J, ']')) return false;
    break;
  }
  *count = j;
  return J.ok;
}

/* ---- packets ---------------------------------------------------------------------------------------------------- */
/* one thread per packet: the top level.  A wrapper (PT 37) gets the member candidates inside its PP array; a bare
 * ACCEPT_REPLY / BatchedAcceptReply / BatchedCommit one member, the whole packet; any other type is unhandled. */
__global__ void k_json_packet(const __grid_constant__ WireJsonArgs A) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= A.n) return;
  if (A.status[k] != GPX_WS_OK) return;
  int32_t st = GPX_WS_OK;
  const gpx_wire_ref r = A.pkts[k];
  const uint32_t ib = A.poff[k], ni = A.pcnt[k];
  uint32_t members = 0;
  if (A.bad[k] || ib + ni > A.cap_items) {
    st = GPX_WS_MALFORMED;
  } else {
    const uint32_t il = ib + ni - 1u;
    JsonJump jump;
    jump.close = A.ev_close;
    jump.lo = A.eoff[A.cap_items + ib];
    jump.hi = A.eoff[A.cap_items + il] + A.ecnt[A.cap_items + il];
    JRd J;
    J.b = A.bytes;
    J.n = r.off;
    J.end = r.off + r.len;
    J.ok = true;
    uint32_t pos[JK_N], ppc = GPX_JSON_NONE;
    json_keys(J, pos, &jump, &ppc);
    jr_ws(J);
    if (J.n != J.end) J.ok = false; /* trailing bytes */
    int32_t type = 0, pt = 0, ver = 0;
    if (!J.ok || !json_get_i32(J, pos[JK_TYPE], &type) || type != GPX_PT_PAXOS_PACKET || !json_get_i32(J, pos[JK_PT], &pt)) {
      st = GPX_WS_MALFORMED;
    } else if (pt == 37) { /* BatchedPaxosPacket: no ID, version -1, PP an array of objects */
      if (pos[JK_ID] || !json_get_i32(J, pos[JK_V], &ver) || ver != -1 || !pos[JK_PP] || J.b[pos[JK_PP]] != '[' ||
          ppc == GPX_JSON_NONE) {
        st = GPX_WS_MALFORMED;
      } else {
        const uint32_t p = pos[JK_PP];
        const uint32_t olo = A.eoff[ib], ohi = A.eoff[il] + A.ecnt[il];
        const uint32_t lo = json_first_above(A.ev_open, olo, ohi, p);
        const uint32_t hi = json_first_above(A.ev_open, lo, ohi, ppc);
        members = hi - lo;
        if ((uint64_t)members * GPX_JSON_MIN_MEMBER > ppc - p - 1u) {
          st = GPX_WS_MALFORMED; /* a member too short to hold its required keys */
          members = 0;
        } else if (members == 0) { /* empty PP: nothing but whitespace inside */
          for (uint32_t q = p + 1; q < ppc; q++)
            if (!json_ws(J.b[q])) {
              st = GPX_WS_MALFORMED;
              break;
            }
        }
        A.pp[k] = lo;
        A.pp[A.n + k] = p;
        A.pp[2 * A.n + k] = ppc;
      }
    } else {
      if (ppc != GPX_JSON_NONE) { /* a jumped PP of another type: validate it here */
        JRd V = J;
        V.n = pos[JK_PP];
        jr_skip(V);
        if (!V.ok || V.n != ppc + 1u) st = GPX_WS_MALFORMED;
      }
      if (st == GPX_WS_OK) {
        if (pt == GPX_PT_ACCEPT_REPLY || pt == GPX_PT_BATCHED_ACCEPT_REPLY || pt == GPX_PT_BATCHED_COMMIT) members = 1;
        else st = GPX_WS_UNHANDLED;
      }
    }
  }
  if (st != GPX_WS_OK) members = 0;
  A.status[k] = st;
  A.pcnt[A.n + k] = members;
}

/* ---- members ---------------------------------------------------------------------------------------------------- */
struct JsonRepSink { /* BatchedAcceptReply SLOTS: [slot, requestID, ...] */
  gpx_accept_reply_rec x;
  gpx_accept_reply_rec* out;
  uint32_t* key;
  __device__ __forceinline__ void put(uint32_t j, int64_t v) {
    if (!(j & 1u)) {
      x.slot = (int32_t)v;
      return;
    }
    x.req_id = v;
    out[j >> 1] = x;
    key[j >> 1] = x.gid;
  }
};
struct JsonDecSink { /* BatchedCommit SLOTS */
  gpx_decision_rec d;
  gpx_decision_rec* out;
  uint32_t* key;
  __device__ __forceinline__ void put(uint32_t j, int64_t v) {
    d.slot = (int32_t)v;
    out[j] = d;
    key[j] = d.gid;
  }
};

/* the gid named by the "ID" string at `at` (id: what jr_string read of it), unescaped before the lookup, or
 * GPX_NAME_NONE; a name with a character above U+00FF or longer than GPX_WIRE_MAX_ID names no gid */
__device__ __forceinline__ uint32_t json_id_gid(const WireNames& W, const JRd& J, uint32_t at, const JStr& id) {
  if (id.wide || id.len > GPX_WIRE_MAX_ID) return GPX_NAME_NONE;
  uint8_t buf[GPX_WIRE_MAX_ID];
  const uint8_t* name = J.b + at + 1u;
  if (id.esc) {
    JRd I = J;
    I.n = at + 1u;
    uint32_t u = 0;
    for (uint32_t q = 0; q < id.len; q++) {
      jr_unit(I, &u);
      buf[q] = (uint8_t)u;
    }
    name = buf;
  }
  return wire_name_find(W, name, id.len);
}

/* one thread per member (the device count of them; cap_mem slots).  Pass 0: parse and validate the member, the
 * separators after it, its name, version and locality: status and record counts, the packet's bad flag on a schema
 * failure.  Pass 1 (members kept): the member row and the records at the scanned offsets. */
__global__ void k_json_member(const __grid_constant__ DevState S, const __grid_constant__ WireNames W,
                              const __grid_constant__ WireJsonArgs A) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= A.cap_mem) return;
  const uint32_t* moffs = A.poff + A.n;
  const uint32_t* mcnts = A.pcnt + A.n;
  const uint32_t total = moffs[A.n - 1] + mcnts[A.n - 1];
  if (i >= total) {
    if (!A.emit) A.mcnt[i] = A.mcnt[A.cap_mem + i] = A.mcnt[2 * A.cap_mem + i] = 0;
    return;
  }
  if (A.emit && A.mcnt[i] == 0) return;
  const uint32_t k = json_upper(moffs, A.n, i);
  const uint32_t j = i - moffs[k], m = mcnts[k];
  const gpx_wire_ref r = A.pkts[k];
  const bool bare = A.pp[A.n + k] == GPX_JSON_NONE;
  JRd J;
  J.b = A.bytes;
  J.ok = true;
  uint32_t at, end;
  if (A.emit) { /* the span pass 0 found (the event lists are gone by now) */
    at = A.mem[i].off;
    end = at + A.mem[i].len;
  } else if (bare) {
    at = r.off;
    end = r.off + r.len;
  } else {
    at = A.ev_open[A.pp[k] + j];
    end = A.pp[2 * A.n + k];
  }
  J.n = at;
  J.end = end;
  uint32_t pos[JK_N], ppc = GPX_JSON_NONE;
  if (!bare && J.b[at] != '{') J.ok = false;
  json_keys(J, pos, nullptr, &ppc);
  const uint32_t mend = J.n;
  /* what may follow: the rest of a bare packet is whitespace; in PP, whitespace, then ',' before the next member */
  bool ok = J.ok;
  if (ok && !A.emit) {
    if (bare) {
      jr_ws(J);
      ok = J.n == J.end;
    } else {
      jr_ws(J);
      if (j + 1u < m) {
        ok = jr_peek(J) == ',';
        J.n++;
        jr_ws(J);
        ok = ok && J.n == A.ev_open[A.pp[k] + j + 1u];
      } else {
        ok = J.n == end;
      }
      if (j == 0) { /* between PP's '[' and the first member */
        for (uint32_t q = A.pp[A.n + k] + 1u; q < at && ok; q++)
          if (!json_ws(J.b[q])) ok = false;
      }
    }
  }
  J.ok = true;
  int32_t type = 0, pt = 0, ver = 0, sndr = 0, slot = 0, cp = 0, gc = 0, bnum = 0, bcoord = 0;
  int64_t qid = 0;
  bool nack = false;
  uint32_t n_slots = 0, n_group = 0;
  ok = ok && json_get_i32(J, pos[JK_TYPE], &type) && type == GPX_PT_PAXOS_PACKET && json_get_i32(J, pos[JK_PT], &pt);
  JStr id;
  id.len = 0;
  id.wide = id.esc = false;
  if (ok && pt != 37) {
    ok = pos[JK_ID] != 0;
    if (ok) {
      JRd I = J;
      I.n = pos[JK_ID];
      id = jr_string(I);
      ok = I.ok;
    }
  }
  ok = ok && json_get_i32(J, pos[JK_V], &ver);
  const bool reply = pt == GPX_PT_ACCEPT_REPLY || pt == GPX_PT_BATCHED_ACCEPT_REPLY;
  if (ok && reply) {
    ok = json_get_i32(J, pos[JK_SNDR], &sndr) && json_get_ballot(J, pos[JK_B], &bnum, &bcoord) &&
         json_get_i32(J, pos[JK_S], &slot) && json_get_i32(J, pos[JK_CP_S], &cp) && pos[JK_QID] != 0;
    if (ok) {
      JRd Q = J;
      Q.n = pos[JK_QID];
      qid = jr_i64(Q);
      ok = Q.ok;
    }
    if (ok && pos[JK_NACK]) {
      JRd Q = J;
      Q.n = pos[JK_NACK];
      if (jr_peek(Q) == 't') nack = jr_word(Q, "true", 4);
      else ok = jr_word(Q, "false", 5);
    }
    if (ok && pt == GPX_PT_BATCHED_ACCEPT_REPLY)
      ok = json_get_ints<JsonNoSink>(J, pos[JK_SLOTS], true, &n_slots, nullptr) && (n_slots & 1u) == 0;
  } else if (ok && pt == GPX_PT_BATCHED_COMMIT) {
    ok = json_get_ballot(J, pos[JK_B], &bnum, &bcoord) && json_get_i32(J, pos[JK_GC_S], &gc) &&
         json_get_ints<JsonNoSink>(J, pos[JK_GROUP], false, &n_group, nullptr) &&
         json_get_ints<JsonNoSink>(J, pos[JK_SLOTS], false, &n_slots, nullptr);
  }
  int32_t st = GPX_WS_OK;
  if (!ok) st = GPX_WS_MALFORMED;
  else if (!(reply || pt == GPX_PT_BATCHED_COMMIT) || (pt == GPX_PT_ACCEPT_REPLY && nack)) st = GPX_WS_UNHANDLED;
  uint32_t gid = GPX_NAME_NONE;
  GroupCtx g;
  uint8_t acc_idx = 0xffu, dst_idx = 0xffu;
  if (st == GPX_WS_OK) {
    gid = json_id_gid(W, J, pos[JK_ID], id);
    st = wire_group(S, W, gid, ver, g);
  }
  if (st == GPX_WS_OK) {
    if (reply) {
      acc_idx = wire_member_idx(g.ms, g.R, sndr);
      /* a singleton reply goes to the node that received it: a NACK's ballot names another coordinator */
      dst_idx = wire_member_idx(g.ms, g.R, pt == GPX_PT_ACCEPT_REPLY ? r.node : bcoord);
      if (acc_idx == 0xffu || (pt == GPX_PT_BATCHED_ACCEPT_REPLY && dst_idx == 0xffu)) st = GPX_WS_MALFORMED;
      else if (dst_idx == 0xffu || g.ms->lane_of_idx[dst_idx] == 0xffu) st = GPX_WS_NOT_LOCAL;
    } else if (g.ms->lane_mask == 0) {
      st = GPX_WS_NOT_LOCAL;
    }
  }
  if (!A.emit) {
    if (st == GPX_WS_MALFORMED && !ok) A.bad[k] = 1u; /* a schema failure loses the whole packet */
    gpx_wire_member w;
    w.pkt = k;
    w.off = bare ? r.off : at;
    w.len = bare ? r.len : mend - at;
    w.status = st;
    A.mem[i] = w;
    A.mcnt[i] = 1u;
    A.mcnt[A.cap_mem + i] = st == GPX_WS_OK && reply ? (pt == GPX_PT_ACCEPT_REPLY ? 1u : n_slots / 2u) : 0u;
    A.mcnt[2 * A.cap_mem + i] = st == GPX_WS_OK && pt == GPX_PT_BATCHED_COMMIT ? n_slots : 0u;
    return;
  }
  A.mem_out[A.moff[i]] = A.mem[i];
  if (st != GPX_WS_OK) return;
  if (reply) {
    JsonRepSink s;
    s.x = wire_reply_rec(gid, bnum, bcoord, cp, GPX_WHO(acc_idx, dst_idx, 0u));
    s.x.slot = slot;
    s.x.req_id = (int64_t)(int32_t)(uint32_t)(uint64_t)qid; /* AcceptReplyPacket(JSONObject) :115 reads QID with getInt */
    const uint32_t o = A.moff[A.cap_mem + i];
    s.out = A.rep + o;
    s.key = A.rep_key + o;
    if (pt == GPX_PT_ACCEPT_REPLY) {
      s.out[0] = s.x;
      s.key[0] = gid;
    } else {
      json_get_ints<JsonRepSink>(J, pos[JK_SLOTS], true, &n_slots, &s);
    }
  } else {
    JsonDecSink s;
    s.d = wire_decision_rec(gid, bnum, bcoord, gc, g.ms->lane_mask);
    const uint32_t o = A.moff[2 * A.cap_mem + i];
    s.out = A.dec + o;
    s.key = A.dec_key + o;
    json_get_ints<JsonDecSink>(J, pos[JK_SLOTS], false, &n_slots, &s);
  }
}

/* members (the device count of them) of a packet with a schema failure are dropped; the packet is malformed */
__global__ void k_json_fix(const __grid_constant__ WireJsonArgs A) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < A.n && A.bad[i] && A.status[i] == GPX_WS_OK) A.status[i] = GPX_WS_MALFORMED;
  if (i >= A.cap_mem) return;
  const uint32_t* moffs = A.poff + A.n;
  const uint32_t total = moffs[A.n - 1] + A.pcnt[2 * A.n - 1];
  if (i >= total) return;
  if (A.bad[A.mem[i].pkt]) A.mcnt[i] = A.mcnt[A.cap_mem + i] = A.mcnt[2 * A.cap_mem + i] = 0;
}
