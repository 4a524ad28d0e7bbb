/*
 * gpx_oracle.cpp -- CPU ORACLE for the gigapaxos phase-2 hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under gigapaxos_b200/ may include, link, load or
 * call this file; only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * --impl reference legs do, and only as the checker / the CPU arm.
 *
 * This is a single-threaded restatement of the reference's Java semantics, class by
 * class, with java.util.TreeMap -> std::map.  Each function cites the reference
 * file:line it follows (paths relative to /root/reference/src/edu/umass/cs/gigapaxos/).
 *
 * PARITY PINNING: the reference holds no golden vectors for this path (SURVEY.md 8c);
 * the reference JVM cannot run in the build container (no java/javac).  The oracle is
 * pinned by transliterations of the reference's own self-checking main() tests
 * (gpxo_selftest below): PaxosAcceptor.java:749-776, PaxosCoordinatorState.java:1179-1214,
 * paxosutil/WaitforUtility.java:147-163, PaxosPacketBatcher.java:556-567 (Ballot),
 * paxosutil/HotRestoreInfo.java:159-175 (the one literal-valued test), RFC 1321 vectors
 * for MD5 (digest bytes are "parity unpinned" by the reference, SURVEY.md a19).
 *
 * Beyond phase 2 it restates, for the batch entry points added next to the hot path: phase 1a at the acceptors
 * (gpxo_handle_prepares: PISM.handlePrepare, PaxosAcceptor.handlePrepare :239-297), phase 1b at the would-be
 * coordinator (gpxo_handle_prepare_replies: PaxosCoordinatorState.java:264-587 -- from the CODE; where the class's
 * own main() asserts something else, see DESIGN.md 6), the deactivation sweep (gpxo_pause_groups: PISM.tryPause
 * :2004-2035) and the journal look-ups (gpxo_log_find: SQLPaxosLogger.getLoggedFromMessageLog :3674-3756).  Of these
 * only HotRestoreInfo's literal pins anything the reference produced: parity unpinned, as above.
 *
 * It exposes the same record-level C ABI as include/gpx.h with the prefix gpxo_ so that
 * tests feed identical batches to the CUDA engine and to this file and compare bytes.
 *
 * Two deliberate, documented modelling choices (DESIGN.md "Canonical execution"):
 *  (1) per-group FIFO arrival order and "all requests of the group present in the call,
 *      cut by MAX_BATCH_SIZE / byte limit" batching -- one admissible execution of
 *      RequestBatcher.dequeueImpl (RequestBatcher.java:168-234);
 *  (2) decisions are delivered value-less to every replica (the BATCHED_COMMIT form,
 *      PISM.handleBatchedCommit :1480-1528), i.e. SHORT_CIRCUIT_LOCAL does not
 *      short-circuit commits; a replica resolves the value from its accepted window.
 * With window == 0 the maps are unbounded exactly like the Java TreeMaps; with
 * window == W the bounded-window rules of the device engine are applied on top.
 */
#include "../include/gpx.h"

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <set>
#include <string>
#include <vector>

namespace {

typedef int32_t i32;
typedef uint32_t u32;
typedef int64_t i64;
typedef uint64_t u64;

/* Java int subtraction (wraps) */
static inline i32 jsub(i32 a, i32 b) { return (i32)((u32)a - (u32)b); }

/* paxosutil/Ballot.java:34-116 */
struct Ballot {
  i32 num, coord;
  /* compareTo :60-66 */
  i32 compareTo(const Ballot& b) const { return num != b.num ? jsub(num, b.num) : jsub(coord, b.coord); }
  bool equals(const Ballot& b) const { return compareTo(b) == 0; } /* :76 */
  i32 hashCode() const { return (i32)((u32)(100 + num) * (u32)(100 + num) + (u32)coord); } /* :86 */
  std::string toString() const { return std::to_string(num) + ":" + std::to_string(coord); }
};

/* PValuePacket essentials (paxospackets/PValuePacket.java) */
struct PValue {
  i32 slot = 0;
  Ballot bal{0, 0};
  i64 req_id = 0;
  bool stop = false;
  bool has_value = false; /* RequestPacket.hasRequestValue :1369 */
  i32 median_cp = -1;
  u32 nreq = 0, plen = 0, frame_ref = 0;
};

enum { ST_RECOVERY = 0, ST_ACTIVE_1 = 1, ST_ACTIVE_2 = 2, ST_STOPPED = 3, ST_FREE = 255 };

/* group flags surfaced to the host slow path */
enum { GF_OVERFLOW = 1, GF_NEEDS_SYNC = 2 };

/* ------------------------------------------------------------------------------
 * PaxosAcceptor.java
 * ---------------------------------------------------------------------------- */
struct Acceptor {
  i32 _slot = 0, ballotNum = -1, ballotCoord = -1, acceptedGCSlot = -1; /* :94-99 */
  uint8_t state = ST_FREE;
  uint8_t flags = 0;
  std::map<i32, PValue> acceptedProposals, committedRequests; /* :108-109 */
  bool journaling = true; /* GET_ACCEPTED_PVALUES_FROM_DISK :75-76 */
  int W = 0;

  bool isStopped() const { return state == ST_STOPPED; }
  Ballot getBallot() const { return Ballot{ballotNum, ballotCoord}; }

  /* bounded-window store rule (device ring indexed by slot mod W) */
  void accStore(const PValue& pv) {
    if (W > 0) {
      bool staleNew = jsub(pv.slot, _slot) < 0;
      for (auto it = acceptedProposals.begin(); it != acceptedProposals.end();) {
        if (it->first != pv.slot && (((u32)it->first) & (u32)(W - 1)) == (((u32)pv.slot) & (u32)(W - 1))) {
          bool occStale = jsub(it->first, _slot) < 0;
          if (staleNew && !occStale) return; /* never evict a live entry for a stale accept */
          it = acceptedProposals.erase(it);
        } else
          ++it;
      }
    }
    acceptedProposals[pv.slot] = pv;
  }

  /* handlePrepare ballot bump :245-251 (phase 1 itself is host slow path) */
  void bumpBallot(Ballot b) {
    if (b.compareTo(getBallot()) > 0) {
      ballotNum = b.num;
      ballotCoord = b.coord;
    }
  }

  /* handlePrepare :239-275 with pruneAcceptedProposals :285-297 and getMaxGCSlotFirstUndecidedSlot :277-282.
   * Returns false iff stopped (Java null).  `accepted` comes back in slot order (wrap-aware, relative to the GC
   * slot); empty when NACKing. */
  bool handlePrepare(Ballot prepareBallot, i32 firstUndecidedSlot, Ballot* replyBallot, std::vector<PValue>* accepted,
                     i32* firstSlot) {
    if (isStopped()) return false;
    if (prepareBallot.compareTo(getBallot()) > 0) { /* :245-251 */
      ballotNum = prepareBallot.num;
      ballotCoord = prepareBallot.coord;
    }
    *replyBallot = getBallot();
    accepted->clear();
    if (!(getBallot().compareTo(prepareBallot) > 0)) /* send pvalues only if not NACKing :262-270 */
      for (auto& kv : acceptedProposals)
        if (jsub(kv.first, firstUndecidedSlot) >= 0) accepted->push_back(kv.second); /* :291-293 */
    std::sort(accepted->begin(), accepted->end(), [this](const PValue& a, const PValue& b) {
      return jsub(a.slot, acceptedGCSlot) < jsub(b.slot, acceptedGCSlot);
    });
    *firstSlot = jsub(acceptedGCSlot, firstUndecidedSlot - 1) < 0 ? firstUndecidedSlot - 1 : acceptedGCSlot; /* :277-282 */
    return true;
  }

  /* acceptAndUpdateBallot :302-322; returns false iff stopped (Java null) */
  bool acceptAndUpdateBallot(const PValue& accept, Ballot* out) {
    if (isStopped()) return false;
    if (accept.bal.compareTo(getBallot()) >= 0) { /* :311 */
      ballotNum = accept.bal.num;
      ballotCoord = accept.bal.coord;
      if (jsub(accept.slot, acceptedGCSlot) > 0) accStore(accept); /* :315-316 */
    }
    garbageCollectAccepted(accept.median_cp); /* :320 */
    *out = getBallot();
    return true;
  }

  /* garbageCollectAccepted :476-494 */
  void garbageCollectAccepted(i32 gcSlot) {
    if (jsub(_slot, gcSlot) <= 0) gcSlot = _slot - 1; /* :481-482 */
    if (jsub(gcSlot, acceptedGCSlot) > 0) {           /* :484 */
      acceptedGCSlot = gcSlot;
      for (auto it = acceptedProposals.begin(); it != acceptedProposals.end();)
        if (jsub(it->first, gcSlot) <= 0)
          it = acceptedProposals.erase(it);
        else
          ++it;
    }
    garbageCollectDecisions(gcSlot);
  }

  /* garbageCollectDecisions :496-506 */
  void garbageCollectDecisions(i32 slot) {
    if (jsub(slot, _slot) >= 0) return;
    for (auto it = committedRequests.begin(); it != committedRequests.end();)
      if (jsub(slot, it->first) > 0)
        it = committedRequests.erase(it);
      else
        ++it;
  }

  /* reconstructDecision :369-385 */
  bool reconstructDecision(i32 slot, PValue* out) const {
    auto c = committedRequests.find(slot);
    if (c == committedRequests.end()) return false;
    if (c->second.has_value) {
      *out = c->second;
      return true;
    }
    auto a = acceptedProposals.find(slot);
    if (a != acceptedProposals.end() && a->second.bal.equals(c->second.bal)) {
      *out = a->second; /* new PValuePacket(accept).makeDecision(committed.medianCP) */
      out->median_cp = c->second.median_cp;
      out->has_value = true;
      return true;
    }
    return false;
  }

  /* executed :462-474 */
  void executed(i32 s, bool stop) {
    if (s == _slot) {
      _slot = (i32)((u32)_slot + 1u);
      if (stop) state = ST_STOPPED;
      if (isStopped()) committedRequests.clear();
    } else {
      fprintf(stderr, "oracle: YIKES asked to execute %d when expecting %d\n", s, _slot);
      abort();
    }
  }

  /* putAndRemoveNextExecutable :325-366; decision is never null on this path */
  bool putAndRemoveNextExecutable(const PValue& decision, PValue* out) {
    if (isStopped()) return false;
    garbageCollectAccepted(decision.median_cp); /* :340 */
    if (jsub(decision.slot, _slot) >= 0) {      /* :343 */
      auto it = committedRequests.find(decision.slot);
      if (it == committedRequests.end() || !it->second.has_value) committedRequests[decision.slot] = decision;
    }
    bool have = false;
    if (committedRequests.count(_slot)) { /* :352 */
      PValue nx;
      if (reconstructDecision(_slot, &nx) && nx.has_value) {
        committedRequests.erase(_slot);
        executed(nx.slot, nx.stop);
        *out = nx;
        have = true;
      }
    }
    if (have && journaling) acceptedProposals.erase(out->slot); /* :360-362 */
    return have;
  }

  /* jumpSlot :564-578 */
  void jumpSlot(i32 slotNumber) {
    for (i32 i = _slot; jsub(i, slotNumber) < 0; i = (i32)((u32)i + 1u)) {
      executed(i, false);
      committedRequests.erase(i);
      if (journaling) acceptedProposals.erase(i);
    }
  }
};

/* ------------------------------------------------------------------------------
 * paxosutil/WaitforUtility.java:34-115
 * ---------------------------------------------------------------------------- */
struct WaitforUtility {
  std::vector<i32> members;
  std::vector<bool> responded;
  int heardCount = 0;
  WaitforUtility() {}
  explicit WaitforUtility(const std::vector<i32>& m) : members(m), responded(m.size(), false) {}
  int getIndex(i32 node) const { /* :108-115 (last match wins) */
    int index = -1;
    for (size_t i = 0; i < members.size(); i++)
      if (members[i] == node) index = (int)i;
    return index;
  }
  bool updateHeardFrom(i32 node) { /* :51-62 */
    bool changed = false;
    int index = getIndex(node);
    if (index >= 0 && index < (int)members.size()) {
      if (!responded[index]) {
        changed = true;
        heardCount++;
      }
      responded[index] = true;
    }
    return changed;
  }
  bool heardFromMajority() const { return heardCount > (int)members.size() / 2; } /* :64-68 */
  bool contains(i32 node) const { return getIndex(node) >= 0; }
  u32 mask() const {
    u32 m = 0;
    for (size_t i = 0; i < responded.size() && i < 32; i++)
      if (responded[i]) m |= 1u << i;
    return m;
  }
};

/* ------------------------------------------------------------------------------
 * PaxosCoordinator.java + PaxosCoordinatorState.java (phase 2 only)
 * ---------------------------------------------------------------------------- */
struct Proposal {
  PValue pvalue;
  WaitforUtility waitfor;
};
enum { PT_NONE = 0, PT_DECISION = 1, PT_PREEMPTED = 2 };

struct Coordinator {
  bool exists = false;
  bool active = false;
  i32 myBallotNum = 0, myBallotCoord = 0;
  i32 nextProposalSlotNumber = 0;
  std::vector<i32> nodeSlotNumbers;
  std::map<i32, Proposal> myProposals;
  int W = 0;

  Ballot getBallot() const { return Ballot{myBallotNum, myBallotCoord}; }

  /* PaxosCoordinatorState ctor :163-178 / PaxosCoordinator.createCoordinator :91-104 */
  void create(i32 bnum, i32 coord, i32 slot, size_t nMembers, bool recoveryOrZero) {
    exists = true;
    myBallotNum = bnum;
    myBallotCoord = coord;
    nextProposalSlotNumber = slot;
    nodeSlotNumbers.assign(nMembers, -1);
    myProposals.clear();
    active = (bnum == 0 || recoveryOrZero);
  }

  /* getMedianMinus :867-875 */
  i32 getMajorityCommittedSlot() const {
    std::vector<i32> copy(nodeSlotNumbers);
    std::sort(copy.begin(), copy.end());
    size_t medianMinus = copy.size() % 2 == 0 ? copy.size() / 2 - 1 : copy.size() / 2;
    return copy[medianMinus];
  }

  /* PCS.propose :233-263 (+ initCommander :841-851).  rc: 0 accept issued, 1 queued
   * pre-active (no accept), -3 refused after stop, -4 window full (device rule) */
  int propose(const std::vector<i32>& members, PValue req, PValue* acceptOut) {
    auto prev = myProposals.find(nextProposalSlotNumber - 1);
    if (prev != myProposals.end() && prev->second.pvalue.stop) return GPX_RS_REFUSED_STOP; /* :235-239 */
    if (W > 0)
      for (auto& kv : myProposals)
        if ((((u32)kv.first) & (u32)(W - 1)) == (((u32)nextProposalSlotNumber) & (u32)(W - 1)))
          return GPX_RS_BACKPRESSURE;
    req.slot = nextProposalSlotNumber;
    nextProposalSlotNumber = (i32)((u32)nextProposalSlotNumber + 1u);
    req.bal = getBallot();
    Proposal p;
    p.pvalue = req;
    p.waitfor = WaitforUtility(members);
    myProposals[req.slot] = p; /* :247 */
    if (active) {
      *acceptOut = req;
      acceptOut->median_cp = getMajorityCommittedSlot(); /* AcceptPacket(coord, pvalue, medianMinus) */
      return 0;
    }
    return 1;
  }

  /* recordSlotNumber :809-825 -- NOTE plain '<', not wrap-aware */
  void recordSlotNumber(const std::vector<i32>& members, i32 acceptor, i32 maxCheckpointedSlot) {
    for (size_t i = 0; i < members.size(); i++)
      if (members[i] == acceptor)
        if (nodeSlotNumbers[i] < maxCheckpointedSlot) nodeSlotNumbers[i] = maxCheckpointedSlot;
  }

  /* handleAcceptReplyMyBallot :597-640 */
  int handleAcceptReplyMyBallot(const std::vector<i32>& members, i32 acceptor, i32 slot, i32 maxCP, PValue* out) {
    recordSlotNumber(members, acceptor, maxCP);
    auto it = myProposals.find(slot);
    if (it == myProposals.end()) return PT_NONE;
    it->second.waitfor.updateHeardFrom(acceptor);
    if (it->second.waitfor.heardFromMajority()) {
      *out = it->second.pvalue;
      out->median_cp = getMajorityCommittedSlot(); /* makeDecision(getMajorityCommittedSlot()) :630 */
      myProposals.erase(it);                       /* :635 */
      return PT_DECISION;
    }
    return PT_NONE;
  }

  /* handleAcceptReplyHigherBallot :661-675 */
  int handleAcceptReplyHigherBallot(i32 slot, PValue* out) {
    auto it = myProposals.find(slot);
    if (it == myProposals.end()) return PT_NONE;
    *out = it->second.pvalue;
    myProposals.erase(it);
    return PT_PREEMPTED;
  }

  bool preemptedFully() const { return myProposals.empty(); } /* :677-683 */

  /* PaxosCoordinator.handleAcceptReply PaxosCoordinator.java:210-250 */
  int handleAcceptReply(const std::vector<i32>& members, i32 acceptor, Ballot rb, i32 slot, i32 maxCP, PValue* out) {
    if (!exists || !active) return PT_NONE; /* :212 */
    i32 c = rb.compareTo(getBallot());
    if (c > 0) return handleAcceptReplyHigherBallot(slot, out);
    if (c == 0) return handleAcceptReplyMyBallot(members, acceptor, slot, maxCP, out);
    return PT_NONE; /* :241 lower ballot ignored */
  }
};

/* Java String.hashCode */
static i32 javaStringHash(const char* s, size_t n) {
  u32 h = 0;
  for (size_t i = 0; i < n; i++) h = 31u * h + (u32)(unsigned char)s[i];
  return (i32)h;
}
/* Math.abs (abs(MIN_VALUE) stays negative) */
static i32 javaAbs(i32 v) { return v < 0 ? (i32)(0u - (u32)v) : v; }
/* Java % on ints truncates toward zero, same as C */

/* PISM.roundRobinCoordinator :2251-2256 */
static i32 roundRobinCoordinator(i32 nameHash, const i32* members, i32 n, i32 ballotnum) {
  i32 idx = javaAbs((i32)((u32)ballotnum + (u32)nameHash)) % n;
  if (idx < 0) idx = -idx; /* abs(MIN_VALUE) % n is <= 0 in Java and would throw on the array access */
  return members[idx];
}
/* PISM.getCPI :2694-2697 */
static i32 getCPI(i32 cpi, double noise, i32 nameHash) {
  return (i32)(cpi * (1 - noise) + (javaAbs(nameHash) % cpi) * 2 * noise);
}
/* PISM.lastCheckpointSlot :2594-2599 */
static i32 lastCheckpointSlot(i32 slot, i32 checkpointInterval) {
  i32 lcp = slot - slot % checkpointInterval;
  if (lcp < 0 && ((lcp = jsub(lcp, checkpointInterval)) > 0)) lcp = lastCheckpointSlot(INT32_MAX, checkpointInterval);
  return lcp;
}

/* ------------------------------------------------------------------------------
 * MD5 (RFC 1321) -- RequestPacket.getDigest paxospackets/RequestPacket.java:1414-1430
 * uses java.security.MessageDigest("MD5"), which is not under /root/reference.
 * ---------------------------------------------------------------------------- */
static void md5(const uint8_t* msg, size_t len, uint8_t out[16]) {
  static const u32 K[64] = {
      0xd76aa478, 0xe8c7b756, 0x242070db, 0xc1bdceee, 0xf57c0faf, 0x4787c62a, 0xa8304613, 0xfd469501,
      0x698098d8, 0x8b44f7af, 0xffff5bb1, 0x895cd7be, 0x6b901122, 0xfd987193, 0xa679438e, 0x49b40821,
      0xf61e2562, 0xc040b340, 0x265e5a51, 0xe9b6c7aa, 0xd62f105d, 0x02441453, 0xd8a1e681, 0xe7d3fbc8,
      0x21e1cde6, 0xc33707d6, 0xf4d50d87, 0x455a14ed, 0xa9e3e905, 0xfcefa3f8, 0x676f02d9, 0x8d2a4c8a,
      0xfffa3942, 0x8771f681, 0x6d9d6122, 0xfde5380c, 0xa4beea44, 0x4bdecfa9, 0xf6bb4b60, 0xbebfbc70,
      0x289b7ec6, 0xeaa127fa, 0xd4ef3085, 0x04881d05, 0xd9d4d039, 0xe6db99e5, 0x1fa27cf8, 0xc4ac5665,
      0xf4292244, 0x432aff97, 0xab9423a7, 0xfc93a039, 0x655b59c3, 0x8f0ccc92, 0xffeff47d, 0x85845dd1,
      0x6fa87e4f, 0xfe2ce6e0, 0xa3014314, 0x4e0811a1, 0xf7537e82, 0xbd3af235, 0x2ad7d2bb, 0xeb86d391};
  static const int S[64] = {7, 12, 17, 22, 7, 12, 17, 22, 7, 12, 17, 22, 7, 12, 17, 22, 5, 9,  14, 20, 5, 9,
                            14, 20, 5, 9,  14, 20, 5, 9,  14, 20, 4, 11, 16, 23, 4, 11, 16, 23, 4, 11, 16, 23,
                            4, 11, 16, 23, 6, 10, 15, 21, 6, 10, 15, 21, 6, 10, 15, 21, 6, 10, 15, 21};
  u32 a0 = 0x67452301, b0 = 0xefcdab89, c0 = 0x98badcfe, d0 = 0x10325476;
  size_t padded = ((len + 8) / 64 + 1) * 64;
  std::vector<uint8_t> m(padded, 0);
  memcpy(m.data(), msg, len);
  m[len] = 0x80;
  u64 bits = (u64)len * 8;
  for (int i = 0; i < 8; i++) m[padded - 8 + i] = (uint8_t)(bits >> (8 * i));
  for (size_t off = 0; off < padded; off += 64) {
    u32 M[16];
    for (int i = 0; i < 16; i++)
      M[i] = (u32)m[off + 4 * i] | ((u32)m[off + 4 * i + 1] << 8) | ((u32)m[off + 4 * i + 2] << 16) |
             ((u32)m[off + 4 * i + 3] << 24);
    u32 A = a0, B = b0, C = c0, D = d0;
    for (int i = 0; i < 64; i++) {
      u32 F;
      int g;
      if (i < 16) {
        F = (B & C) | (~B & D);
        g = i;
      } else if (i < 32) {
        F = (D & B) | (~D & C);
        g = (5 * i + 1) % 16;
      } else if (i < 48) {
        F = B ^ C ^ D;
        g = (3 * i + 5) % 16;
      } else {
        F = C ^ (B | ~D);
        g = (7 * i) % 16;
      }
      F = F + A + K[i] + M[g];
      A = D;
      D = C;
      C = B;
      B = B + ((F << S[i]) | (F >> (32 - S[i])));
    }
    a0 += A;
    b0 += B;
    c0 += C;
    d0 += D;
  }
  u32 r[4] = {a0, b0, c0, d0};
  for (int i = 0; i < 4; i++)
    for (int j = 0; j < 4; j++) out[4 * i + j] = (uint8_t)(r[i] >> (8 * j));
}

/* ------------------------------------------------------------------------------
 * paxosutil/HotRestoreInfo.java:60-120 string form ('|' separated)
 * Util.arrayOfIntToString (utils/Util.java:241-248) -> "[a,b,c]" (no blanks; stringToIntArray :184-193 strips any)
 * ---------------------------------------------------------------------------- */
static std::string arrayOfIntToString(const std::vector<i32>& a) {
  std::string s = "[";
  for (size_t i = 0; i < a.size(); i++) {
    s += std::to_string(a[i]);
    if (i + 1 < a.size()) s += ",";
  }
  return s + "]";
}
static std::vector<i32> stringToIntArray(const std::string& s) {
  std::vector<i32> out;
  std::string cur;
  for (char ch : s) {
    if ((ch >= '0' && ch <= '9') || ch == '-')
      cur += ch;
    else if (!cur.empty()) {
      out.push_back((i32)atol(cur.c_str()));
      cur.clear();
    }
  }
  if (!cur.empty()) out.push_back((i32)atol(cur.c_str()));
  return out;
}
struct HotRestoreInfo {
  std::string paxosID;
  i32 version = 0;
  std::vector<i32> members;
  i32 accSlot = 0;
  Ballot accBallot{0, 0};
  i32 accGCSlot = 0;
  bool hasCoord = false;
  Ballot coordBallot{0, 0};
  i32 nextProposalSlot = 0;
  bool hasNodeSlots = false;
  std::vector<i32> nodeSlots;
  std::string toString() const {
    return paxosID + "|" + std::to_string(version) + "|" + arrayOfIntToString(members) + "|" +
           std::to_string(accSlot) + "|" + accBallot.toString() + "|" + std::to_string(accGCSlot) + "|" +
           (hasCoord ? coordBallot.toString() : std::string("null")) + "|" + std::to_string(nextProposalSlot) + "|" +
           (hasNodeSlots ? arrayOfIntToString(nodeSlots) : std::string("null"));
  }
  static Ballot parseBallot(const std::string& s) {
    size_t c = s.find(':');
    return Ballot{(i32)atol(s.substr(0, c).c_str()), (i32)atol(s.substr(c + 1).c_str())};
  }
  static HotRestoreInfo parse(const std::string& ser) {
    std::vector<std::string> t;
    size_t start = 0;
    while (true) {
      size_t p = ser.find('|', start);
      if (p == std::string::npos) {
        t.push_back(ser.substr(start));
        break;
      }
      t.push_back(ser.substr(start, p - start));
      start = p + 1;
    }
    HotRestoreInfo h;
    h.paxosID = t[0];
    h.version = (i32)atol(t[1].c_str());
    h.members = stringToIntArray(t[2]);
    h.accSlot = (i32)atol(t[3].c_str());
    h.accGCSlot = (i32)atol(t[5].c_str());
    h.accBallot = parseBallot(t[4]);
    h.hasCoord = t[6] != "null";
    if (h.hasCoord) h.coordBallot = parseBallot(t[6]);
    h.nextProposalSlot = (i32)atol(t[7].c_str());
    h.hasNodeSlots = t[8] != "null";
    if (h.hasNodeSlots) h.nodeSlots = stringToIntArray(t[8]);
    return h;
  }
};

/* ------------------------------------------------------------------------------
 * record-level engine (same C ABI as the CUDA engine, prefix gpxo_)
 * ---------------------------------------------------------------------------- */
struct Group {
  bool live = false;
  i32 version = 0;
  i32 name_hash = 0;
  std::vector<i32> members; /* sorted (PISM ctor :205) */
  i32 cpi = 400;
};
struct Lane {
  i32 node = 0;
  std::vector<Acceptor> acc;
  std::vector<Coordinator> coord;
  std::vector<uint8_t> ring;
  u64 seg_seq = 0;
};

static thread_local std::string g_err;

}  // namespace

struct gpxo_engine {
  gpx_config cfg;
  std::vector<Group> groups;
  std::vector<Lane> lanes;
  gpx_counters ctr;
  std::set<std::vector<i32>> msets; /* the distinct sorted member sets seen (the engine's table holds GPX_MAX_MSETS) */
  u32 L() const { return cfg.n_lanes; }
  int W() const { return (int)cfg.window; }

  int laneOfNode(i32 node) const {
    for (u32 l = 0; l < cfg.n_lanes; l++)
      if (lanes[l].node == node) return (int)l;
    return -1;
  }
  int memberIdx(const Group& g, i32 node) const {
    int idx = -1;
    for (size_t i = 0; i < g.members.size(); i++)
      if (g.members[i] == node) idx = (int)i;
    return idx;
  }
  u32 localMask(const Group& g) const {
    u32 m = 0;
    for (u32 l = 0; l < cfg.n_lanes; l++)
      if (memberIdx(g, lanes[l].node) >= 0) m |= 1u << l;
    return m;
  }
  bool usable(u32 gid, u32 lane) const {
    if (gid >= groups.size() || !groups[gid].live) return false;
    uint8_t st = lanes[lane].acc[gid].state;
    return st == ST_ACTIVE_1 || st == ST_ACTIVE_2;
  }

  /* ring: append a segment, return offset of header */
  u64 segBegin(u32 lane, uint16_t type, u32 n_slots, u32 rec_bytes, u64 payload_bytes, u32 n_valid = 0xffffffffu) {
    Lane& ln = lanes[lane];
    u64 off = ln.ring.size();
    u64 total = (64 + (u64)n_slots * rec_bytes + ((payload_bytes + 15) & ~(u64)15) + 31) & ~(u64)31;
    ln.ring.resize(off + total, 0);
    gpx_log_seg_hdr h;
    memset(&h, 0, sizeof h);
    h.magic = GPX_SEG_MAGIC;
    h.type = type;
    h.lane = (uint16_t)lane;
    h.n_slots = n_slots;
    h.n_valid = n_valid == 0xffffffffu ? n_slots : n_valid;
    h.payload_bytes = (payload_bytes + 15) & ~(u64)15;
    h.seq = ln.seg_seq++;
    h.ring_off = off;
    h.rec_bytes = rec_bytes;
    memcpy(&ln.ring[off], &h, sizeof h);
    return off;
  }

  /* PISM.shouldCheckpoint :2037-2041 */
  bool shouldCheckpoint(const Group& g, const PValue& d) const { return (d.slot % g.cpi == 0) || d.stop; }

  gpx_exec_rec makeExec(u32 gid, u32 lane, const Group& g, const PValue& x, bool extra) const {
    gpx_exec_rec r;
    r.gid = gid;
    r.slot = x.slot;
    r.req_id = x.req_id;
    r.payload_off = x.frame_ref;
    u32 f = (x.stop ? GPX_F_STOP : 0) | (shouldCheckpoint(g, x) ? GPX_F_CKPT : 0) | (extra ? GPX_F_EXTRA : 0);
    r.flags = f | (lane << 12) | (x.nreq << 16);
    return r;
  }

  /* PISM.extractExecuteAndCheckpoint :1619-1701 (execution itself is the host app's) */
  void EEC(const Group& g, Acceptor& A, const PValue& loggedDecision, std::vector<PValue>& out) {
    if (A.isStopped()) return;
    PValue nx;
    while (A.putAndRemoveNextExecutable(loggedDecision, &nx)) {
      out.push_back(nx);
      ctr.executed++;
      if (shouldCheckpoint(g, nx)) ctr.checkpoints_due++;
      if (nx.stop) {
        ctr.stops_executed++;
        break;
      }
    }
  }

  /* the logged form of a decision, PISM.handleCommittedRequest :1446-1466 */
  bool decisionLogImage(const Acceptor& A, u32 gid, u32 lane, const PValue& committed, gpx_decision_rec* img) const {
    if (!(committed.has_value || cfg.log_meta_decisions)) return false;
    auto ca = A.acceptedProposals.find(committed.slot);
    bool meta = cfg.log_meta_decisions && ca != A.acceptedProposals.end() &&
                ca->second.bal.compareTo(committed.bal) >= 0;
    img->gid = gid;
    img->slot = committed.slot;
    img->bnum = committed.bal.num;
    img->bcoord = committed.bal.coord;
    img->median_cp = meta ? -1 : committed.median_cp; /* getMetaDecision() resets medianCP :212-218 */
    img->flags = (uint16_t)(GPX_F_DECISION | (meta ? GPX_F_META : 0) | (committed.stop ? GPX_F_STOP : 0));
    img->dst_mask = (uint16_t)(1u << lane);
    img->req_id = committed.req_id;
    return true;
  }
};

namespace {
static void put_event_exec(std::vector<gpx_exec_rec>& v, const gpx_exec_rec& r) { v.push_back(r); }
}

extern "C" {

const char* gpxo_last_error(void) { return g_err.c_str(); }
const char* gpxo_build_info(void) { return "oracle (CPU restatement of the Java reference; test infrastructure)"; }

void gpxo_config_defaults(gpx_config* c) {
  memset(c, 0, sizeof *c);
  c->abi_version = GPX_ABI_VERSION;
  c->device = 0;
  c->max_groups = 1024;
  c->n_lanes = 3;
  c->lane_node[0] = 100; /* TC.TEST_START_NODE_ID testing/TESTPaxosConfig.java:100 */
  c->lane_node[1] = 101;
  c->lane_node[2] = 102;
  c->window = 8;
  c->max_group_size = 3;
  c->log_ring_bytes = 1ull << 26;
  c->max_batch_recs = 1u << 16;
  c->max_batch_payload = 1ull << 24;
  c->batching_enabled = 1;
  c->max_batch_size = 2000;
  c->max_batch_bytes = 4 * 1024 * 1024;
  c->request_size_estimate = 512;
  c->checkpoint_interval = 400;
  c->cpi_noise = 0;
  c->gc_majority_executed = 1;
  c->log_meta_decisions = 1;
  c->journaling_enabled = 1;
}

int gpxo_engine_create(const gpx_config* cfg, gpxo_engine** out) {
  if (!cfg || !out || cfg->abi_version != GPX_ABI_VERSION) return GPX_EINVAL;
  if (cfg->n_lanes == 0 || cfg->n_lanes > GPX_MAX_LANES) return GPX_EINVAL;
  if (cfg->max_group_size == 0 || cfg->max_group_size > GPX_MAX_GROUP_SIZE) return GPX_EINVAL;
  for (u32 a = 0; a < cfg->n_lanes; a++) /* a node holds one instance of a group: one lane per node */
    for (u32 b = a + 1; b < cfg->n_lanes; b++)
      if (cfg->lane_node[a] == cfg->lane_node[b]) return GPX_EINVAL;
  if (cfg->window != 0 && (cfg->window > GPX_MAX_WINDOW || (cfg->window & (cfg->window - 1)))) return GPX_EINVAL;
  gpxo_engine* e = new gpxo_engine();
  e->cfg = *cfg;
  memset(&e->ctr, 0, sizeof e->ctr);
  e->groups.resize(cfg->max_groups);
  e->lanes.resize(cfg->n_lanes);
  for (u32 l = 0; l < cfg->n_lanes; l++) {
    e->lanes[l].node = cfg->lane_node[l];
    e->lanes[l].acc.resize(cfg->max_groups);
    e->lanes[l].coord.resize(cfg->max_groups);
  }
  *out = e;
  return GPX_OK;
}
void gpxo_engine_destroy(gpxo_engine* e) { delete e; }

/* what gpx_create_groups / gpx_load_rows check, for every record of a call before any is applied (a refused call
 * changes nothing): gid and lane in range, 1..max_group_size members, none listed twice (PISM.groupMembers is a set,
 * sorted by the ctor :205), and at most GPX_MAX_MSETS distinct member sets per engine.  -> every record's sorted member
 * list */
struct MemberRec {
  u32 gid, lane;
  i32 n_members;
  const i32* members;
};
static int checkMembers(gpxo_engine* e, const std::vector<MemberRec>& recs, std::vector<std::vector<i32>>* sorted) {
  std::set<std::vector<i32>> fresh;
  sorted->resize(recs.size());
  for (size_t k = 0; k < recs.size(); k++) {
    const MemberRec& r = recs[k];
    if (r.gid >= e->cfg.max_groups || r.lane >= e->L() || r.n_members <= 0 || r.n_members > (i32)e->cfg.max_group_size)
      return GPX_ERANGE;
    std::vector<i32>& m = (*sorted)[k];
    m.assign(r.members, r.members + r.n_members);
    std::sort(m.begin(), m.end());
    if (std::adjacent_find(m.begin(), m.end()) != m.end()) return GPX_ERANGE;
    if (!e->msets.count(m)) fresh.insert(m);
  }
  if (e->msets.size() + fresh.size() > GPX_MAX_MSETS) return GPX_ERANGE;
  e->msets.insert(fresh.begin(), fresh.end());
  return GPX_OK;
}

/* PaxosManager.createPaxosInstance(Map,Set) :664-691 -> HotRestoreInfo.createHRI :145-157 (GPX_INIT_BATCH)
 * or PISM.initiateRecovery :591-675 + putInitialState :692-699 (GPX_INIT_DEFAULT) */
int gpxo_create_groups(gpxo_engine* e, uint32_t n, const gpx_group_desc* d) {
  std::vector<MemberRec> recs(n);
  for (u32 k = 0; k < n; k++) recs[k] = MemberRec{d[k].gid, 0, d[k].n_members, d[k].members};
  std::vector<std::vector<i32>> sorted;
  int rc = checkMembers(e, recs, &sorted);
  if (rc) return rc;
  for (u32 k = 0; k < n; k++) {
    Group& g = e->groups[d[k].gid];
    g.live = true;
    g.version = d[k].version;
    g.name_hash = d[k].name_hash;
    g.members = sorted[k];
    g.cpi = getCPI(e->cfg.checkpoint_interval, e->cfg.cpi_noise, g.name_hash);
    i32 coord0 = roundRobinCoordinator(g.name_hash, g.members.data(), (i32)g.members.size(), 0);
    for (u32 l = 0; l < e->L(); l++) {
      Acceptor& A = e->lanes[l].acc[d[k].gid];
      Coordinator& C = e->lanes[l].coord[d[k].gid];
      A = Acceptor();
      C = Coordinator();
      A.W = e->W();
      C.W = e->W();
      A.journaling = e->cfg.journaling_enabled != 0;
      if (e->memberIdx(g, e->lanes[l].node) < 0) continue; /* lane not a member: no instance */
      if (d[k].init_mode == GPX_INIT_BATCH) {
        /* createHRI: accSlot=1, accBallot=(0,coord), accGCSlot=-1, coordBallot=(0,coord),
         * nextProposalSlot=1, nodeSlots=new int[R] (zeros); PISM.hotRestore :677-689 */
        A._slot = 1;
        A.ballotNum = 0;
        A.ballotCoord = coord0;
        A.acceptedGCSlot = -1;
        A.state = ST_ACTIVE_1;
        if (coord0 == e->lanes[l].node) {
          C.create(0, coord0, 1, g.members.size(), true);
          C.nodeSlotNumbers.assign(g.members.size(), 0); /* setNodeSlots(hri.nodeSlots) */
        }
      } else {
        /* initiateRecovery: acceptor (0, rrCoord(0)), slot 0; putInitialState ->
         * handleCheckpoint -> jumpSlot(1); setGCSlotAfterPuttingInitialSlot -> gc 0;
         * coordinator at rr node with nextProposalSlot=1, nodeSlots=-1 */
        A._slot = 0;
        A.ballotNum = 0;
        A.ballotCoord = coord0;
        A.acceptedGCSlot = -1;
        A.state = ST_ACTIVE_1;
        A.jumpSlot(1);
        A.acceptedGCSlot = 0;
        if (coord0 == e->lanes[l].node) C.create(0, coord0, 1, g.members.size(), true);
      }
    }
  }
  return GPX_OK;
}

int gpxo_destroy_groups(gpxo_engine* e, uint32_t n, const uint32_t* gids) {
  for (u32 k = 0; k < n; k++) {
    if (gids[k] >= e->cfg.max_groups) return GPX_ERANGE;
    e->groups[gids[k]].live = false;
    for (u32 l = 0; l < e->L(); l++) {
      e->lanes[l].acc[gids[k]] = Acceptor();
      e->lanes[l].coord[gids[k]] = Coordinator();
    }
  }
  return GPX_OK;
}

int gpxo_dump_rows(gpxo_engine* e, uint32_t n, const uint32_t* gids, uint32_t lane, gpx_row* out) {
  if (lane >= e->L()) return GPX_ERANGE;
  for (u32 k = 0; k < n; k++) {
    u32 gid = gids[k];
    if (gid >= e->cfg.max_groups) return GPX_ERANGE;
    const Group& g = e->groups[gid];
    const Acceptor& A = e->lanes[lane].acc[gid];
    const Coordinator& C = e->lanes[lane].coord[gid];
    gpx_row& r = out[k];
    memset(&r, 0, sizeof r);
    r.gid = gid;
    r.lane = lane;
    r.version = g.version;
    r.name_hash = g.name_hash;
    r.acc_slot = A._slot;
    r.acc_bnum = A.ballotNum;
    r.acc_bcoord = A.ballotCoord;
    r.acc_gc_slot = A.acceptedGCSlot;
    r.state = g.live ? A.state : GPX_ST_FREE;
    r.coord_exists = C.exists;
    r.coord_active = C.exists && C.active;
    r.coord_bnum = C.exists ? C.myBallotNum : 0;
    r.coord_bcoord = C.exists ? C.myBallotCoord : 0;
    r.next_proposal_slot = C.exists ? C.nextProposalSlotNumber : 0;
    r.n_members = (i32)g.members.size();
    for (size_t i = 0; i < g.members.size(); i++) {
      r.members[i] = g.members[i];
      r.node_slots[i] = C.exists ? C.nodeSlotNumbers[i] : 0;
    }
  }
  return GPX_OK;
}

int gpxo_load_rows(gpxo_engine* e, uint32_t n, const gpx_row* rows) {
  std::vector<MemberRec> recs(n);
  for (u32 k = 0; k < n; k++) recs[k] = MemberRec{rows[k].gid, rows[k].lane, rows[k].n_members, rows[k].members};
  std::vector<std::vector<i32>> sorted;
  int rc = checkMembers(e, recs, &sorted);
  if (rc) return rc;
  for (u32 k = 0; k < n; k++) {
    const gpx_row& r = rows[k];
    Group& g = e->groups[r.gid];
    g.live = true;
    g.version = r.version;
    g.name_hash = r.name_hash; /* HotRestoreInfo carries the paxosID: getCPI :2694-2697 follows the name, not the gid */
    g.cpi = getCPI(e->cfg.checkpoint_interval, e->cfg.cpi_noise, g.name_hash);
    g.members = sorted[k];
    Acceptor& A = e->lanes[r.lane].acc[r.gid];
    Coordinator& C = e->lanes[r.lane].coord[r.gid];
    A = Acceptor();
    C = Coordinator();
    A.W = e->W();
    C.W = e->W();
    A.journaling = e->cfg.journaling_enabled != 0;
    A._slot = r.acc_slot;
    A.ballotNum = r.acc_bnum;
    A.ballotCoord = r.acc_bcoord;
    A.acceptedGCSlot = r.acc_gc_slot;
    A.state = (uint8_t)r.state;
    if (r.coord_exists) {
      C.create(r.coord_bnum, r.coord_bcoord, r.next_proposal_slot, g.members.size(), true);
      C.active = r.coord_active != 0;
      C.nodeSlotNumbers.assign(r.node_slots, r.node_slots + r.n_members);
    }
  }
  return GPX_OK;
}

int gpxo_patch(gpxo_engine* e, uint32_t n, const gpx_patch_rec* p) {
  for (u32 k = 0; k < n; k++) {
    if (p[k].gid >= e->cfg.max_groups || p[k].lane >= e->L()) return GPX_ERANGE;
    Group& g = e->groups[p[k].gid];
    Acceptor& A = e->lanes[p[k].lane].acc[p[k].gid];
    Coordinator& C = e->lanes[p[k].lane].coord[p[k].gid];
    switch (p[k].op) {
      case GPX_PATCH_SET_BALLOT: A.bumpBallot(Ballot{p[k].a, p[k].b}); break;
      case GPX_PATCH_JUMP_SLOT:
        if (jsub(p[k].a, A._slot) > 0) A.jumpSlot(p[k].a);
        break;
      case GPX_PATCH_SET_STATE:
        A.state = (uint8_t)p[k].a;
        if (A.isStopped()) A.committedRequests.clear();
        break;
      case GPX_PATCH_INSTALL_COORD:
        C.create(p[k].a, p[k].b, p[k].c, g.members.size(), p[k].d != 0);
        C.active = p[k].d != 0;
        break;
      case GPX_PATCH_RESIGN_COORD: C = Coordinator(); C.W = e->W(); break;
      case GPX_PATCH_SET_GC: A.acceptedGCSlot = p[k].a; break;
      case GPX_PATCH_SET_NODE_SLOT:
        if (C.exists && p[k].a >= 0 && (size_t)p[k].a < C.nodeSlotNumbers.size() &&
            jsub(C.nodeSlotNumbers[p[k].a], p[k].b) < 0)
          C.nodeSlotNumbers[p[k].a] = p[k].b;
        break;
      default: return GPX_EINVAL;
    }
  }
  return GPX_OK;
}

/* RequestBatcher.dequeueImpl RequestBatcher.java:168-234 (canonical rule) +
 * PISM.handleRequest :767 / handleProposal :818-888 + PCS.propose :233-263 */
/* acc_req (or null): [ACCEPT k] = the request index that started its slot.  A status is a slot or a GPX_RS_* code
 * and slots wrap, so a slot may be 0 or negative: the caller cannot pair ACCEPTs with requests by its sign. */
static int proposeImpl(gpxo_engine* e, uint32_t n, const gpx_request_rec* reqs, const uint8_t* payload,
                       uint64_t payload_bytes, gpx_accept_rec* out_accepts, uint32_t* n_accepts, uint8_t* out_blob,
                       uint64_t blob_cap, uint64_t* blob_bytes, int32_t* status, u32* acc_req) {
  /* blob layout (same as the device engine): [payload arena, 16-B padded][constructed blobs of
   * batched slots]; an unbatched slot's blob is the request's own payload (zero copy) */
  const u64 pal = (payload_bytes + 15) & ~(u64)15;
  if (pal > blob_cap) return GPX_ERANGE;
  if (payload_bytes) memcpy(out_blob, payload, payload_bytes);
  if (pal > payload_bytes) memset(out_blob + payload_bytes, 0, pal - payload_bytes);
  u32 na = 0;
  u64 bb = pal;
  u32 i = 0;
  while (i < n) {
    u32 gid = reqs[i].gid;
    u32 j = i;
    while (j < n && reqs[j].gid == gid) j++;
    /* run [i, j) */
    u32 entry = (reqs[i].flags >> 8) & 0xf;
    auto setAll = [&](u32 a, u32 b, i32 code) {
      for (u32 k = a; k < b; k++) status[k] = code;
      e->ctr.requests_rejected += (b - a);
    };
    if (entry >= e->L() || !e->usable(gid, entry)) {
      setAll(i, j, GPX_RS_DROPPED);
      i = j;
      continue;
    }
    Group& g = e->groups[gid];
    /* handleProposal at the entry lane: PaxosCoordinator.exists(c, paxosState.getBallot()) :824 */
    int clane = -1;
    {
      Acceptor& Ae = e->lanes[entry].acc[gid];
      Coordinator& Ce = e->lanes[entry].coord[gid];
      if (Ce.exists && Ce.getBallot().compareTo(Ae.getBallot()) >= 0)
        clane = (int)entry;
      else {
        int fl = e->laneOfNode(Ae.ballotCoord); /* forward to paxosState.getBallotCoord() :862 */
        if (fl < 0) {
          setAll(i, j, GPX_RS_FORWARD);
          i = j;
          continue;
        }
        if (fl == (int)entry) { /* coordinator == myID: force run for coordinator (host) :874-885 */
          setAll(i, j, GPX_RS_NOCOORD);
          i = j;
          continue;
        }
        if (!e->usable(gid, (u32)fl)) {
          setAll(i, j, GPX_RS_DROPPED);
          i = j;
          continue;
        }
        Acceptor& Af = e->lanes[fl].acc[gid];
        Coordinator& Cf = e->lanes[fl].coord[gid];
        if (Cf.exists && Cf.getBallot().compareTo(Af.getBallot()) >= 0)
          clane = fl;
        else {
          setAll(i, j, GPX_RS_NOCOORD);
          i = j;
          continue;
        }
      }
    }
    Coordinator& C = e->lanes[clane].coord[gid];
    u32 k = i;
    while (k < j) {
      /* one batch: first + following within limits (RequestBatcher :198-219) */
      i64 totalByteLength = (i64)reqs[k].payload_len + e->cfg.request_size_estimate;
      i32 totalBatchSize = 1;
      u32 b = k + 1;
      if (e->cfg.batching_enabled)
        while (b < j) {
          totalByteLength += (i64)reqs[b].payload_len + e->cfg.request_size_estimate;
          if (totalByteLength > e->cfg.max_batch_bytes) break;
          totalBatchSize += 1;
          if (totalBatchSize > e->cfg.max_batch_size) break;
          b++;
        }
      u32 nreq = b - k;
      PValue req;
      req.req_id = reqs[k].req_id;
      req.stop = false;
      for (u32 q = k; q < b; q++) req.stop = req.stop || (reqs[q].flags & GPX_F_STOP); /* isStopRequest :1069 */
      req.has_value = true;
      req.nreq = nreq;
      PValue acc;
      int rc = C.propose(g.members, req, &acc);
      if (rc == GPX_RS_REFUSED_STOP || rc == GPX_RS_BACKPRESSURE) {
        setAll(k, j, rc); /* the rest of the run meets the same refusal */
        break;
      }
      if (rc == 1) { /* pre-active: queued at the coordinator without an ACCEPT */
        for (u32 q = k; q < b; q++) status[q] = GPX_RS_PREACTIVE;
        k = b;
        continue;
      }
      /* blob */
      u64 boff = bb;
      u32 plen;
      if (nreq == 1) {
        plen = reqs[k].payload_len;
        boff = reqs[k].payload_off;
      } else {
        u64 total = (u64)nreq * 16;
        for (u32 q = k; q < b; q++) total += reqs[q].payload_len;
        plen = (u32)total;
        if (bb + ((total + 15) & ~(u64)15) > blob_cap) return GPX_ERANGE;
        u64 w = bb;
        for (u32 q = k; q < b; q++) {
          gpx_batch_ent be;
          be.req_id = reqs[q].req_id;
          be.len = reqs[q].payload_len;
          be.flags = reqs[q].flags;
          memcpy(out_blob + w, &be, 16);
          w += 16;
        }
        for (u32 q = k; q < b; q++) {
          memcpy(out_blob + w, payload + reqs[q].payload_off, reqs[q].payload_len);
          w += reqs[q].payload_len;
        }
        if (w & 15) memset(out_blob + w, 0, 16 - (w & 15));
        bb += ((u64)plen + 15) & ~(u64)15;
      }
      gpx_accept_rec& a = out_accepts[na++];
      a.h.gid = gid;
      a.h.slot = acc.slot;
      a.h.bnum = acc.bal.num;
      a.h.bcoord = acc.bal.coord;
      a.h.median_cp = acc.median_cp;
      a.h.flags = (uint16_t)(GPX_F_ACCEPT | (req.stop ? GPX_F_STOP : 0));
      a.h.dst_mask = (uint16_t)e->localMask(g);
      a.h.req_id = req.req_id;
      a.payload_off = (u32)boff;
      a.payload_len = plen;
      a.nreq = nreq;
      a.sender = C.myBallotCoord;
      if (acc_req) acc_req[na - 1] = k;
      status[k] = acc.slot;
      for (u32 q = k + 1; q < b; q++) status[q] = GPX_RS_BATCHED;
      e->ctr.proposals++;
      e->ctr.requests_batched += nreq;
      k = b;
    }
    i = j;
  }
  *n_accepts = na;
  *blob_bytes = bb;
  return GPX_OK;
}

int gpxo_propose(gpxo_engine* e, uint32_t n, const gpx_request_rec* reqs, const uint8_t* payload,
                 uint64_t payload_bytes, gpx_accept_rec* out_accepts, uint32_t* n_accepts, uint8_t* out_blob,
                 uint64_t blob_cap, uint64_t* blob_bytes, int32_t* status) {
  return proposeImpl(e, n, reqs, payload, payload_bytes, out_accepts, n_accepts, out_blob, blob_cap, blob_bytes, status,
                     nullptr);
}

/* ---- per-record bodies (shared by the phase-by-phase and the fused entry points) ---------- */

/* PISM.handleAccept :1080-1166 for ACCEPT i at lane l */
static void acceptAtLane(gpxo_engine* e, u32 i, u32 l, const gpx_accept_rec& r, const uint8_t* blob, u64 seg, u64 pay,
                         gpx_accept_reply_rec& rep, std::vector<gpx_exec_rec>& extras) {
  memset(&rep, 0, sizeof rep);
  rep.gid = r.h.gid;
  rep.slot = r.h.slot;
  rep.who = GPX_WHO(0xff, 0xff, GPX_F_VOID);
  gpx_accept_rec img = r;
  img.h.flags = GPX_F_VOID;
  /* ACCEPT segment: [hdr][n x 32 B pvalue-header plane][n x 16 B extension plane][payload] */
  const u32 nslots = ((const gpx_log_seg_hdr*)&e->lanes[l].ring[seg])->n_slots;
  auto writeImg = [&]() {
    memcpy(&e->lanes[l].ring[seg + 64 + (u64)i * 32], &img, 32);
    memcpy(&e->lanes[l].ring[seg + 64 + (u64)nslots * 32 + (u64)i * 16], (const uint8_t*)&img + 32, 16);
  };
  if (!(r.h.dst_mask & (1u << l)) || (r.h.flags & GPX_F_VOID)) {
    writeImg();
    return;
  }
  if (!e->usable(r.h.gid, l)) { /* PISM :456-460 stopped / no instance -> dropped */
    e->ctr.accepts_dropped++;
    writeImg();
    return;
  }
  Group& g = e->groups[r.h.gid];
  Acceptor& A = e->lanes[l].acc[r.h.gid];
  int myIdx = e->memberIdx(g, e->lanes[l].node);
  if (myIdx < 0) {
    e->ctr.accepts_dropped++;
    writeImg();
    return;
  }
  if (e->W() > 0 && jsub(r.h.slot, A._slot) >= e->W()) { /* device window rule */
    A.flags |= GF_OVERFLOW;
    e->ctr.window_overflow++;
    e->ctr.accepts_dropped++;
    writeImg();
    return;
  }
  e->ctr.accepts_handled++;
  PValue accept;
  accept.slot = r.h.slot;
  accept.bal = Ballot{r.h.bnum, r.h.bcoord};
  accept.req_id = r.h.req_id;
  accept.stop = (r.h.flags & GPX_F_STOP) != 0;
  accept.has_value = true;
  accept.median_cp = r.h.median_cp;
  accept.nreq = r.nreq;
  accept.plen = r.payload_len;
  accept.frame_ref = (u32)((pay + r.payload_off) / 16);
  /* prev = paxosState.getAccept(accept.slot) :1123 */
  bool hasPrev = A.acceptedProposals.count(accept.slot) != 0;
  PValue prev;
  if (hasPrev) prev = A.acceptedProposals[accept.slot];
  /* a duplicate of an already accepted pvalue keeps the frame it was logged in */
  if (hasPrev && prev.bal.equals(accept.bal)) accept.frame_ref = prev.frame_ref;
  Ballot ballot;
  if (!A.acceptAndUpdateBallot(accept, &ballot)) {
    writeImg();
    return;
  }
  /* AcceptReplyPacket :1139-1143 */
  rep.bnum = ballot.num;
  rep.bcoord = ballot.coord;
  rep.max_cp = e->cfg.gc_majority_executed ? A._slot - 1 : lastCheckpointSlot(A._slot - 1, g.cpi);
  rep.req_id = r.h.req_id;
  int dstIdx = e->memberIdx(g, r.sender);
  /* toLog :1146-1149 */
  bool toLog = accept.bal.compareTo(ballot) >= 0 && jsub(accept.slot, A.acceptedGCSlot) > 0 &&
               (!hasPrev || prev.bal.compareTo(accept.bal) < 0);
  bool nack = ballot.compareTo(accept.bal) > 0;
  u32 rf = (toLog ? GPX_F_LOGGED : 0) | (nack ? GPX_F_NACK : 0);
  rep.who = GPX_WHO(myIdx, dstIdx < 0 ? 0xff : dstIdx, rf);
  if (nack)
    e->ctr.accepts_nacked++;
  else
    e->ctr.accepts_acked++;
  if (toLog) {
    e->ctr.accepts_logged++;
    img = r;
    img.h.dst_mask = (uint16_t)(1u << l);
    memcpy(&e->lanes[l].ring[pay + r.payload_off], blob + r.payload_off, r.payload_len);
  }
  writeImg();
  /* reconstructDecision(accept.slot) -> handleCommittedRequest :1158-1161 */
  PValue rd;
  if (A.reconstructDecision(accept.slot, &rd)) {
    /* the re-log of the reconstructed decision (logDecision :1446) is deliberately omitted:
     * its placeholder was logged on arrival and replay of {placeholder, accept} is
     * idempotent (DESIGN.md "Deliberate omissions") */
    std::vector<PValue> ex;
    e->EEC(g, A, rd, ex);
    for (auto& x : ex) put_event_exec(extras, e->makeExec(r.h.gid, l, g, x, true));
  }
}

/* the local lane that must tally this reply, or -1 (void / unknown group / remote or unusable coordinator) */
static int replyLane(gpxo_engine* e, const gpx_accept_reply_rec& r, bool count) {
  u32 wf = GPX_WHO_FLAGS(r.who);
  if (wf & GPX_F_VOID) return -1;
  int lane = -1;
  if (r.gid < e->cfg.max_groups && e->groups[r.gid].live) {
    Group& g = e->groups[r.gid];
    u32 dstIdx = GPX_WHO_DST(r.who);
    if (dstIdx < g.members.size()) {
      lane = e->laneOfNode(g.members[dstIdx]);
      if (lane >= 0 && !e->usable(r.gid, (u32)lane)) lane = -1;
    }
  }
  if (lane < 0 && count) e->ctr.replies_ignored++;
  return lane;
}

/* PISM.handleAcceptReply :1248-1365 for one reply at coordinator lane `lane`; true iff a DECISION results */
static bool replyAtLane(gpxo_engine* e, int lane, const gpx_accept_reply_rec& r, gpx_decision_rec* d) {
  Group& g = e->groups[r.gid];
  u32 accIdx = GPX_WHO_ACC(r.who);
  e->ctr.replies_handled++;
  Coordinator& C = e->lanes[lane].coord[r.gid];
  i32 acceptorNode = accIdx < g.members.size() ? g.members[accIdx] : INT32_MIN;
  Ballot rb{r.bnum, r.bcoord};
  PValue pv;
  int t = C.handleAcceptReply(g.members, acceptorNode, rb, r.slot, r.max_cp, &pv);
  /* nullifyCoordinatorIfPreemptedFully :1353-1356 / PaxosCoordinator.isPreemptedFully :109-114 */
  if (C.exists && rb.compareTo(C.getBallot()) > 0 && C.preemptedFully()) {
    C = Coordinator();
    C.W = e->W();
    e->ctr.coordinators_resigned++;
  }
  if (t == PT_DECISION) {
    d->gid = r.gid;
    d->slot = pv.slot;
    d->bnum = pv.bal.num;
    d->bcoord = pv.bal.coord;
    d->median_cp = pv.median_cp;
    d->flags = (uint16_t)(GPX_F_DECISION | (pv.stop ? GPX_F_STOP : 0));
    d->dst_mask = (uint16_t)e->localMask(g);
    d->req_id = pv.req_id;
    e->ctr.decisions_made++;
    return true;
  }
  if (t == PT_PREEMPTED) e->ctr.preempted++; /* dropped: FORWARD_PREEMPTED_REQUESTS=false PaxosConfig.java:927 */
  return false;
}

/* PISM.handleBatchedCommit :1480-1528 (one slot) -> handleCommittedRequest :1432-1478 ->
 * extractExecuteAndCheckpoint :1619-1701, for DECISION i at lane l */
static void decisionAtLane(gpxo_engine* e, u32 i, u32 l, const gpx_decision_rec& r, u64 seg, gpx_exec_rec& ex,
                           std::vector<gpx_exec_rec>& extras) {
  memset(&ex, 0, sizeof ex);
  ex.gid = r.gid;
  ex.slot = r.slot;
  ex.flags = GPX_F_VOID | (l << 12);
  gpx_decision_rec img = r;
  img.flags = GPX_F_VOID;
  auto writeImg = [&]() { memcpy(&e->lanes[l].ring[seg + 64 + (u64)i * 32], &img, 32); };
  if (!(r.dst_mask & (1u << l)) || (r.flags & GPX_F_VOID)) {
    writeImg();
    return;
  }
  if (!e->usable(r.gid, l)) {
    e->ctr.decisions_dropped++;
    writeImg();
    return;
  }
  Group& g = e->groups[r.gid];
  Acceptor& A = e->lanes[l].acc[r.gid];
  if (e->W() > 0 && jsub(r.slot, A._slot) >= e->W()) {
    A.flags |= GF_OVERFLOW | GF_NEEDS_SYNC;
    e->ctr.window_overflow++;
    e->ctr.decisions_dropped++;
    writeImg();
    return;
  }
  e->ctr.decisions_handled++;
  Ballot cb{r.bnum, r.bcoord};
  PValue d;
  auto a = A.acceptedProposals.find(r.slot);
  if (a != A.acceptedProposals.end() && a->second.bal.equals(cb)) { /* :1488 */
    d = a->second;
    d.median_cp = r.median_cp;
    d.has_value = true;
  } else { /* placeholder :1514-1522 */
    d = PValue();
    d.slot = r.slot;
    d.bal = cb;
    d.median_cp = r.median_cp;
    d.has_value = false;
    e->ctr.placeholders++;
  }
  (void)e->decisionLogImage(A, r.gid, l, d, &img); /* logDecision :1446-1466 (img stays VOID when not logged) */
  writeImg();
  std::vector<PValue> xs;
  e->EEC(g, A, d, xs);
  for (size_t k = 0; k < xs.size(); k++) {
    if (k == 0)
      ex = e->makeExec(r.gid, l, g, xs[k], false);
    else
      extras.push_back(e->makeExec(r.gid, l, g, xs[k], true));
  }
  if (!A.isStopped() && !d.has_value && jsub(d.slot, A._slot) >= 0 && xs.empty()) A.flags |= GF_NEEDS_SYNC;
}

static void emitExtras(const std::vector<gpx_exec_rec>& extras, gpx_exec_rec* out, uint32_t cap, uint32_t* n_extra) {
  u32 ne = 0;
  for (auto& x : extras)
    if (ne < cap && out) out[ne++] = x;
  if (n_extra) *n_extra = (u32)extras.size();
}

/* PISM.handleAccept :1080-1166 at every addressed local lane */
/* n ACCEPTs into a segment with n_slots >= n image slots (the phase pipeline of a round reserves one slot per
 * REQUEST before it knows how many ACCEPTs the batcher emits, like the device) */
static int acceptsImpl(gpxo_engine* e, u32 n, u32 n_slots, const gpx_accept_rec* accepts, const uint8_t* blob,
                       u64 blob_bytes, gpx_accept_reply_rec* out_replies, gpx_exec_rec* out_extra_exec, u32 extra_cap,
                       u32* n_extra) {
  u32 L = e->L();
  std::vector<u64> seg(L), pay(L);
  for (u32 l = 0; l < L; l++) {
    seg[l] = e->segBegin(l, GPX_F_ACCEPT, n_slots, 48, blob_bytes, n);
    pay[l] = seg[l] + 64 + (u64)n_slots * 48;
  }
  std::vector<gpx_exec_rec> extras;
  for (u32 i = 0; i < n; i++)
    for (u32 l = 0; l < L; l++)
      acceptAtLane(e, i, l, accepts[i], blob, seg[l], pay[l], out_replies[(u64)i * L + l], extras);
  emitExtras(extras, out_extra_exec, extra_cap, n_extra);
  return GPX_OK;
}
static int decisionsImpl(gpxo_engine* e, u32 n, u32 n_slots, const gpx_decision_rec* decisions, gpx_exec_rec* out_exec,
                         gpx_exec_rec* out_extra_exec, u32 extra_cap, u32* n_extra);

int gpxo_handle_accepts(gpxo_engine* e, uint32_t n, const gpx_accept_rec* accepts, const uint8_t* blob,
                        uint64_t blob_bytes, gpx_accept_reply_rec* out_replies, gpx_exec_rec* out_extra_exec,
                        uint32_t extra_cap, uint32_t* n_extra) {
  if (n == 0) { /* an empty batch is a no-op: nothing is logged (the engine's calls return at once, too) */
    if (n_extra) *n_extra = 0;
    return GPX_OK;
  }
  return acceptsImpl(e, n, n, accepts, blob, blob_bytes, out_replies, out_extra_exec, extra_cap, n_extra);
}

/* PISM.handlePrepare :896-955 at every addressed local lane (phase 1a; the coordinator side stays on the host) */
int gpxo_handle_prepares(gpxo_engine* e, uint32_t n, const gpx_pvalue_hdr* prepares, gpx_prepare_reply_rec* out_replies) {
  if (n == 0) return GPX_OK;
  u32 L = e->L();
  std::vector<u64> seg(L);
  for (u32 l = 0; l < L; l++) seg[l] = e->segBegin(l, GPX_F_PREPARE, n, 32, 0);
  for (u32 i = 0; i < n; i++)
    for (u32 l = 0; l < L; l++) {
      const gpx_pvalue_hdr& r = prepares[i];
      gpx_prepare_reply_rec& rep = out_replies[(u64)i * L + l];
      memset(&rep, 0, sizeof rep);
      rep.gid = r.gid;
      rep.who = GPX_WHO(0xff, 0xff, GPX_F_VOID);
      gpx_pvalue_hdr img = r;
      img.flags = GPX_F_VOID;
      auto writeImg = [&]() { memcpy(&e->lanes[l].ring[seg[l] + 64 + (u64)i * 32], &img, 32); };
      if (!(r.dst_mask & (1u << l)) || (r.flags & GPX_F_VOID) || !e->usable(r.gid, l)) { /* PISM :456-460 */
        writeImg();
        continue;
      }
      Group& g = e->groups[r.gid];
      Acceptor& A = e->lanes[l].acc[r.gid];
      const int myIdx = e->memberIdx(g, e->lanes[l].node);
      if (myIdx < 0) {
        writeImg();
        continue;
      }
      const Ballot prev = A.getBallot(), pb{r.bnum, r.bcoord};
      Ballot rb{0, 0};
      std::vector<PValue> acc;
      i32 firstSlot = 0;
      if (!A.handlePrepare(pb, r.slot, &rb, &acc, &firstSlot)) { /* stopped: null */
        writeImg();
        continue;
      }
      const int dstIdx = e->memberIdx(g, r.bcoord);
      u32 fl = 0;
      if (rb.compareTo(pb) > 0) fl |= GPX_F_NACK;
      if (prev.compareTo(rb) < 0) { /* the ballot was raised: log the PREPARE, then reply (LogMessagingTask :940-944) */
        fl |= GPX_F_LOGGED;
        img.flags = (uint16_t)GPX_F_PREPARE;
        img.dst_mask = (uint16_t)(1u << l);
      }
      /* GET_ACCEPTED_PVALUES_FROM_DISK :927-931: a preparer that is behind also needs the executed slots' accepts */
      if (!(fl & GPX_F_NACK) && A.journaling && jsub(r.slot, A._slot) < 0) fl |= GPX_F_FROM_LOG;
      writeImg();
      rep.first_slot = firstSlot;
      rep.bnum = rb.num;
      rep.bcoord = rb.coord;
      rep.who = GPX_WHO((u32)myIdx, dstIdx < 0 ? 0xffu : (u32)dstIdx, fl);
      u32 k = 0;
      for (const PValue& pv : acc) {
        if (k >= GPX_MAX_WINDOW) break;
        gpx_accepted_pvalue& o = rep.accepted[k++];
        o.slot = pv.slot;
        o.bnum = pv.bal.num;
        o.bcoord = pv.bal.coord;
        o.frame_ref = pv.frame_ref;
        o.req_id = pv.req_id;
        o.payload_len = pv.plen;
        o.flags = (pv.stop ? 2u : 0u) | (pv.nreq << 16);
      }
      rep.n_accepted = k;
    }
  return GPX_OK;
}

/* ------------------------------------------------------------------------------
 * Phase 1b at the would-be coordinator: PISM.handlePrepareReply :1017-1068 ->
 * PaxosCoordinator.getPreActivesIfPreempted PaxosCoordinator.java:313-318 / handlePrepareReply :281-299 ->
 * PaxosCoordinatorState.java:264-587.  The pre-active PaxosCoordinatorState lives for the duration of the call.
 * ---------------------------------------------------------------------------- */
namespace {
struct PrepareReplyPacket { /* paxospackets/PrepareReplyPacket.java:36-87 */
  Ballot ballot{0, 0};
  i32 acceptor = 0;   /* node id */
  i32 firstSlot = 0;  /* gcSlot + 1 :80 */
  std::vector<std::pair<gpx_accepted_pvalue, u32>> accepted; /* (pvalue, index of the record that carried it) */
  /* getMinSlot() :151-164: starts at firstSlot, wrap-aware */
  i32 getMinSlot() const {
    i32 minSlot = firstSlot;
    for (auto& a : accepted)
      if (jsub(a.first.slot, minSlot) < 0) minSlot = a.first.slot;
    return minSlot;
  }
};

struct Phase1Proposal { /* ProposalStateAtCoordinator :148-162, as far as phase 1 uses it */
  i32 slot;
  u32 kind; /* GPX_CO_* */
  u32 src;
  gpx_accepted_pvalue pv;
  bool isStopRequest() const { return kind == GPX_CO_STOP_NEW || (kind == GPX_CO_PVALUE && (pv.flags & 2u)); }
  bool isNoop() const { return kind == GPX_CO_NOOP; } /* requestValue.equals(NO_OP) */
};

struct PreActiveCoordinatorState { /* PaxosCoordinatorState.java:67-178 in the pre-active state */
  i32 myBallotNum, myBallotCoord, nextProposalSlotNumber;
  std::vector<i32> nodeSlotNumbers;
  std::vector<i32> members;
  WaitforUtility waitforMyBallot;
  std::map<i32, std::pair<gpx_accepted_pvalue, u32>> carryoverProposals;
  std::vector<Phase1Proposal> myProposals; /* in slot order (the range loop of combinePValuesOntoProposals) */
  bool overflow = false, stopOrder = false;

  PreActiveCoordinatorState(i32 bnum, i32 coord, i32 slot, const std::vector<i32>& m) /* ctor :163-178 + prepare :213-219 */
      : myBallotNum(bnum), myBallotCoord(coord), nextProposalSlotNumber(slot), nodeSlotNumbers(m.size(), -1), members(m),
        waitforMyBallot(m) {}
  Ballot getBallot() const { return Ballot{myBallotNum, myBallotCoord}; }

  bool isPreemptable(const PrepareReplyPacket& r) const { return r.ballot.compareTo(getBallot()) > 0; } /* :271-278 */

  bool canIgnorePrepareReply(const PrepareReplyPacket& r) const { /* :287-316 */
    if (r.ballot.compareTo(getBallot()) < 0) return true;
    if (!waitforMyBallot.contains(r.acceptor)) return true;
    int idx = waitforMyBallot.getIndex(r.acceptor);
    return waitforMyBallot.responded[idx]; /* alreadyHeardFrom */
  }

  void recordSlotNumber(const PrepareReplyPacket& r) { /* :786-807 */
    for (size_t i = 0; i < members.size(); i++)
      if (members[i] == r.acceptor)
        if (jsub(nodeSlotNumbers[i], r.getMinSlot()) < 0) nodeSlotNumbers[i] = r.getMinSlot();
  }

  bool isPrepareAcceptedByMajority(const PrepareReplyPacket& r) { /* :326-391 */
    if (canIgnorePrepareReply(r)) return false;
    recordSlotNumber(r);
    for (auto& a : r.accepted) {
      const i32 curSlot = a.first.slot;
      auto ex = carryoverProposals.find(curSlot);
      if (ex == carryoverProposals.end() ||
          Ballot{a.first.bnum, a.first.bcoord}.compareTo(Ballot{ex->second.first.bnum, ex->second.first.bcoord}) > 0) {
        carryoverProposals[curSlot] = a;
        if (carryoverProposals.size() > GPX_MAX_CARRY) { /* device rule */
          overflow = true;
          return false;
        }
      }
    }
    waitforMyBallot.updateHeardFrom(r.acceptor);
    return waitforMyBallot.heardFromMajority();
  }

  i32 getMaxPValueSlot() const { /* :903-914 */
    bool have = false;
    i32 maxSlot = 0;
    for (auto& kv : carryoverProposals) {
      if (!have) {
        maxSlot = kv.first;
        have = true;
      }
      if (jsub(kv.first, maxSlot) > 0) maxSlot = kv.first;
    }
    return maxSlot;
  }
  i32 getMaxMinCarryoverSlot() const { /* :921-931 */
    i32 maxSlot = nodeSlotNumbers[0];
    for (size_t i = 0; i < nodeSlotNumbers.size(); i++)
      if (jsub(nodeSlotNumbers[i], maxSlot) > 0) maxSlot = nodeSlotNumbers[i];
    return maxSlot;
  }

  /* PCS.propose :233-263 while not active: the proposal is queued at the next slot, no ACCEPT */
  void proposePreActive(u32 kind) {
    if (!myProposals.empty() && myProposals.back().slot == nextProposalSlotNumber - 1 && myProposals.back().isStopRequest())
      return; /* :235-239 */
    Phase1Proposal p;
    memset(&p, 0, sizeof p);
    p.slot = nextProposalSlotNumber;
    p.kind = kind;
    nextProposalSlotNumber = (i32)((u32)nextProposalSlotNumber + 1u);
    myProposals.push_back(p);
  }

  void combinePValuesOntoProposals() { /* :393-444; preActives is empty (header comment of gpx_handle_prepare_replies) */
    if (carryoverProposals.empty()) return;
    const i32 maxCarryoverSlot = getMaxPValueSlot();
    const i32 maxMinCarryoverSlot = getMaxMinCarryoverSlot();
    const i32 span = jsub(maxCarryoverSlot, maxMinCarryoverSlot);
    if (span >= GPX_MAX_PLAN) { /* device rule */
      overflow = true;
      return;
    }
    /* for (curSlot = maxMin; curSlot - maxCarry <= 0; curSlot++) :408 -- counted (span < 0: no iteration), so that two
     * slots 2^31 apart in a hostile record cannot make it run away */
    for (i32 d = 0; d <= span; d++) {
      const i32 curSlot = (i32)((u32)maxMinCarryoverSlot + (u32)d);
      Phase1Proposal p;
      memset(&p, 0, sizeof p);
      p.slot = curSlot;
      auto c = carryoverProposals.find(curSlot);
      if (c != carryoverProposals.end()) {
        p.kind = GPX_CO_PVALUE;
        p.pv = c->second.first;
        p.src = c->second.second;
      } else {
        p.kind = GPX_CO_NOOP; /* makeNoopPValue(curSlot, null, ...) :886-897 */
      }
      myProposals.push_back(p);
    }
    nextProposalSlotNumber = (i32)((u32)maxCarryoverSlot + 1u); /* :436 */
    processStop();
  }

  void processStop() { /* :478-554 */
    bool stopExists = false;
    for (const Phase1Proposal& psac1 : myProposals) {
      if (!psac1.isStopRequest()) continue;
      stopExists = true;
      for (const Phase1Proposal& psac2 : myProposals)
        if (!psac2.isStopRequest() && !psac2.isNoop() && jsub(psac1.slot, psac2.slot) < 0) {
          /* both pvalues carry MY ballot here (ProposalStateAtCoordinator's ctor :153-157 re-stamps it), so neither
           * "stop ballot > other ballot" :495 nor "<" :510 can hold: the reference reaches its assert(false) :524 */
          stopOrder = true;
        }
    }
    if (stopExists && !myProposals.empty()) {
      const Phase1Proposal& last = myProposals.back(); /* myProposals.get(nextProposalSlotNumber - 1) */
      if (!last.isStopRequest()) proposePreActive(GPX_CO_STOP_NEW); /* :538-542 */
    }
  }
};
}  // namespace

int gpxo_handle_prepare_replies(gpxo_engine* e, uint32_t n, const gpx_election_rec* elections, uint32_t n_reply_recs,
                                const gpx_prepare_reply_rec* replies, gpx_election_out* out) {
  if (!e || (n && (!elections || !out)) || (n_reply_recs && !replies)) return GPX_EINVAL;
  {
    std::vector<u32> seen(n);
    for (u32 i = 0; i < n; i++) {
      if ((u64)elections[i].first_reply + elections[i].n_replies > n_reply_recs) return GPX_ERANGE;
      seen[i] = elections[i].gid;
    }
    std::sort(seen.begin(), seen.end());
    if (std::adjacent_find(seen.begin(), seen.end()) != seen.end()) return GPX_EINVAL; /* one election per group per call */
  }
  for (u32 i = 0; i < n; i++) {
    const gpx_election_rec& el = elections[i];
    gpx_election_out& o = out[i];
    memset(&o, 0, sizeof o);
    o.gid = el.gid;
    o.verdict = GPX_EL_DROPPED;
    for (int m = 0; m < GPX_MAX_GROUP_SIZE; m++) o.node_slots[m] = -1;
    if (el.lane >= e->L() || !e->usable(el.gid, el.lane)) continue; /* PISM :456-460 */
    Group& g = e->groups[el.gid];
    if (e->memberIdx(g, e->lanes[el.lane].node) < 0) continue;
    PreActiveCoordinatorState pcs(el.bnum, el.bcoord, el.slot, g.members);
    int verdict = GPX_EL_WAITING;
    for (u32 k = el.first_reply; k < el.first_reply + el.n_replies && verdict == GPX_EL_WAITING;) {
      /* one PREPARE_REPLY = a record and its GPX_F_MORE continuations */
      const gpx_prepare_reply_rec& h = replies[k];
      PrepareReplyPacket pr;
      pr.ballot = Ballot{h.bnum, h.bcoord};
      const u32 idx = GPX_WHO_ACC(h.who);
      const bool isVoid = GPX_WHO_FLAGS(h.who) & GPX_F_VOID;
      pr.acceptor = idx < g.members.size() ? g.members[idx] : -1;
      pr.firstSlot = (i32)((u32)h.first_slot + 1u); /* the record holds gcSlot */
      for (;;) {
        const gpx_prepare_reply_rec& r = replies[k];
        for (u32 a = 0; a < r.n_accepted && a < GPX_MAX_WINDOW; a++) pr.accepted.push_back({r.accepted[a], k});
        const bool more = (GPX_WHO_FLAGS(r.who) & GPX_F_MORE) && !(GPX_WHO_FLAGS(r.who) & GPX_F_VOID);
        k++;
        if (!more || k >= el.first_reply + el.n_replies) break;
      }
      if (isVoid) continue;
      if (pcs.isPreemptable(pr)) { /* getPreActivesIfPreempted: the election is lost, the coordinator resigns */
        verdict = GPX_EL_PREEMPTED;
        break;
      }
      if (idx >= g.members.size()) continue; /* !Util.contains(acceptor, members) */
      if (pcs.isPrepareAcceptedByMajority(pr)) { /* PaxosCoordinator.handlePrepareReply :281-299 */
        pcs.combinePValuesOntoProposals();
        verdict = GPX_EL_MAJORITY;
      }
      if (pcs.overflow) verdict = GPX_EL_OVERFLOW;
    }
    o.verdict = verdict;
    for (size_t m = 0; m < pcs.nodeSlotNumbers.size() && m < GPX_MAX_GROUP_SIZE; m++) o.node_slots[m] = pcs.nodeSlotNumbers[m];
    if (verdict != GPX_EL_MAJORITY) continue;
    o.flags = pcs.stopOrder ? GPX_ELF_STOP_ORDER : 0;
    o.n_plan = (uint16_t)pcs.myProposals.size();
    for (size_t k = 0; k < pcs.myProposals.size(); k++) {
      const Phase1Proposal& p = pcs.myProposals[k];
      o.plan[k].slot = p.slot;
      o.plan[k].kind = p.kind;
      o.plan[k].src_reply = p.kind == GPX_CO_PVALUE ? p.src : 0;
      if (p.kind == GPX_CO_PVALUE) o.plan[k].pv = p.pv;
    }
    /* spawnCommandersForProposals :556-575 is the caller's re-proposal of the plan; the coordinator it proposes
     * through starts at the plan's first slot, ACTIVE (setCoordinatorActive :577-587), with the nodeSlotNumbers heard */
    o.next_slot = pcs.myProposals.empty() ? pcs.nextProposalSlotNumber : pcs.myProposals[0].slot;
    const Ballot nb = pcs.getBallot();
    for (u32 l = 0; l < e->L(); l++) { /* coordinators of a lower ballot resign (PISM.handlePrepare at their node) */
      Coordinator& C = e->lanes[l].coord[el.gid];
      if (l != el.lane && C.exists && C.getBallot().compareTo(nb) > 0) continue;
      C = Coordinator();
      C.W = e->W();
    }
    Coordinator& C = e->lanes[el.lane].coord[el.gid];
    C.create(nb.num, nb.coord, o.next_slot, g.members.size(), true);
    C.active = true;
    for (size_t m = 0; m < g.members.size(); m++)
      if (jsub(C.nodeSlotNumbers[m], pcs.nodeSlotNumbers[m]) < 0) C.nodeSlotNumbers[m] = pcs.nodeSlotNumbers[m];
  }
  return GPX_OK;
}

/* PISM.handleBatchedAcceptReply :1370-1419 -> handleAcceptReply :1248-1365 per slot */
int gpxo_handle_accept_replies(gpxo_engine* e, uint32_t n, const gpx_accept_reply_rec* replies,
                               gpx_decision_rec* out_decisions, uint32_t* n_decisions) {
  u32 nd = 0;
  for (u32 i = 0; i < n; i++) {
    int lane = replyLane(e, replies[i], true);
    if (lane < 0) continue;
    if (replyAtLane(e, lane, replies[i], &out_decisions[nd])) nd++;
  }
  *n_decisions = nd;
  return GPX_OK;
}

/* PISM.handleBatchedCommit :1480-1528 per slot -> handleCommittedRequest -> extractExecuteAndCheckpoint */
int gpxo_handle_decisions(gpxo_engine* e, uint32_t n, const gpx_decision_rec* decisions, gpx_exec_rec* out_exec,
                          gpx_exec_rec* out_extra_exec, uint32_t extra_cap, uint32_t* n_extra) {
  if (n == 0) { /* an empty batch is a no-op: nothing is logged (the engine's calls return at once, too) */
    if (n_extra) *n_extra = 0;
    return GPX_OK;
  }
  return decisionsImpl(e, n, n, decisions, out_exec, out_extra_exec, extra_cap, n_extra);
}
static int decisionsImpl(gpxo_engine* e, u32 n, u32 n_slots, const gpx_decision_rec* decisions, gpx_exec_rec* out_exec,
                         gpx_exec_rec* out_extra_exec, u32 extra_cap, u32* n_extra) {
  u32 L = e->L();
  std::vector<u64> seg(L);
  for (u32 l = 0; l < L; l++) seg[l] = e->segBegin(l, GPX_F_DECISION, n_slots, 32, 0, n);
  std::vector<gpx_exec_rec> extras;
  for (u32 i = 0; i < n; i++)
    for (u32 l = 0; l < L; l++) decisionAtLane(e, i, l, decisions[i], seg[l], out_exec[(u64)i * L + l], extras);
  emitExtras(extras, out_extra_exec, extra_cap, n_extra);
  return GPX_OK;
}

/* Fused co-located path (the order the device's k_act kernel defines): per ACCEPT, in batch order --
 * handleAccept at every addressed lane; replies whose destination coordinator is a LOCAL lane are handled
 * at once (PaxosManager.send loopback, PaxosManager.java:2116-2128), the others are returned in
 * out_replies; a resulting DECISION is handled at every local lane before the next ACCEPT.
 * out_replies[n*L] (VOID where consumed locally), out_decisions[n] (VOID where none), out_exec[n*L]. */
int gpxo_handle_accepts_fused(gpxo_engine* e, uint32_t n, const gpx_accept_rec* accepts, const uint8_t* blob,
                              uint64_t blob_bytes, gpx_accept_reply_rec* out_replies, gpx_decision_rec* out_decisions,
                              gpx_exec_rec* out_exec, gpx_exec_rec* out_extra_exec, uint32_t extra_cap,
                              uint32_t* n_extra) {
  if (n == 0) { /* an empty batch is a no-op: nothing is logged (the engine's calls return at once, too) */
    if (n_extra) *n_extra = 0;
    return GPX_OK;
  }
  u32 L = e->L();
  std::vector<u64> seg(L), pay(L), dseg(L);
  for (u32 l = 0; l < L; l++) {
    seg[l] = e->segBegin(l, GPX_F_ACCEPT, n, 48, blob_bytes);
    pay[l] = seg[l] + 64 + (u64)n * 48;
    dseg[l] = e->segBegin(l, GPX_F_DECISION, n, 32, 0);
  }
  std::vector<gpx_exec_rec> extras;
  for (u32 i = 0; i < n; i++) {
    for (u32 l = 0; l < L; l++)
      acceptAtLane(e, i, l, accepts[i], blob, seg[l], pay[l], out_replies[(u64)i * L + l], extras);
    gpx_decision_rec d;
    memset(&d, 0, sizeof d);
    d.gid = accepts[i].h.gid;
    d.slot = accepts[i].h.slot;
    d.flags = GPX_F_VOID;
    bool decided = false;
    for (u32 l = 0; l < L; l++) {
      gpx_accept_reply_rec& rep = out_replies[(u64)i * L + l];
      int lane = replyLane(e, rep, false);
      if (lane < 0) continue; /* void, or addressed to a remote coordinator: stays in out_replies */
      gpx_decision_rec dd;
      if (replyAtLane(e, lane, rep, &dd) && !decided) {
        d = dd;
        decided = true;
      }
      rep.bnum = rep.bcoord = rep.max_cp = 0; /* consumed locally */
      rep.req_id = 0;
      rep.who = GPX_WHO(0xff, 0xff, GPX_F_VOID);
    }
    out_decisions[i] = d;
    for (u32 l = 0; l < L; l++) decisionAtLane(e, i, l, d, dseg[l], out_exec[(u64)i * L + l], extras);
  }
  emitExtras(extras, out_extra_exec, extra_cap, n_extra);
  return GPX_OK;
}

/* one full round, phase by phase (all ACCEPTs, then all replies, then all DECISIONs) */
int gpxo_round_phases(gpxo_engine* e, uint32_t n, const gpx_request_rec* reqs, const uint8_t* payload,
                      uint64_t payload_bytes, int32_t* status, gpx_exec_rec* out_exec, uint32_t* n_exec_slots,
                      gpx_exec_rec* out_extra_exec, uint32_t extra_cap, uint32_t* n_extra) {
  if (n == 0) { /* an empty batch is a no-op: nothing is logged (the engine's calls return at once, too) */
    if (n_exec_slots) *n_exec_slots = 0;
    if (n_extra) *n_extra = 0;
    return GPX_OK;
  }
  u32 L = e->L();
  std::vector<gpx_accept_rec> acc(n);
  std::vector<uint8_t> blob(2 * ((payload_bytes + 15) & ~15ull) + 32ull * n + 64);
  u32 na = 0;
  u64 bb = 0;
  int rc = gpxo_propose(e, n, reqs, payload, payload_bytes, acc.data(), &na, blob.data(), blob.size(), &bb, status);
  if (rc) return rc;
  std::vector<gpx_accept_reply_rec> rep((size_t)na * L + 1);
  u32 nx1 = 0, nx2 = 0;
  /* one image slot per REQUEST in both segments, as the device reserves them before the counts are known */
  rc = acceptsImpl(e, na, n, acc.data(), blob.data(), bb, rep.data(), out_extra_exec, extra_cap, &nx1);
  if (rc) return rc;
  std::vector<gpx_decision_rec> dec((size_t)na * L + 1);
  u32 nd = 0;
  rc = gpxo_handle_accept_replies(e, na * L, rep.data(), dec.data(), &nd);
  if (rc) return rc;
  u32 used = nx1 < extra_cap ? nx1 : extra_cap;
  rc = decisionsImpl(e, nd, n, dec.data(), out_exec, out_extra_exec + used, extra_cap - used, &nx2);
  if (rc) return rc;
  *n_exec_slots = nd * L;
  if (n_extra) *n_extra = nx1 + nx2;
  return GPX_OK;
}

/* one full round for co-located replicas in the fused order (PaxosManager.send routing with loopback
 * :2098-2128): RequestBatcher + propose, then per ACCEPT accept -> tally -> commit.  Records, log images
 * and EXEC rows are indexed by REQUEST (the ACCEPT of a batch sits at the index of its first request; the
 * other indices are VOID), exactly like the device's k_round kernel. */
int gpxo_round(gpxo_engine* e, uint32_t n, const gpx_request_rec* reqs, const uint8_t* payload,
               uint64_t payload_bytes, int32_t* status, gpx_exec_rec* out_exec, uint32_t* n_exec_slots,
               gpx_exec_rec* out_extra_exec, uint32_t extra_cap, uint32_t* n_extra) {
  if (n == 0) { /* an empty batch is a no-op: nothing is logged (the engine's calls return at once, too) */
    if (n_exec_slots) *n_exec_slots = 0;
    if (n_extra) *n_extra = 0;
    return GPX_OK;
  }
  u32 L = e->L();
  const u64 pal = (payload_bytes + 15) & ~(u64)15;
  const u64 blob1_res = e->cfg.batching_enabled ? 16ull * n + pal : 0;
  std::vector<gpx_accept_rec> acc(n);
  std::vector<uint8_t> blob(pal + blob1_res + 64);
  u32 na = 0;
  u64 bb = 0;
  std::vector<u32> acc_req(n);
  int rc = proposeImpl(e, n, reqs, payload, payload_bytes, acc.data(), &na, blob.data(), blob.size(), &bb, status,
                       acc_req.data());
  if (rc) return rc;
  std::vector<gpx_accept_rec> full(n);
  for (u32 i = 0; i < n; i++) {
    memset(&full[i], 0, sizeof full[i]);
    full[i].h.gid = reqs[i].gid;
    full[i].h.flags = GPX_F_VOID;
  }
  for (u32 k = 0; k < na; k++) full[acc_req[k]] = acc[k];
  std::vector<gpx_accept_reply_rec> rep((size_t)n * L + 1);
  std::vector<gpx_decision_rec> dec((size_t)n + 1);
  rc = gpxo_handle_accepts_fused(e, n, full.data(), blob.data(), pal + blob1_res, rep.data(), dec.data(), out_exec,
                                 out_extra_exec, extra_cap, n_extra);
  if (rc) return rc;
  *n_exec_slots = n * L;
  return GPX_OK;
}

int gpxo_log_read(gpxo_engine* e, uint32_t lane, uint64_t from, void* dst, uint64_t cap, uint64_t* n_copied,
                  uint64_t* head) {
  if (lane >= e->L()) return GPX_ERANGE;
  const std::vector<uint8_t>& r = e->lanes[lane].ring;
  u64 h = r.size();
  u64 nb = from < h ? std::min<u64>(cap, h - from) : 0;
  if (nb) memcpy(dst, r.data() + from, nb);
  if (n_copied) *n_copied = nb;
  if (head) *head = h;
  return GPX_OK;
}

/* AbstractPaxosLogger.getLoggedDecisions :582 / getLoggedAccepts :568 in the journaling form
 * (SQLPaxosLogger.getLoggedFromMessageLog :3674-3756 over paxosutil/LogIndex.java:213-248): per wanted slot the entry
 * logged LAST (`accepts.put(packet.slot, packet)` :3746, log order) */
int gpxo_log_find(gpxo_engine* e, uint32_t lane, uint64_t from, uint32_t n, const gpx_log_want* wants, gpx_log_hit* out) {
  if (!e || (n && (!wants || !out))) return GPX_EINVAL;
  if (lane >= e->L()) return GPX_ERANGE;
  for (u32 i = 0; i < n; i++) {
    if (wants[i].n_slots > GPX_LOG_SPAN) return GPX_ERANGE;
    if (i && wants[i - 1].gid >= wants[i].gid) return GPX_EINVAL; /* sorted by gid, one want per group */
  }
  const std::vector<uint8_t>& r = e->lanes[lane].ring;
  for (u64 t = 0; t < (u64)n * GPX_LOG_SPAN; t++) {
    memset(&out[t], 0, sizeof out[t]);
    out[t].decision.flags = GPX_F_VOID;
    out[t].accept.h.flags = GPX_F_VOID;
  }
  u64 off = from;
  while (off + 64 <= r.size()) {
    gpx_log_seg_hdr h;
    memcpy(&h, &r[off], sizeof h);
    if (h.magic != GPX_SEG_MAGIC || h.ring_off != off) return GPX_EINVAL; /* `from` is not a segment boundary */
    const u64 imgs = off + 64, pay = imgs + (u64)h.n_slots * h.rec_bytes;
    const bool isAcc = h.rec_bytes == 48, isDec = h.rec_bytes == 32 && h.type == GPX_F_DECISION;
    for (u32 j = 0; (isAcc || isDec) && j < h.n_valid; j++) {
      gpx_pvalue_hdr img;
      memcpy(&img, &r[imgs + (u64)j * 32], 32);
      if (img.flags & GPX_F_VOID) continue;
      const gpx_log_want* w = std::lower_bound(wants, wants + n, img.gid,
                                               [](const gpx_log_want& a, u32 g) { return a.gid < g; });
      if (w == wants + n || w->gid != img.gid) continue;
      const i32 k = jsub(img.slot, w->min_slot);
      if (k < 0 || (u32)k >= w->n_slots) continue;
      gpx_log_hit& hit = out[(u64)(w - wants) * GPX_LOG_SPAN + (u32)k];
      if (isDec) {
        hit.decision = img;
      } else {
        hit.accept.h = img;
        memcpy(&hit.accept.payload_off, &r[imgs + (u64)h.n_slots * 32 + (u64)j * 16], 16);
        hit.blob_pos = pay + hit.accept.payload_off;
      }
    }
    off = (pay + ((h.payload_bytes + 15) & ~(u64)15) + 31) & ~(u64)31;
  }
  return GPX_OK;
}

/* SQLPaxosLogger.getJournaledMessage(FileOffsetLength[]) :3712: the indexed frames read back in one pass */
int gpxo_log_gather(gpxo_engine* e, uint32_t lane, uint32_t n, const gpx_log_range* ranges, void* dst, uint64_t dst_bytes) {
  if (!e || (n && (!ranges || !dst))) return GPX_EINVAL;
  if (lane >= e->L()) return GPX_ERANGE;
  const std::vector<uint8_t>& r = e->lanes[lane].ring;
  u64 top = 0;
  for (u32 i = 0; i < n; i++) {
    const u64 nb = (((u64)ranges[i].len + 15) >> 4) << 4;
    if ((ranges[i].pos & 15) || (ranges[i].dst_off & 15)) return GPX_EINVAL;
    if (ranges[i].pos + nb > r.size() || (u64)ranges[i].dst_off + nb > dst_bytes) return GPX_ERANGE;
    top = std::max<u64>(top, (u64)ranges[i].dst_off + nb);
  }
  memset(dst, 0, top);
  for (u32 i = 0; i < n; i++) memcpy((uint8_t*)dst + ranges[i].dst_off, &r[ranges[i].pos], (((u64)ranges[i].len + 15) >> 4) << 4);
  return GPX_OK;
}

/* drop the in-memory log (a drained / garbage-collected journal); used by long CPU-baseline runs */
int gpxo_log_truncate(gpxo_engine* e) {
  for (auto& ln : e->lanes) {
    std::vector<uint8_t>().swap(ln.ring);
  }
  return GPX_OK;
}

int gpxo_get_counters(gpxo_engine* e, gpx_counters* out) {
  *out = e->ctr;
  return GPX_OK;
}
int gpxo_reset_counters(gpxo_engine* e) {
  memset(&e->ctr, 0, sizeof e->ctr);
  return GPX_OK;
}
/* group flags (GF_*) of one lane, for the host slow-path list */
int gpxo_get_group_flags(gpxo_engine* e, uint32_t lane, uint32_t n, const uint32_t* gids, uint8_t* out) {
  if (lane >= e->L()) return GPX_ERANGE;
  for (u32 k = 0; k < n; k++) {
    out[k] = 0;
    if (gids[k] >= e->cfg.max_groups) continue;
    const Acceptor& A = e->lanes[lane].acc[gids[k]];
    const Coordinator& C = e->lanes[lane].coord[gids[k]];
    /* PaxosAcceptor.caughtUp :452-459, PaxosCoordinator.caughtUp :369-371 / PCS.caughtUp :758-761 */
    bool caughtUp = A.committedRequests.empty() && (A.acceptedProposals.empty() || A.journaling);
    if (C.exists && !C.myProposals.empty()) caughtUp = false;
    out[k] = (uint8_t)(A.flags | (caughtUp ? 0u : GPX_GF_NOT_CAUGHT_UP_BIT));
  }
  return GPX_OK;
}

/* PISM.requestMissingDecisions :2292-2320 for a batch: PaxosAcceptor.getMaxCommittedSlot :425-438,
 * getMissingCommittedSlots :405-423, PISM.isMissingTooMuch :2367-2370 / shouldSync :2341-2361 */
int gpxo_missing_decisions(gpxo_engine* e, uint32_t lane, uint32_t n, const uint32_t* gids, int32_t size_limit,
                           int32_t too_much_gap, gpx_missing_rec* out) {
  if (!e || ((!gids || !out) && n)) return GPX_EINVAL;
  if (lane >= e->L()) return GPX_ERANGE;
  for (u32 k = 0; k < n; k++) {
    gpx_missing_rec& r = out[k];
    memset(&r, 0, sizeof r);
    const u32 gid = gids[k];
    r.gid = gid;
    if (gid >= e->groups.size() || !e->groups[gid].live || e->memberIdx(e->groups[gid], e->lanes[lane].node) < 0) continue;
    const Acceptor& A = e->lanes[lane].acc[gid];
    r.slot = A._slot;
    uint8_t fl = 0;
    gpxo_get_group_flags(e, lane, 1, &gid, &fl);
    r.flags = fl;
    /* getMaxCommittedSlot :425-438 */
    i32 maxCommitted = (i32)((u32)A._slot - 1u);
    if (!A.isStopped() && !A.committedRequests.empty()) {
      maxCommitted = (i32)((u32)A._slot - 1u);
      for (auto& kv : A.committedRequests)
        if (jsub(kv.first, maxCommitted) > 0) maxCommitted = kv.first;
    }
    r.max_decision_slot = maxCommitted;
    if (!e->usable(gid, lane)) continue; /* getMissingCommittedSlots returns null when stopped :407-408 */
    /* getMissingCommittedSlots(sizeLimit) :405-423 */
    u32 nm = 0;
    const i32 limitSlot = (i32)((u32)A._slot + (u32)size_limit);
    for (i32 i = A._slot; jsub(i, maxCommitted) < 0 && jsub(i, limitSlot) < 0 && nm < GPX_MAX_WINDOW; i = (i32)((u32)i + 1u)) {
      auto c = A.committedRequests.find(i);
      if (c == A.committedRequests.end() || (!c->second.has_value && !A.acceptedProposals.count(i))) r.missing[nm++] = i;
    }
    if (nm == 0) r.missing[nm++] = A._slot; /* requestMissingDecisions :2297-2298 */
    r.n_missing = (uint16_t)nm;
    /* shouldSync(maxDecisionSlot, threshold, DEFAULT_SYNC) :2341-2361 */
    const i32 gap = jsub(maxCommitted, A._slot);
    const bool nontrivialInitialGap = gap >= too_much_gap / 100, smallGapThreshold = too_much_gap <= 1;
    r.missing_too_much = (gap >= too_much_gap) || ((A._slot == 0 || A._slot == 1) && (nontrivialInitialGap || smallGapThreshold));
  }
  return GPX_OK;
}

int gpxo_clear_group_flags(gpxo_engine* e, uint32_t lane, uint32_t n, const uint32_t* gids, uint32_t mask) {
  if (!e || (!gids && n)) return GPX_EINVAL;
  if (lane >= e->L()) return GPX_ERANGE;
  for (u32 k = 0; k < n; k++)
    if (gids[k] < e->groups.size()) e->lanes[lane].acc[gids[k]].flags &= (uint8_t) ~(mask & (GF_OVERFLOW | GF_NEEDS_SYNC));
  return GPX_OK;
}

/* the test of a sweep over all instances (PaxosManager.syncAndDeactivate :2806-2900 iterates pinstances) */
int gpxo_select_groups(gpxo_engine* e, uint32_t lane, uint32_t mask, uint32_t value, uint32_t* out_gids, uint32_t cap,
                       uint32_t* n_found) {
  if (!e || !n_found || (!out_gids && cap)) return GPX_EINVAL;
  if (lane >= e->L()) return GPX_ERANGE;
  u32 found = 0;
  for (u32 gid = 0; gid < e->groups.size(); gid++) {
    if (!e->usable(gid, lane) || e->memberIdx(e->groups[gid], e->lanes[lane].node) < 0) continue;
    uint8_t fl = 0;
    int rc = gpxo_get_group_flags(e, lane, 1, &gid, &fl);
    if (rc) return rc;
    if ((fl & mask) != value) continue;
    if (found < cap) out_gids[found] = gid;
    found++;
  }
  *n_found = found;
  return GPX_OK;
}

/* PaxosManager.pause(Map, dequeue) :2327-2366 over PISM.tryPause :2004-2035 at every local replica of each group */
int gpxo_pause_groups(gpxo_engine* e, uint32_t n, const uint32_t* gids, gpx_row* out_rows, uint8_t* out_paused) {
  if (!e || (n && (!gids || !out_rows || !out_paused))) return GPX_EINVAL;
  {
    std::vector<u32> seen(gids, gids + n);
    std::sort(seen.begin(), seen.end());
    if (std::adjacent_find(seen.begin(), seen.end()) != seen.end()) return GPX_EINVAL;
  }
  for (u32 i = 0; i < n; i++) {
    const u32 gid = gids[i];
    bool ok = gid < e->groups.size() && e->groups[gid].live;
    for (u32 l = 0; ok && l < e->L(); l++) {
      if (e->memberIdx(e->groups[gid], e->lanes[l].node) < 0) continue;
      uint8_t fl = 0;
      if (!e->usable(gid, l)) ok = false; /* tryPause is for a running instance */
      else if (gpxo_get_group_flags(e, l, 1, &gid, &fl) != GPX_OK || (fl & GPX_GF_NOT_CAUGHT_UP_BIT)) ok = false;
    }
    out_paused[i] = ok ? 1 : 0;
    if (!ok) continue;
    for (u32 l = 0; l < e->L(); l++) {
      int rc = gpxo_dump_rows(e, 1, &gid, l, &out_rows[(u64)i * e->L() + l]); /* the HotRestoreInfo :2009-2021 */
      if (rc) return rc;
    }
    int rc = gpxo_destroy_groups(e, 1, &gid); /* forceStop :2025 + softCrash PaxosManager.java:2298 */
    if (rc) return rc;
  }
  return GPX_OK;
}

int32_t gpxo_java_string_hash(const char* s, size_t len) { return javaStringHash(s, len); }
int32_t gpxo_round_robin_coordinator(int32_t name_hash, const int32_t* sorted_members, int32_t n, int32_t ballotnum) {
  return roundRobinCoordinator(name_hash, sorted_members, n, ballotnum);
}
int32_t gpxo_get_cpi(int32_t cpi, double noise, int32_t name_hash) { return getCPI(cpi, noise, name_hash); }
int32_t gpxo_last_checkpoint_slot(int32_t slot, int32_t cpi) { return lastCheckpointSlot(slot, cpi); }
void gpxo_md5(const uint8_t* msg, size_t len, uint8_t out[16]) { md5(msg, len, out); }
int gpxo_digest_requests(gpxo_engine* e, uint32_t n, const gpx_request_rec* reqs, const uint8_t* payload,
                         uint64_t payload_bytes, uint8_t* out_digests) {
  (void)e;
  (void)payload_bytes;
  for (u32 i = 0; i < n; i++) md5(payload + reqs[i].payload_off, reqs[i].payload_len, out_digests + 16ull * i);
  return GPX_OK;
}

/* HotRestoreInfo string round trip: parse `in`, re-serialise into out (cap bytes) */
int gpxo_hri_roundtrip(const char* in, char* out, size_t cap) {
  HotRestoreInfo h = HotRestoreInfo::parse(in);
  std::string s = h.toString();
  if (s.size() + 1 > cap) return GPX_ERANGE;
  memcpy(out, s.c_str(), s.size() + 1);
  return GPX_OK;
}
int gpxo_hri_from_row(const char* paxosID, const gpx_row* r, char* out, size_t cap) {
  HotRestoreInfo h;
  h.paxosID = paxosID;
  h.version = r->version;
  h.members.assign(r->members, r->members + r->n_members);
  h.accSlot = r->acc_slot;
  h.accBallot = Ballot{r->acc_bnum, r->acc_bcoord};
  h.accGCSlot = r->acc_gc_slot;
  /* PISM.tryPause :2004-2025: getBallotIfActive / getNextProposalSlotIfActive / getNodeSlotsIfActive
   * (PaxosCoordinator.java:375-402): null, -1, null unless the coordinator is ACTIVE */
  const bool active = r->coord_exists != 0 && r->coord_active != 0;
  h.hasCoord = active;
  h.coordBallot = Ballot{r->coord_bnum, r->coord_bcoord};
  h.nextProposalSlot = active ? r->next_proposal_slot : -1;
  h.hasNodeSlots = active;
  h.nodeSlots.assign(r->node_slots, r->node_slots + r->n_members);
  std::string s = h.toString();
  if (s.size() + 1 > cap) return GPX_ERANGE;
  memcpy(out, s.c_str(), s.size() + 1);
  return GPX_OK;
}

/* ------------------------------------------------------------------------------
 * Self-tests: transliterations of the reference's own main()/JUnit tests.
 * Returns 0 on success, else the number of the failing check (message in last_error).
 * ---------------------------------------------------------------------------- */
static u64 g_rng = 0x9E3779B97F4A7C15ull;
static u64 splitmix() {
  u64 z = (g_rng += 0x9E3779B97F4A7C15ull);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
static double rnd() { return (double)(splitmix() >> 11) / (double)(1ull << 53); }

#define CHECK(n, cond)                                      \
  do {                                                      \
    if (!(cond)) {                                          \
      g_err = std::string("selftest check failed: ") + #cond; \
      return (n);                                           \
    }                                                       \
  } while (0)

int gpxo_selftest(uint64_t seed) {
  g_rng = seed ? seed : 1;
  /* 1. Ballot: PaxosPacketBatcher.main :556-567 + compareTo wraparound */
  {
    Ballot b1{43, 578}, b2{43, 578};
    CHECK(1, b1.equals(b2));
    CHECK(2, b1.hashCode() == b2.hashCode());
    CHECK(3, (Ballot{1, 0}).compareTo(Ballot{0, 5}) > 0);
    CHECK(4, (Ballot{0, 2}).compareTo(Ballot{0, 1}) > 0);
    CHECK(5, (Ballot{INT32_MIN, 0}).compareTo(Ballot{INT32_MAX, 0}) > 0); /* wraparound :62-63 */
  }
  /* 2. WaitforUtility.main :147-163 */
  {
    WaitforUtility w(std::vector<i32>{0, 9, 4, 23});
    CHECK(10, !w.contains(32));
    CHECK(11, w.contains(9));
    CHECK(12, w.getIndex(4) == 2);
    CHECK(13, w.updateHeardFrom(9));
    CHECK(14, !w.heardFromMajority());
    CHECK(15, w.updateHeardFrom(23));
    CHECK(16, !w.heardFromMajority());
    CHECK(17, w.updateHeardFrom(0));
    CHECK(18, w.heardFromMajority());
    CHECK(19, !w.updateHeardFrom(0)); /* idempotent */
  }
  /* 3. PaxosAcceptor.testAcceptor :749-776 (100k random accepts, then 100k random prepares) */
  {
    Acceptor acceptor;
    acceptor.ballotNum = 22;
    acceptor.ballotCoord = 1;
    acceptor._slot = 7;
    acceptor.state = ST_ACTIVE_1;
    const int numTests = 100000;
    for (int i = 0; i < numTests; i++) {
      PValue accept;
      accept.slot = (i32)(rnd() * INT32_MAX); /* getRandomAccept :728-738 */
      accept.bal = Ballot{(i32)(rnd() * INT32_MAX), (i32)(rnd() * INT32_MAX)};
      accept.req_id = (i64)splitmix();
      accept.has_value = true;
      accept.median_cp = 0;
      Ballot before = acceptor.getBallot(), response;
      CHECK(30, acceptor.acceptAndUpdateBallot(accept, &response));
      CHECK(31, response.compareTo(accept.bal) >= 0);
      CHECK(32, response.compareTo(before) >= 0);
    }
    for (int i = 0; i < numTests; i++) {
      Ballot pb{(i32)(rnd() * INT32_MAX), (i32)(rnd() * INT32_MAX)};
      Ballot before = acceptor.getBallot();
      acceptor.bumpBallot(pb); /* handlePrepare :239-251 */
      CHECK(33, acceptor.getBallot().compareTo(pb) >= 0);
      CHECK(34, acceptor.getBallot().compareTo(before) >= 0);
    }
  }
  /* 4. PaxosCoordinatorState.main, phase-2 half :1179-1214 (43 members, random preemption) */
  {
    const int numMembers = 43;
    std::vector<i32> members(numMembers);
    members[0] = 21;
    for (int i = 1; i < numMembers; i++) members[i] = members[i - 1] + 1 + (int)(rnd() * 10);
    Coordinator pcs;
    pcs.create(2, 21, 0, numMembers, true);
    pcs.active = true;
    for (int i = 0; i < 100; i++) {
      PValue req, acc;
      req.req_id = (i64)splitmix();
      req.has_value = true;
      CHECK(40, pcs.propose(members, req, &acc) == 0);
      CHECK(41, acc.slot == i && acc.bal.num == 2 && acc.bal.coord == 21);
    }
    std::vector<i32> slots;
    for (auto& kv : pcs.myProposals) slots.push_back(kv.first);
    for (i32 s : slots) {
      CHECK(42, !pcs.preemptedFully());
      for (int j = 0; j < numMembers; j++) {
        PValue out;
        if (rnd() > 0.99) { /* a single member's higher-ballot reply preempts */
          int t = pcs.handleAcceptReplyHigherBallot(s, &out);
          CHECK(43, t == PT_NONE || t == PT_PREEMPTED);
          if (t == PT_PREEMPTED) CHECK(44, !pcs.myProposals.count(out.slot));
        } else {
          bool present = pcs.myProposals.count(s) != 0;
          int heardBefore = present ? pcs.myProposals[s].waitfor.heardCount : 0;
          int t = pcs.handleAcceptReplyMyBallot(members, members[j], s, -1, &out);
          CHECK(45, t == PT_NONE || t == PT_DECISION);
          if (t == PT_DECISION) {
            CHECK(46, !pcs.myProposals.count(out.slot));
            CHECK(47, heardBefore + 1 > numMembers / 2); /* decisions only on majority */
          }
        }
      }
    }
    CHECK(48, pcs.myProposals.empty());
  }
  /* 5. HotRestoreInfoTest.testToStringAndBack paxosutil/HotRestoreInfo.java:159-175 (literal values) */
  {
    HotRestoreInfo h;
    h.paxosID = "paxos0";
    h.version = 2;
    h.members = {1, 4, 67};
    h.accSlot = 5;
    h.accBallot = Ballot{3, 4};
    h.accGCSlot = 3;
    h.hasCoord = true;
    h.coordBallot = Ballot{45, 67};
    h.nextProposalSlot = 34;
    h.hasNodeSlots = true;
    h.nodeSlots = {1, 3, 5};
    std::string s1 = h.toString();
    CHECK(50, s1 == "paxos0|2|[1,4,67]|5|3:4|3|45:67|34|[1,3,5]"); /* Util.arrayOfIntToString: no blanks */
    CHECK(51, HotRestoreInfo::parse(s1).toString() == s1);
  }
  /* 6. medianMinus :867-875, roundRobinCoordinator :2251-2256, String.hashCode */
  {
    Coordinator c;
    c.create(0, 1, 1, 3, true);
    c.nodeSlotNumbers = {5, 1, 3};
    CHECK(60, c.getMajorityCommittedSlot() == 3);
    c.nodeSlotNumbers = {5, 1, 3, 9};
    CHECK(61, c.getMajorityCommittedSlot() == 3); /* even: index n/2-1 */
    CHECK(62, javaStringHash("paxos0", 6) == -995235643);
    CHECK(63, javaStringHash("", 0) == 0);
    i32 m[3] = {100, 101, 102};
    CHECK(64, roundRobinCoordinator(javaStringHash("paxos0", 6), m, 3, 0) == m[995235643 % 3]);
    CHECK(65, getCPI(400, 0.0, 12345) == 400);
    CHECK(66, lastCheckpointSlot(805, 400) == 800);
  }
  /* 7. MD5: RFC 1321 appendix A.5 test suite */
  {
    struct { const char* in; const char* hex; } v[] = {
        {"", "d41d8cd98f00b204e9800998ecf8427e"},
        {"a", "0cc175b9c0f1b6a831c399e269772661"},
        {"abc", "900150983cd24fb0d6963f7d28e17f72"},
        {"message digest", "f96b697d7cb7938d525a2f31aaf161d0"},
        {"abcdefghijklmnopqrstuvwxyz", "c3fcd3d76192e4007dfb496cca67e13b"},
        {"ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789", "d174ab98d277d9f5a5611c2c9f419d9f"},
        {"12345678901234567890123456789012345678901234567890123456789012345678901234567890",
         "57edf4a22be3c955ac49da2e2107b67a"}};
    for (auto& t : v) {
      uint8_t d[16];
      md5((const uint8_t*)t.in, strlen(t.in), d);
      char hex[33];
      for (int i = 0; i < 16; i++) snprintf(hex + 2 * i, 3, "%02x", d[i]);
      CHECK(70, std::string(hex) == t.hex);
    }
  }
  return 0;
}

} /* extern "C" */
