/*
 * gpx.h -- C ABI of the H100-native batched-Paxos engine (gigapaxos hot path).
 *
 * This is the drop-in boundary (SURVEY.md 8b). gigapaxos has no FFI seam on this
 * path today; the seam defined here is the narrow waist already present in the
 * Java code.  Every entry point cites the reference interface it replaces
 * (paths relative to /root/reference/src/edu/umass/cs/gigapaxos/):
 *
 *   gpx_engine_create / gpx_config_from_properties
 *        <- PaxosConfig.java:64,83-90 (gigapaxos.properties), PaxosManager ctor
 *           PaxosManager.java:392-462
 *   gpx_create_groups        <- PaxosManager.createPaxosInstance :632, batch form :664-691,
 *                               HotRestoreInfo.createHRI paxosutil/HotRestoreInfo.java:145-157,
 *                               PaxosInstanceStateMachine.initiateRecovery :591-675
 *   gpx_destroy_groups       <- PaxosManager.kill :2162
 *   gpx_dump_rows/load_rows  <- PaxosManager pause/unpause :2284,:2370 (HotRestoreInfo field set)
 *   gpx_patch                <- PaxosAcceptor.handlePrepare :245-251 (ballot bump),
 *                               jumpSlot :564-578, forceStop :154; coordinator install/resign
 *   gpx_propose              <- RequestBatcher.enqueueImpl/dequeueImpl RequestBatcher.java:112-234,
 *                               PISM.handleRequest :767 / handleProposal :818,
 *                               PaxosCoordinatorState.propose :233-263
 *   gpx_handle_accepts       <- PISM.handleAccept :1080-1166 (+ AbstractPaxosLogger.logAndMessage :157)
 *   gpx_handle_accept_replies<- PISM.handleBatchedAcceptReply :1370 / handleAcceptReply :1248
 *   gpx_handle_decisions     <- PISM.handleBatchedCommit :1480 / handleCommittedRequest :1432 /
 *                               extractExecuteAndCheckpoint :1619 (EXEC records replace app.execute :1802)
 *   gpx_round                <- one full pass of the above for co-located replicas
 *                               (PaxosManager.send :2098-2128 routing incl. loopback)
 *   gpx_log_read             <- SQLPaxosLogger.journal :965-1036 / Journaler.appendToLogFile :814-826
 *   gpx_handle_prepares      <- PISM.handlePrepare :900-955, PaxosAcceptor.handlePrepare :239-297
 *   gpx_handle_prepare_replies <- PISM.handlePrepareReply :1017-1068, PaxosCoordinatorState.java:264-587 (phase 1b)
 *   gpx_select_groups / gpx_missing_decisions / gpx_clear_group_flags / gpx_pause_groups
 *                            <- PaxosManager.syncAndDeactivate :2806-2900 (the sweep over pinstances),
 *                               PISM.requestMissingDecisions :2292-2320, tryPause :2004-2035, pause(Map, dequeue) :2327-2366
 *   gpx_log_find / gpx_log_gather <- AbstractPaxosLogger.getLoggedDecisions :582 / getLoggedAccepts :568
 *                               (SQLPaxosLogger.getLoggedFromMessageLog :3674-3756, paxosutil/LogIndex.java:213-248)
 *   gpx_wire_*               <- paxospackets byte codecs (RequestPacket.java:819-1024,
 *                               AcceptPacket.java:95-138, BatchedAcceptReply.java:103-173,
 *                               BatchedCommit.java:184-252, PaxosPacket.java:443-476)
 *   gpx_response_cache_*     <- PaxosManager.handleIncomingPacket :1084, retransmittedRequest :332-349,
 *                               executed :311-330 (ENABLE_RESPONSE_CACHING)
 *
 * Conventions (mirror the reference, SURVEY.md 8b): int return codes are for API
 * misuse only; protocol-level rejects (stopped group, stale ballot, unknown
 * acceptor, window overflow) are counted and dropped, never fatal.  The engine is
 * single-submitter and batch-synchronous: one call = one batch, per-group order
 * inside a batch is the order of the records in the batch.  The caller owns all
 * input and output buffers; the engine owns device memory.
 *
 * All records are little-endian, fixed size, 16-byte multiples.
 * A `gid` is a dense handle for one (paxosID, version) instance -- the analogue
 * of a PaxosInstanceStateMachine object reference; the version drop rule
 * (PISM :441-447) is applied where (paxosID, version) is mapped to a gid
 * (gpx_wire_decode_*).
 */
#ifndef GPX_H
#define GPX_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GPX_ABI_VERSION 2

#define GPX_MAX_GROUP_SIZE 16 /* PC.MAX_GROUP_SIZE, PaxosConfig.java:532 */
#define GPX_MAX_LANES 8       /* co-located replicas (lanes) per engine */
#define GPX_MAX_WINDOW 8      /* per-group in-flight slot window W (power of two) */
#define GPX_MAX_MSETS 4096    /* distinct member sets per engine */

/* return codes (API misuse / environment only) */
enum {
  GPX_OK = 0,
  GPX_EINVAL = -1,
  GPX_ENOMEM = -2,
  GPX_ECUDA = -3,
  GPX_ENOGPU = -4,
  GPX_ERANGE = -5,
  GPX_EIO = -6,
  GPX_EAGAIN = -7, /* log ring full (log_backpressure): drain + release, then repeat the call; nothing was done */
  GPX_ENOENT = -8  /* gpx_log_frame_device: a logged request or group name is not known; the misses are listed */
};

/* PaxosAcceptor.STATES ordinals (PaxosAcceptor.java:87-92); FREE = no instance */
enum {
  GPX_ST_RECOVERY = 0,
  GPX_ST_ACTIVE_1 = 1,
  GPX_ST_ACTIVE_2 = 2,
  GPX_ST_STOPPED = 3,
  GPX_ST_FREE = 255
};

/* record flags (uint16 `flags` of gpx_pvalue_hdr, low half of request/exec flags) */
#define GPX_F_STOP 0x0001u       /* RequestPacket.stop */
#define GPX_F_VOID 0x0002u       /* hole: ignore this record / frame */
#define GPX_F_ACCEPT 0x0004u     /* log frame / record is an ACCEPT (48 B + blob) */
#define GPX_F_DECISION 0x0008u   /* log frame / record is a DECISION (32 B) */
#define GPX_F_META 0x0010u       /* decision log frame is PValuePacket.getMetaDecision() form */
#define GPX_F_CKPT 0x0020u       /* exec: PISM.shouldCheckpoint() is true for this slot */
#define GPX_F_LOGGED 0x0040u     /* accept reply was released by a log append (LogMessagingTask) */
#define GPX_F_NACK 0x0080u       /* accept reply carries a ballot higher than the accept's */
#define GPX_F_EXTRA 0x0100u      /* exec/decision came from the reconstructDecision path */
#define GPX_F_PREPARE 0x0200u    /* log frame / record is a PREPARE (32 B pvalue header, slot = firstUndecidedSlot) */
#define GPX_F_FROM_LOG 0x0400u   /* prepare reply: journaling serves accepted pvalues from the log (GET_ACCEPTED_
                                  * PVALUES_FROM_DISK) and the preparer is behind this acceptor -> the host adds the
                                  * logged accepts of [firstUndecidedSlot, acceptor's slot) from the journal */

/* request status written by gpx_propose (one int32 per request): the slot, or one of these codes.  A wrapped slot
 * may equal a code (gpx_propose) */
#define GPX_RS_BATCHED (-1)      /* latched into the batch of an earlier request of the group */
#define GPX_RS_FORWARD (-2)      /* coordinator is a remote node: forward PROPOSAL (host) */
#define GPX_RS_REFUSED_STOP (-3) /* PCS.propose refused: previous proposal is a STOP */
#define GPX_RS_BACKPRESSURE (-4) /* proposal window full (W in flight); resubmit later */
#define GPX_RS_DROPPED (-5)      /* group stopped / free (PISM :456-460) */
#define GPX_RS_PREACTIVE (-6)    /* coordinator exists but is not active: host slow path */
#define GPX_RS_NOCOORD (-7)      /* no usable coordinator on any local lane: host slow path */

/* ---- records -------------------------------------------------------------- */

/* client request handed to the RequestBatcher (RequestPacket essentials), 32 B */
typedef struct gpx_request_rec {
  uint32_t gid;
  uint32_t flags;       /* bit0 GPX_F_STOP; bits 8..11 entry lane */
  int64_t req_id;       /* RequestPacket.requestID */
  uint32_t payload_off; /* byte offset of requestValue in the batch payload arena */
  uint32_t payload_len;
  int32_t entry_node;   /* RequestPacket.entryReplica (node id) */
  uint32_t client;      /* opaque client handle, carried through */
} gpx_request_rec;

/* common prefix of ACCEPT and DECISION (PValuePacket), 32 B */
typedef struct gpx_pvalue_hdr {
  uint32_t gid;
  int32_t slot;      /* ProposalPacket.slot */
  int32_t bnum;      /* Ballot.ballotNumber */
  int32_t bcoord;    /* Ballot.coordinatorID (node id) */
  int32_t median_cp; /* PValuePacket.medianCheckpointedSlot */
  uint16_t flags;    /* GPX_F_* */
  uint16_t dst_mask; /* local lanes this record is addressed to */
  int64_t req_id;    /* requestID of the first request of the slot */
} gpx_pvalue_hdr;

typedef gpx_pvalue_hdr gpx_decision_rec; /* DECISION / one slot of a BATCHED_COMMIT, 32 B */

/* ACCEPT (AcceptPacket), 48 B.  The request body ("blob") lives in a payload
 * arena: nreq==1 -> the raw requestValue bytes; nreq>1 -> nreq x gpx_batch_ent
 * followed by the concatenated requestValues (RequestPacket.batched). */
typedef struct gpx_accept_rec {
  gpx_pvalue_hdr h;
  uint32_t payload_off;
  uint32_t payload_len;
  uint32_t nreq;
  int32_t sender; /* AcceptPacket.sender (node id) == coordinator that issued it */
} gpx_accept_rec;

/* per-request entry of a batched blob, 16 B */
typedef struct gpx_batch_ent {
  int64_t req_id;
  uint32_t len;
  uint32_t flags; /* bit0 STOP; bits 8.. entry lane (as gpx_request_rec.flags) */
} gpx_batch_ent;

/* ACCEPT_REPLY / one slot of a BATCHED_ACCEPT_REPLY, 32 B */
typedef struct gpx_accept_reply_rec {
  uint32_t gid;
  int32_t slot;   /* AcceptReplyPacket.slotNumber */
  int32_t bnum;   /* acceptor's ballot after handling the accept */
  int32_t bcoord;
  int32_t max_cp; /* AcceptReplyPacket.maxCheckpointedSlot (= acceptor slot - 1) */
  uint32_t who;   /* bits 0..7 acceptor member index, 8..15 destination member index
                     (the accept's sender), 16..31 flags (GPX_F_VOID|LOGGED|NACK) */
  int64_t req_id;
} gpx_accept_reply_rec;

#define GPX_WHO(acc_idx, dst_idx, flags) \
  ((uint32_t)(acc_idx) | ((uint32_t)(dst_idx) << 8) | ((uint32_t)(flags) << 16))
#define GPX_WHO_ACC(w) ((w) & 0xffu)
#define GPX_WHO_DST(w) (((w) >> 8) & 0xffu)
#define GPX_WHO_FLAGS(w) ((w) >> 16)

/* in-order execution record handed to the Replicable app, 24 B */
typedef struct gpx_exec_rec {
  uint32_t gid;
  int32_t slot;
  int64_t req_id;
  uint32_t payload_off; /* (byte offset of the blob in the lane's log ring) / 16 */
  uint32_t flags;       /* bits 0..11 GPX_F_STOP|VOID|CKPT|EXTRA; bits 12..15 lane; bits 16..31 nreq */
} gpx_exec_rec;

/* ---- log ring ---------------------------------------------------------------
 * One ring per lane.  A ring is a sequence of segments, one per kernel launch
 * that logs: [gpx_log_seg_hdr 64 B][n_slots record images][payload area].
 * ACCEPT segment (rec_bytes 48): the images are stored as two planes, n_slots x 32 B pvalue
 * headers followed by n_slots x 16 B {payload_off,payload_len,nreq,sender}, so that every image
 * moves as one 32-byte plus one 16-byte aligned store; image.payload_off is relative to the
 * segment's payload area; unlogged records have GPX_F_VOID.  Segments are 32-byte multiples.
 * DECISION segment: images are gpx_decision_rec (32 B), no payload area.
 * (SQLPaxosLogger.journal frames {int32 len}{packet bytes}, :1000-1003; gpx_log_frame_device
 * re-frames segments into that byte format.) */
#define GPX_SEG_MAGIC 0x53585047u /* "GPXS" */
typedef struct gpx_log_seg_hdr {
  uint32_t magic;
  uint16_t type; /* GPX_F_ACCEPT or GPX_F_DECISION */
  uint16_t lane;
  uint32_t n_slots;       /* record images reserved */
  uint32_t n_valid;       /* leading image slots in use (<= n_slots); some of them may be VOID holes */
  uint64_t payload_bytes; /* payload area bytes (ACCEPT segments) */
  uint64_t seq;           /* segment sequence number of this lane */
  uint64_t ring_off;      /* absolute ring offset of this header */
  uint32_t rec_bytes;     /* 48 or 32 */
  uint32_t reserved[5];
} gpx_log_seg_hdr;

/* ---- group management ------------------------------------------------------- */

/* HotRestoreInfo field set for one (lane, gid) row, paxosutil/HotRestoreInfo.java:31-120 */
typedef struct gpx_row {
  uint32_t gid;
  uint32_t lane;
  int32_t version;
  int32_t acc_slot;       /* accSlot */
  int32_t acc_bnum;       /* accBallot */
  int32_t acc_bcoord;
  int32_t acc_gc_slot;    /* accGCSlot */
  int32_t state;          /* GPX_ST_* */
  int32_t coord_exists;   /* coordBallot != null */
  int32_t coord_active;
  int32_t coord_bnum;
  int32_t coord_bcoord;
  int32_t next_proposal_slot;
  int32_t n_members;
  int32_t members[GPX_MAX_GROUP_SIZE];    /* sorted ascending node ids */
  int32_t node_slots[GPX_MAX_GROUP_SIZE]; /* PaxosCoordinatorState.nodeSlotNumbers */
  int32_t name_hash;      /* String.hashCode() of the paxosID (HotRestoreInfo.paxosID): getCPI :2694-2697 is a function of
                           * the paxosID, and a restored instance may get a different gid than it was created under */
} gpx_row;

#define GPX_INIT_BATCH 0   /* HotRestoreInfo.createHRI path (PaxosManager.java:664-691) */
#define GPX_INIT_DEFAULT 1 /* PISM.initiateRecovery + putInitialState path (:591-703) */

typedef struct gpx_group_desc {
  uint32_t gid;
  int32_t version;
  int32_t name_hash; /* Java String.hashCode() of the paxosID */
  int32_t n_members;
  int32_t members[GPX_MAX_GROUP_SIZE]; /* distinct node ids, any order (sorted by the engine); a call with a
                                        * node listed twice is refused (GPX_ERANGE) and changes nothing */
  int32_t init_mode;                   /* GPX_INIT_* */
} gpx_group_desc;

/* host -> device state patch (slow path effects), applied between batches */
enum {
  GPX_PATCH_SET_BALLOT = 1,    /* acceptor ballot <- (a,b) if higher (handlePrepare) */
  GPX_PATCH_JUMP_SLOT = 2,     /* acceptor.jumpSlot(a) */
  GPX_PATCH_SET_STATE = 3,     /* acceptor state <- a (forceStop, setActive) */
  GPX_PATCH_INSTALL_COORD = 4, /* coordinator (bnum=a, bcoord=b, next=c, active=d) */
  GPX_PATCH_RESIGN_COORD = 5,  /* coordinator <- null */
  GPX_PATCH_SET_GC = 6,        /* acceptedGCSlot <- a */
  GPX_PATCH_SET_NODE_SLOT = 7  /* coordinator's nodeSlotNumbers[a] <- b if higher (recordSlotNumber :786-807 on a
                                * PREPARE_REPLY, host side of phase 1) */
};
typedef struct gpx_patch_rec {
  uint32_t gid;
  uint32_t lane;
  int32_t op;
  int32_t a, b, c, d;
  int32_t reserved;
} gpx_patch_rec;

/* ---- configuration ----------------------------------------------------------- */

typedef struct gpx_config {
  uint32_t abi_version;
  int32_t device;            /* CUDA device ordinal */
  uint32_t max_groups;       /* PINSTANCES_CAPACITY analogue: rows per lane */
  uint32_t n_lanes;          /* co-located replicas */
  int32_t lane_node[GPX_MAX_LANES]; /* node id served by each lane, distinct (GPX_EINVAL otherwise) */
  uint32_t window;           /* W: 1,2,4,8 */
  uint32_t max_group_size;   /* <= GPX_MAX_GROUP_SIZE: node_slots columns allocated */
  uint64_t log_ring_bytes;   /* per lane, power of two; 0 => logging disabled (DISABLE_LOGGING) */
  uint32_t max_batch_recs;   /* largest record batch one call may carry */
  uint64_t max_batch_payload;/* largest payload arena one call may carry */
  /* gigapaxos.properties subset (PaxosConfig.java PC enum), same defaults */
  int32_t batching_enabled;        /* BATCHING_ENABLED :309 (true) */
  int32_t max_batch_size;          /* MAX_BATCH_SIZE :403 (2000) */
  int64_t max_batch_bytes;         /* min(NIO MAX_PAYLOAD_SIZE 4MB, MAX_LOG_MESSAGE_SIZE 5MB) */
  int32_t request_size_estimate;   /* RequestPacket.SIZE_ESTIMATE (:1351-1367) */
  int32_t checkpoint_interval;     /* CHECKPOINT_INTERVAL :410 (400) */
  double cpi_noise;                /* CPI_NOISE :746 (0) */
  int32_t gc_majority_executed;    /* GC_MAJORITY_EXECUTED :882 (true) */
  int32_t log_meta_decisions;      /* LOG_META_DECISIONS :588 (true) */
  int32_t journaling_enabled;      /* ENABLE_JOURNALING :240 (true): executed accepts leave memory */
  /* (BATCHED_ACCEPT_REPLIES :458, BATCHED_COMMITS :466, MIN_PP_BATCH_SIZE :860 shape how PaxosPacketBatcher packs
   * records into wire packets -- the engine exchanges fixed-size records, packing happens where packets are formed
   * (gpx_wire_*); SHORT_CIRCUIT_LOCAL :834 and DIGEST_REQUESTS :788 are host-side choices (DESIGN.md 2.3,
   * gpx_digest_requests): none of them is engine configuration, so none is carried here) */
  int32_t log_backpressure;        /* 1: a call that could overwrite log bytes not yet released by gpx_log_release is
                                    * refused with GPX_EAGAIN (log-then-message, AbstractPaxosLogger.java:691-716: the
                                    * journal must be drained before a ring position is reused); 0 (default): the ring
                                    * overwrites the oldest bytes */
  int32_t reserved[7];
} gpx_config;

typedef struct gpx_counters {
  uint64_t accepts_handled, accepts_acked, accepts_nacked, accepts_logged, accepts_dropped;
  uint64_t replies_handled, replies_ignored, preempted, coordinators_resigned;
  uint64_t decisions_made, decisions_handled, decisions_dropped, placeholders;
  uint64_t executed, stops_executed, checkpoints_due;
  uint64_t proposals, requests_batched, requests_rejected;
  uint64_t window_overflow, kernel_launches;
  uint64_t reserved[7];
} gpx_counters;

typedef struct gpx_engine gpx_engine;

/* ---- lifecycle ---------------------------------------------------------------- */
void gpx_config_defaults(gpx_config* cfg);
/* parse the gigapaxos.properties keys the engine consumes; unknown keys ignored */
int gpx_config_from_properties(const char* path, gpx_config* cfg);
int gpx_engine_create(const gpx_config* cfg, gpx_engine** out);
void gpx_engine_destroy(gpx_engine* e);
const char* gpx_last_error(void);
const char* gpx_build_info(void); /* "gpx CUDA engine: ... sm_90a ..." or "oracle" */

/* ---- groups -------------------------------------------------------------------- */
int gpx_create_groups(gpx_engine* e, uint32_t n, const gpx_group_desc* descs);
int gpx_destroy_groups(gpx_engine* e, uint32_t n, const uint32_t* gids);
int gpx_dump_rows(gpx_engine* e, uint32_t n, const uint32_t* gids, uint32_t lane, gpx_row* out);
int gpx_load_rows(gpx_engine* e, uint32_t n, const gpx_row* rows);
int gpx_patch(gpx_engine* e, uint32_t n, const gpx_patch_rec* patches);

/* ---- data path: host buffers in, host buffers out (H2D and D2H inside) ---------- */

/* RequestBatcher + PCS.propose.  reqs must be grouped by gid (per-group FIFO order
 * preserved).  out_accepts capacity n; out_blob capacity blob_cap bytes (>= payload_bytes
 * + 16*n); status[n] receives the slot or a GPX_RS_* code.  Slots are Java ints and wrap
 * (2^31 - 1 is followed by -2^31, then ..., -1, 0, 1), so a slot may equal a GPX_RS_* code or 0:
 * the sign does not tell them apart.  The ACCEPTs do (gpx_propose: one per slot, in request order
 * of the slot's first request), as do the EXEC records and, in compact mode, the summary's
 * lane_mask. */
int gpx_propose(gpx_engine* e, uint32_t n, const gpx_request_rec* reqs, const uint8_t* payload,
                uint64_t payload_bytes, gpx_accept_rec* out_accepts, uint32_t* n_accepts,
                uint8_t* out_blob, uint64_t blob_cap, uint64_t* blob_bytes, int32_t* status);

/* handleAccept at every local lane in rec.dst_mask.  accepts must be grouped by gid.
 * out_replies[n * n_lanes] (index i*n_lanes+lane, GPX_F_VOID where not addressed/dropped).
 * out_extra_exec (cap extra_cap) receives EXEC records released by reconstructDecision. */
int gpx_handle_accepts(gpx_engine* e, uint32_t n, const gpx_accept_rec* accepts,
                       const uint8_t* blob, uint64_t blob_bytes, gpx_accept_reply_rec* out_replies,
                       gpx_exec_rec* out_extra_exec, uint32_t extra_cap, uint32_t* n_extra);

/* handleAcceptReply at the destination lane of each reply; replies grouped by gid.
 * out_decisions capacity n. */
int gpx_handle_accept_replies(gpx_engine* e, uint32_t n, const gpx_accept_reply_rec* replies,
                              gpx_decision_rec* out_decisions, uint32_t* n_decisions);

/* handleBatchedCommit per slot at every local lane in rec.dst_mask; grouped by gid.
 * out_exec[n * n_lanes] primary EXEC record per (decision, lane) (VOID if none);
 * further in-order executions released by the same decision go to out_extra_exec. */
int gpx_handle_decisions(gpx_engine* e, uint32_t n, const gpx_decision_rec* decisions,
                         gpx_exec_rec* out_exec, gpx_exec_rec* out_extra_exec, uint32_t extra_cap,
                         uint32_t* n_extra);

/* Fused co-located path (PaxosManager.sendOrLoopback :2116-2128): per ACCEPT, in batch order,
 * handleAccept at every addressed lane; replies addressed to a usable LOCAL coordinator lane are
 * handled at once (the others are returned in out_replies, VOID where consumed); a resulting
 * DECISION (out_decisions[n], VOID where none) is handled at every local lane before the next
 * ACCEPT.  out_exec[n * n_lanes].  EXEC records of one call are applied per group in slot order
 * (primary and extra records interleave). */
int gpx_handle_accepts_fused(gpx_engine* e, uint32_t n, const gpx_accept_rec* accepts, const uint8_t* blob,
                             uint64_t blob_bytes, gpx_accept_reply_rec* out_replies,
                             gpx_decision_rec* out_decisions, gpx_exec_rec* out_exec,
                             gpx_exec_rec* out_extra_exec, uint32_t extra_cap, uint32_t* n_extra);

/* ---- phase 1a at the acceptors ------------------------------------------------------------------
 * PREPARE = a gpx_pvalue_hdr whose `slot` is PreparePacket.firstUndecidedSlot and whose ballot is the would-be
 * coordinator's.  gpx_handle_prepares runs PISM.handlePrepare :896-955 / PaxosAcceptor.handlePrepare :239-275
 * at every addressed local lane: a stopped instance drops it; a higher ballot is adopted; the reply carries the
 * acceptor's ballot after that (NACK if it is higher than the PREPARE's), firstSlot =
 * getMaxGCSlotFirstUndecidedSlot :277-282 and -- unless NACKing -- the accepted pvalues with slot >=
 * firstUndecidedSlot in slot order (pruneAcceptedProposals :285-297).  When the ballot was raised the PREPARE is
 * appended to the lane's log ring before the reply is visible (LogMessagingTask, :940-944; segment type
 * GPX_F_PREPARE) and the reply is flagged GPX_F_LOGGED.  The coordinator side (PCS.isPrepareAcceptedByMajority,
 * combinePValuesOntoProposals) stays on the host and installs its result with gpx_patch. */
typedef struct gpx_accepted_pvalue { /* one accepted pvalue of a PREPARE_REPLY, 32 B (the accepted-window entry) */
  int32_t slot;
  int32_t bnum;
  int32_t bcoord;
  uint32_t frame_ref;   /* offset / 16 of the request blob inside this acceptor's log ring (its log position modulo
                         * log_ring_bytes: the blob is the latest such position before the ring head) */
  int64_t req_id;
  uint32_t payload_len;
  uint32_t flags;       /* bit1 STOP, bits 16.. nreq */
} gpx_accepted_pvalue;
typedef struct gpx_prepare_reply_rec { /* PrepareReplyPacket, 32 + 32 * GPX_MAX_WINDOW bytes */
  uint32_t gid;
  int32_t first_slot;   /* PrepareReplyPacket.firstSlot */
  int32_t bnum;         /* acceptor's ballot after handling the PREPARE */
  int32_t bcoord;
  uint32_t who;         /* GPX_WHO(acceptor idx, preparer idx, GPX_F_VOID | GPX_F_NACK | GPX_F_LOGGED | GPX_F_FROM_LOG) */
  uint32_t n_accepted;
  int64_t reserved;
  gpx_accepted_pvalue accepted[GPX_MAX_WINDOW];
} gpx_prepare_reply_rec;
/* out_replies[n * n_lanes] */
int gpx_handle_prepares(gpx_engine* e, uint32_t n, const gpx_pvalue_hdr* prepares, gpx_prepare_reply_rec* out_replies);

/* ---- phase 1b at the would-be coordinator -------------------------------------------------------
 * gpx_handle_prepare_replies runs, for a batch of elections (one candidate coordinator of one group each: the mass
 * fail-over after a node is lost is many groups electing at once), what PISM.handlePrepareReply :1017-1068 does per
 * PREPARE_REPLY and what follows a majority:
 *   PaxosCoordinator.getPreActivesIfPreempted :313-318 / PCS.isPreemptable :271-278   a reply with a higher ballot
 *       ends the election (GPX_EL_PREEMPTED; nothing is installed);
 *   PCS.canIgnorePrepareReply :287-316   lower ballot, not a member, already heard: ignored;
 *   PCS.isPrepareAcceptedByMajority :326-391   recordSlotNumber(PrepareReplyPacket) :786-807 with
 *       PrepareReplyPacket.getMinSlot :151-164 (= min(firstSlot, the accepted slots), wrap-aware), the pvalue of the
 *       highest ballot per slot is carried over, WaitforUtility majority;
 *   PCS.combinePValuesOntoProposals :393-444   the slots getMaxMinCarryoverSlot :921 .. getMaxPValueSlot :903 become
 *       the new coordinator's first proposals, carried-over pvalue or no-op (makeNoopPValue :886-897);
 *   PCS.processStop :478-554   every proposal carries the new ballot there (ProposalStateAtCoordinator's constructor
 *       :153-157 re-stamps it), so its two conversion branches cannot be taken; a regular request behind a STOP is the
 *       reference's `assert(false)` and is reported as GPX_ELF_STOP_ORDER; when a STOP was carried over and the last
 *       proposal is not a STOP, a fresh STOP is proposed behind it (:538-542);
 *   PCS.setCoordinatorActive :577-587   the coordinator is installed ACTIVE at `lane` with the recorded
 *       nodeSlotNumbers and nextProposalSlotNumber = the first slot of the plan; coordinators of a lower ballot at the
 *       other local lanes resign (PISM.handlePrepare would have removed them when the PREPARE arrived).
 * The plan is returned, not proposed: spawnCommandersForProposals :556-575 is the caller re-proposing plan[0..n_plan)
 * in order through gpx_propose / gpx_round (the request bodies of a carried-over pvalue are in the log ring of the
 * acceptor that reported it: reply index src_reply, position frame_ref * 16).  The engine keeps no pre-active
 * proposals (a request that finds a pre-active coordinator gets GPX_RS_PREACTIVE and waits at the host), so
 * combinePValuesOntoProposals' preActives and reproposePreemptedProposals :460-468 have nothing to do here.
 *
 * A PREPARE_REPLY longer than GPX_MAX_WINDOW pvalues (accepts added from the journal, GPX_F_FROM_LOG) is given as
 * consecutive records of the same acceptor, all but the last flagged GPX_F_MORE in `who`.
 * Device rules (as for the slot window): more than GPX_MAX_CARRY distinct carried-over slots, or a plan range of more
 * than GPX_MAX_PLAN slots, gives GPX_EL_OVERFLOW and installs nothing -- the candidate is too far behind and syncs
 * first (PISM.syncLongDecisionGaps).  At most one election per gid per call (GPX_EINVAL otherwise). */
#define GPX_F_MORE 0x0800u /* prepare reply record: the same PREPARE_REPLY continues in the next record */
#define GPX_MAX_CARRY 32
#define GPX_MAX_PLAN 16
enum {
  GPX_EL_WAITING = 0,   /* no majority among the replies given */
  GPX_EL_MAJORITY = 1,  /* elected and installed */
  GPX_EL_PREEMPTED = 2, /* a reply carried a higher ballot */
  GPX_EL_DROPPED = 3,   /* no live instance at that lane / stopped / lane not a member (PISM :456-460) */
  GPX_EL_OVERFLOW = 4
};
enum {
  GPX_CO_NOOP = 0,     /* RequestPacket(0, NO_OP, false), entry replica = the new coordinator */
  GPX_CO_PVALUE = 1,   /* the carried-over pvalue's request(s), re-proposed under the new ballot */
  GPX_CO_STOP_NEW = 2  /* RequestPacket(0, STOP, true) :541 */
};
#define GPX_ELF_STOP_ORDER 1u /* a regular request lies behind a STOP in the plan: PCS.processStop's assert(false) */
typedef struct gpx_election_rec { /* one pre-active coordinator (PISM.checkRunForCoordinator :2090-2150), 32 B */
  uint32_t gid;
  uint32_t lane;        /* local lane of the candidate */
  int32_t bnum;         /* the ballot it sent its PREPARE with */
  int32_t bcoord;
  int32_t slot;         /* PCS ctor's nextProposalSlotNumber = paxosState.getSlot() (the PREPARE's firstUndecidedSlot) */
  uint32_t first_reply; /* replies[first_reply .. first_reply + n_replies) are handled in this order */
  uint32_t n_replies;
  uint32_t reserved;
} gpx_election_rec;
typedef struct gpx_carryover { /* one proposal of the view change, 48 B */
  int32_t slot;
  uint32_t kind;        /* GPX_CO_* */
  uint32_t src_reply;   /* GPX_CO_PVALUE: index into replies[] of the record that carried it */
  uint32_t reserved;
  gpx_accepted_pvalue pv; /* GPX_CO_PVALUE: as reported (its own, lower, ballot) */
} gpx_carryover;
typedef struct gpx_election_out { /* 16 + 64 + 17 * 48 = 896 B */
  uint32_t gid;
  int32_t verdict;      /* GPX_EL_* */
  int32_t next_slot;    /* GPX_EL_MAJORITY: the installed nextProposalSlotNumber (plan[0].slot when n_plan > 0) */
  uint16_t n_plan;
  uint16_t flags;       /* GPX_ELF_* */
  int32_t node_slots[GPX_MAX_GROUP_SIZE]; /* nodeSlotNumbers as recorded (-1 = not heard) */
  gpx_carryover plan[GPX_MAX_PLAN + 1];
} gpx_election_out;
/* replies: host array of n_reply_recs records; out[n] */
int gpx_handle_prepare_replies(gpx_engine* e, uint32_t n, const gpx_election_rec* elections, uint32_t n_reply_recs,
                               const gpx_prepare_reply_rec* replies, gpx_election_out* out);

/* One full round for co-located replicas.  gpx_round: RequestBatcher + propose, then the fused
 * accept -> tally -> commit per ACCEPT with replies, decisions and rows kept in registers.
 * gpx_round_phases: the same round phase by phase (all ACCEPTs, then all replies, then all
 * DECISIONs), inter-replica records going through HBM.  Host request buffers in, EXEC records out
 * (out_exec[*n_exec_slots], extras appended to out_extra_exec). */
int gpx_round(gpx_engine* e, uint32_t n, const gpx_request_rec* reqs, const uint8_t* payload,
              uint64_t payload_bytes, int32_t* status, gpx_exec_rec* out_exec, uint32_t* n_exec_slots,
              gpx_exec_rec* out_extra_exec, uint32_t extra_cap, uint32_t* n_extra);
int gpx_round_phases(gpx_engine* e, uint32_t n, const gpx_request_rec* reqs, const uint8_t* payload,
                     uint64_t payload_bytes, int32_t* status, gpx_exec_rec* out_exec, uint32_t* n_exec_slots,
                     gpx_exec_rec* out_extra_exec, uint32_t extra_cap, uint32_t* n_extra);

/* Pipelined form of gpx_round.  The reference's hot path is a pipeline of threads (RequestBatcher ->
 * PISM -> PaxosPacketBatcher / AbstractPaxosLogger.BatchedLogger -> Messenger): a batch is being collected
 * while the previous one is logged and the one before is executed.  gpx_round_submit enqueues the
 * host->device copy of a batch, the round kernels and the device->host copy of its results on three
 * streams and returns at once; up to GPX_PIPE_DEPTH rounds may be in flight, rounds execute in submission
 * order.  All host buffers of the io block must stay valid (and should be page-locked for the copies to
 * overlap) until gpx_round_wait(ticket) returns.
 *
 * Output modes:
 *   full (flags = 0)       status[n], exec[n * n_lanes] as gpx_round.
 *   GPX_ROUND_COMPACT      sum[n]: one 8-byte summary per REQUEST index.  lane_mask != 0: every lane in the
 *                          mask executed exactly this request at `slot`, as its next in-order execution
 *                          (flags: GPX_F_CKPT if PISM.shouldCheckpoint :2037 holds) -- the host runs
 *                          Replicable.execute from its own copy of the request.  lane_mask == 0: `slot` is
 *                          the request's status (slot number or GPX_RS_* code) and every execution it caused
 *                          is a full record in the extra queue.  EXEC records of one call are applied per
 *                          (lane, group) in slot order.
 *   GPX_ROUND_PACKED_REQS  (input) `reqs` holds n gpx_request_packed (16 B) instead of gpx_request_rec (32 B):
 *                          the payloads lie back to back in request order (payload_off = running sum of
 *                          payload_len), entry_node = the node of the entry lane, client = the request
 *                          index.  Halves the host->device bytes of a batch; the engine expands the records
 *                          on the device (k_unpack: block sums, scan, expand). */
#define GPX_PIPE_DEPTH 4
#define GPX_ROUND_COMPACT 1u
#define GPX_ROUND_PACKED_REQS 2u
typedef struct gpx_request_packed {
  uint32_t gid;
  uint16_t payload_len;
  uint16_t flags;  /* as gpx_request_rec.flags: bit0 GPX_F_STOP, bits 8..11 entry lane */
  int64_t req_id;
} gpx_request_packed;
typedef struct gpx_exec_sum {
  int32_t slot;       /* decided slot (lane_mask != 0) or the request's status */
  uint8_t lane_mask;  /* lanes that executed the request in order */
  uint8_t flags;      /* GPX_F_CKPT */
  uint16_t nreq;      /* requests executed with it (1) */
} gpx_exec_sum;
typedef struct gpx_round_io {
  uint32_t n;
  uint32_t flags;              /* GPX_ROUND_COMPACT | GPX_ROUND_PACKED_REQS */
  const gpx_request_rec* reqs; /* [n] host (gpx_request_packed[n] with GPX_ROUND_PACKED_REQS) */
  const uint8_t* payload;      /* host */
  uint64_t payload_bytes;
  int32_t* status;             /* [n] out, full mode */
  gpx_exec_rec* exec;          /* [n * n_lanes] out, full mode */
  gpx_exec_sum* sum;           /* [n] out, compact mode */
  gpx_exec_rec* extra;         /* [extra_cap] out: further executions (filled by gpx_round_wait; *n_extra >
                                * extra_cap = truncated.  compact mode needs up to n * n_lanes + the full mode's) */
  uint32_t extra_cap;
} gpx_round_io;
int gpx_round_submit(gpx_engine* e, const gpx_round_io* io, uint64_t* ticket);
/* blocks until round `ticket` is complete; rounds must be waited for in submission order */
int gpx_round_wait(gpx_engine* e, uint64_t ticket, uint32_t* n_exec_slots, uint32_t* n_extra);

/* Digest path (DIGEST_REQUESTS, paxospackets/RequestPacket.java:1414-1430, AcceptPacket.digest :162-170):
 * MD5 of every request's requestValue, 16 bytes each -- the digest a coordinator puts into an ACCEPT in
 * place of the request body and an acceptor checks against the body it received by broadcast
 * (paxosutil/PendingDigests.java:82-145, host side). */
int gpx_digest_requests(gpx_engine* e, uint32_t n, const gpx_request_rec* reqs, const uint8_t* payload,
                        uint64_t payload_bytes, uint8_t* out_digests);

/* ---- log ring ------------------------------------------------------------------- */
/* copy ring bytes [from, min(head, from+cap)) of `lane` into dst; *head receives the ring head */
int gpx_log_read(gpx_engine* e, uint32_t lane, uint64_t from, void* dst, uint64_t cap,
                 uint64_t* n_copied, uint64_t* head);

/* Drain without stopping the rounds (AbstractPaxosLogger.BatchedLogger :691-716 is a thread beside the protocol
 * threads; SQLPaxosLogger.journal :965-1036 / Journaler.appendToLogFile :814-826 append to the journal file).
 * gpx_log_drain_async enqueues, on the engine's own drain stream and behind the work already enqueued on
 * `after_stream` (a cudaStream_t; NULL = the engine's stream), the copy of the next undrained ring bytes of `lane`
 * -- [*from, *from + *n_bytes), at most cap, in ring order -- into dst (host memory; page-locked to overlap) and
 * returns at once.  The host tracks the ring heads itself (every logging call has a host-known size), so no device
 * read is involved.  gpx_log_drain_wait blocks until the enqueued copies are done; gpx_log_release(lane, upto) tells
 * the engine that everything before `upto` is durable elsewhere: with gpx_config.log_backpressure set, a call
 * that would overwrite unreleased bytes is refused with GPX_EAGAIN before it does anything. */
int gpx_log_drain_async(gpx_engine* e, uint32_t lane, void* dst, uint64_t cap, uint64_t* from, uint64_t* n_bytes,
                        void* after_stream);
int gpx_log_drain_wait(gpx_engine* e);
int gpx_log_drain_skip(gpx_engine* e); /* drop the backlog: drain cursor and tail <- current heads */
int gpx_log_release(gpx_engine* e, uint32_t lane, uint64_t upto);

/* ---- finding logged pvalues: the journal's index as a scan ---------------------------------------------------------
 * A replica that answers a SYNC_DECISIONS_REQUEST (PISM.handleSyncDecisionsPacket :2426-2510) or a PREPARE from a
 * lagging node (PISM.handlePrepare :900-955 with GET_ACCEPTED_PVALUES_FROM_DISK) needs decisions / accepts that have
 * left its memory: AbstractPaxosLogger.getLoggedDecisions :582 / getLoggedAccepts :568, which with journaling are
 * SQLPaxosLogger.getLoggedFromMessageLog :3674-3756 -- look the (paxosID, slot range) up in the per-group
 * paxosutil/LogIndex (:213-248), read those frames back from the journal files, and keep per slot the entry logged
 * LAST (`accepts.put(packet.slot, packet)` :3746 in log order).  The engine keeps no index on the hot path; the log ring
 * is in HBM, so the lookup is a scan of it: one thread walks the segment headers from `from` (a segment boundary:
 * 0 while the ring has not wrapped, else a position handed out by gpx_log_drain_async / gpx_log_release) to the head,
 * one thread per logged image matches (gid, slot) against the batch of wants (sorted by gid, one want per gid, at
 * most GPX_LOG_SPAN slots each), the LAST logged DECISION and ACCEPT image per wanted slot win.
 * out[i * GPX_LOG_SPAN + k] answers slot wants[i].min_slot + k: the two images (flags GPX_F_VOID where there is none;
 * accept.payload_off is relative to its segment's payload area as in the ring) and the absolute ring position of the
 * accept's request blob (gpx_log_read(lane, blob_pos, dst, accept.payload_len, ...)).  getActualDecisions :2539-2583
 * (a meta decision gets its value from the logged accept of the slot) is the caller joining the two. */
#define GPX_LOG_SPAN 16
typedef struct gpx_log_want { /* 16 B */
  uint32_t gid;
  int32_t min_slot;
  uint32_t n_slots;  /* <= GPX_LOG_SPAN */
  uint32_t reserved;
} gpx_log_want;
typedef struct gpx_log_hit { /* 96 B */
  gpx_decision_rec decision;
  gpx_accept_rec accept;
  uint64_t blob_pos;
  uint64_t reserved;
} gpx_log_hit;
int gpx_log_find(gpx_engine* e, uint32_t lane, uint64_t from, uint32_t n, const gpx_log_want* wants, gpx_log_hit* out);

/* ---- journal frames on the device: a drained range of the ring as Journaler bytes ------------------------------------
 * SQLPaxosLogger.journal :965-1036 appends each logged packet to the journal file as {int32 BE length}{packet}, the
 * packet as SQLPaxosLogger.toBytes :1084-1098 writes it: an ACCEPT byteified (AcceptPacket.toBytes), a DECISION or a
 * PREPARE as the JSON string of the packet.  gpx_log_frame_device writes those frames for a range of one lane's ring in
 * HBM, ready for one copy to the host and one write to the file.
 *
 * The ring does not hold two RequestPacket fields a frame needs, entryReplica and entryTime; the caller passes them
 * per request in meta[n_meta] (device memory; PaxosManager.outstanding is the Java node's source), sorted ascending by
 * (gid, req_id) without duplicates, else GPX_EINVAL and nothing is written.  Names and versions come from
 * gpx_set_group_names' table.
 *
 *   Range     [*from, head) of `lane`, head being the engine's head of that lane at the call (as gpx_log_drain_async
 *             reads it, after the calls that log are enqueued; a call on another stream must be ordered before this
 *             one).  *from is a segment boundary: 0 before the ring has wrapped, else a position this call or
 *             gpx_log_drain_async handed out.  Bytes already overwritten are GPX_ERANGE and a segment header that does
 *             not parse is GPX_EINVAL, as in gpx_log_find.  An empty range returns GPX_OK at once with no frame.
 *   Frames    out[*out_bytes] receives, segment by segment in ring order and image by image, one frame per image
 *             that is not VOID, exactly as journal.LogDrainer appends them for the same range:
 *               ACCEPT (48-byte image)   the AcceptPacket bytes of gpx_wire_encode_accept: recovery 0, median_cp and
 *                 sender from the image, every RequestPacket field the ring does not hold at wire.Request's default
 *                 (no client or listen address, forwardCount 0, no digest, no response).  nreq <= 1: the request is
 *                 the image's req_id, STOP flag and blob.  nreq > 1: the blob's gpx_batch_ent list, the first entry
 *                 the outer request (entryReplica and entryTime of the image's req_id), the others its `batched`
 *                 REQUEST packets, each with its own req_id, STOP bit and table entry.
 *               DECISION (32-byte image, no GPX_F_PREPARE)   journal.decision_json:
 *                 {"type":90,"PT":6,"ID","V","B","GC_S","S","QID","ET","E"}, then "STOP":true only with GPX_F_STOP.
 *               PREPARE (GPX_F_PREPARE)   journal.prepare_json: {"type":90,"PT":2,"ID","V","B","PREP_MIN"}; it
 *                 needs no table entry.
 *             The paxosID is escaped as json.dumps with ensure_ascii escapes it (gpx_wire_encode_json_device's rule).
 *             *n_frames receives the number of frames.
 *   Misses    an image whose gid has no name, or one of whose requests is not in meta, gets no frame.  Then no frame
 *             at all is written, *from is unchanged, missing[*n_missing] lists one gpx_journal_miss per request the
 *             table lacks (req_id -1 once for an image whose gid has no name), in image order, and the call returns
 *             GPX_ENOENT.  The caller adds those requests to meta and calls again, so the order of frames is never
 *             broken.
 *   Sizes     *out_bytes, *n_frames and *n_missing are HOST pointers, capacities in / sizes out.  GPX_ERANGE reports the
 *             sizes and writes nothing: the frames' when a frame output is too small, or the misses' (the frame sizes
 *             0) when missing is.  Frames beyond 4 GiB in one call are GPX_ERANGE.
 *   Success   *from becomes head, and the lane's drain position moves up to it, so that gpx_log_release(lane, *from)
 *             is accepted; the caller releases once the frames are durable.
 * meta, out and missing are device pointers.  Stream-ordered on `stream` (NULL = the engine's stream), with the wire
 * calls' scratch and their ordering between streams; one synchronisation reads the totals (and, as in
 * gpx_log_drain_async, one more when a call of unknown log size left the engine's head to be read back). */
typedef struct gpx_journal_req { /* 24 B */
  uint32_t gid;
  int32_t entry_node; /* RequestPacket.entryReplica */
  int64_t req_id;
  int64_t entry_time; /* RequestPacket.entryTime, ms */
} gpx_journal_req;
typedef struct gpx_journal_miss { /* 16 B: a request the call could not frame */
  uint32_t gid;
  uint32_t kind;  /* GPX_F_ACCEPT, GPX_F_DECISION or GPX_F_PREPARE: the image that needs it */
  int64_t req_id; /* the request that is missing, or -1 when the gid has no name */
} gpx_journal_miss;
int gpx_log_frame_device(gpx_engine* e, uint32_t lane, uint64_t* from, const gpx_journal_req* meta, uint32_t n_meta,
                         uint8_t* out, uint64_t* out_bytes, uint32_t* n_frames, gpx_journal_miss* missing,
                         uint32_t* n_missing, void* stream);

/* ---- journal garbage collection on the device: compact journal files to the frames a checkpoint still needs ---------
 * SQLPaxosLogger.compactLogfile :3350-3450 rewrites each journal file to the frames LogIndex.isLogMsgNeeded :331-345
 * still wants, and deletes a file that keeps none.  gpx_journal_compact_device does that for k files of one lane's
 * journal at once, in HBM.
 *
 *   Input     bytes[n_bytes]: the k = n_files files concatenated in roll order, file f at [file_off[f], file_off[f+1])
 *             (file_off[0] = 0, ascending, file_off[k] = n_bytes); starts[n_frames]: the offset of every frame's
 *             {int32 BE length} in bytes, ascending (gpx_journal_index writes them).  gc_slot[n_gids]: the GC slot of
 *             each gid, n_gids >= max_groups; the caller computes gcSlot = (cp - accGC < 0) ? cp : accGC
 *             (SQLPaxosLogger.deleteOutdatedMessages :1480-1482) from the group's last checkpoint slot cp and the
 *             acceptor's acc_gc_slot (gpx_dump_rows), and -1 for a group without a checkpoint (LogIndex.java:41).
 *   Parse     each frame's packet is an ACCEPT (AcceptPacket bytes), a DECISION or a PREPARE (the JSON of
 *             journal.decision_json / prepare_json; other keys are allowed), read as (paxosID, version, slot, ballot);
 *             a PREPARE's slot is PREP_MIN.  (paxosID, version) resolves to a gid as the wire decoders resolve it:
 *             gpx_set_group_names' table, a live group at that version.
 *   Keep      an unresolved frame is kept (a paused group, a stale version or a name not in the table: the call
 *             cannot prove it unneeded).  A resolved one is dropped when slot - gc_slot[gid] <= 0 (int32 wrap
 *             arithmetic).  A resolved PREPARE above the gc slot is also dropped when an indexed frame of its group --
 *             a resolved frame of any type above the group's gc slot, in any of the k files -- has a higher ballot:
 *             bnum - bnum' > 0, or equal bnums and bcoord - bcoord' > 0, tested entry by entry as the reference
 *             does.  Every other frame is kept.
 *             Deliberate divergence: SQLPaxosLogger.getSlot :492-496 returns an ACCEPT's or DECISION's ballot number
 *             as its slot, so compactLogfile compares the ballot number with the GC slot.  The index built at journal
 *             time uses the pvalue's slot (MessageLogDiskMap.add :412), and so does this call: an ACCEPT above the GC
 *             slot whose ballot number is at or below it is kept.
 *   Files     files[f] receives the file's gpx_journal_file.  A file whose last frame does not end at the file's end
 *             (a torn tail: gpx_journal_index stops there) is GPX_JGC_TORN and left as it is, as is the last file
 *             when last_readonly is set (GPX_JGC_UNCHANGED); their frames still count as indexed entries.  Of the
 *             others, a file that keeps every frame is GPX_JGC_UNCHANGED, one that keeps none GPX_JGC_EMPTY (the
 *             caller deletes it), any other GPX_JGC_COMPACTED: its kept frames, unchanged and in order, are at
 *             out[out_off, out_off + out_bytes).  Only compacted files have bytes in out, in file order.
 *   Errors    a frame whose length runs past its file or disagrees with the next start, the first frame of a file
 *             not at the file's start, or a packet that does not parse: no file record and no byte is written,
 *             bad[*n_bad] lists the frame indices in ascending order, and the call returns GPX_EINVAL.  A file_off
 *             that is not ascending from 0 to n_bytes is GPX_EINVAL with no list.
 *   Sizes     *out_bytes and *n_bad are HOST pointers, capacities in / sizes out; GPX_ERANGE reports the sizes and
 *             writes nothing (out_bytes 0 when bad is the one too small).  n_bytes above 4 GiB - 1 is GPX_ERANGE.
 * bytes, file_off, starts, gc_slot, out, files and bad are device pointers.  Stream-ordered on `stream` (NULL = the
 * engine's stream), with the wire calls' scratch and ordering between streams; one synchronisation reads the totals.
 * The call reads no group state but the groups' liveness. */
enum { GPX_JGC_UNCHANGED = 0, GPX_JGC_COMPACTED = 1, GPX_JGC_EMPTY = 2, GPX_JGC_TORN = 3 };
typedef struct gpx_journal_file { /* 24 B */
  uint32_t status;     /* GPX_JGC_* */
  uint32_t kept;       /* frames the file holds after the call */
  uint32_t dropped;    /* frames removed */
  uint32_t unresolved; /* of the frames, those whose name did not resolve (all kept) */
  uint32_t out_off;    /* GPX_JGC_COMPACTED: the file's bytes in out */
  uint32_t out_bytes;
} gpx_journal_file;
int gpx_journal_compact_device(gpx_engine* e, const uint8_t* bytes, uint64_t n_bytes, const uint32_t* file_off,
                               uint32_t n_files, const uint32_t* starts, uint32_t n_frames, const int32_t* gc_slot,
                               uint32_t n_gids, uint32_t last_readonly, uint8_t* out, uint64_t* out_bytes,
                               gpx_journal_file* files, uint32_t* bad, uint32_t* n_bad, void* stream);
/* The frame starts of a journal file in host memory, as journal.read_journal walks it: from offset 0, a frame is
 * {int32 BE length}{length bytes}, and the walk stops at a negative length or at a frame that runs past n_bytes (a
 * torn tail).  starts[k] = base + the offset of frame k, for up to cap frames; *n_frames receives the count and *end
 * the offset where the walk stopped (n_bytes unless the tail is torn).  GPX_ERANGE when the count exceeds cap (the
 * first cap are written), GPX_EINVAL on a null pointer or when base + n_bytes passes 4 GiB.  No engine is involved:
 * the walk is a chain of dependent reads over bytes the caller has just read from the file. */
int gpx_journal_index(const uint8_t* buf, uint64_t n_bytes, uint32_t base, uint32_t* starts, uint32_t cap,
                      uint32_t* n_frames, uint64_t* end);

/* Request bodies for a batch of gpx_log_find hits (blob_pos) or of carried-over pvalues (the latest log position
 * before the head that is congruent to frame_ref * 16 modulo log_ring_bytes) in ONE device->host copy:
 * ranges[i] = {absolute log position, length, offset in dst (a multiple of 16)}; range i lands at
 * dst + dst_off rounded up to whole 16-byte chunks (the ring's payload areas are padded to 16).  The journal analogue is
 * SQLPaxosLogger.getJournaledMessage(FileOffsetLength[]) :3712, which reads the indexed frames back in one pass. */
typedef struct gpx_log_range { /* 16 B */
  uint64_t pos;
  uint32_t len;
  uint32_t dst_off;
} gpx_log_range;
int gpx_log_gather(gpx_engine* e, uint32_t lane, uint32_t n, const gpx_log_range* ranges, void* dst, uint64_t dst_bytes);

/* ---- introspection ---------------------------------------------------------------- */
int gpx_get_counters(gpx_engine* e, gpx_counters* out);
int gpx_reset_counters(gpx_engine* e);
/* slow-path list: per-group flag byte of one lane (bit0 window overflow: a record beyond the
 * in-flight window W was dropped; bit1 needs sync: a commit could not be resolved locally ->
 * host runs PISM.syncLongDecisionGaps :1550 / requestMissingDecisions) */
#define GPX_GF_OVERFLOW_BIT 1u
#define GPX_GF_NEEDS_SYNC_BIT 2u
/* computed on the fly: the lane is NOT caught up -- PaxosAcceptor.caughtUp :452-459 (committedRequests empty, and
 * acceptedProposals empty unless journaling serves accepted pvalues from disk) or PCS.caughtUp :758 (myProposals
 * empty) is false.  PISM.tryPause :2004-2035 pauses an instance only when this bit is clear on every lane. */
#define GPX_GF_NOT_CAUGHT_UP_BIT 4u
int gpx_get_group_flags(gpx_engine* e, uint32_t lane, uint32_t n, const uint32_t* gids, uint8_t* out);
/* ---- the slow-path list (SURVEY.md 8b) / the candidates of a sweep --------------------------------------------------
 * PaxosManager's sweeps walk ALL instances (syncAndDeactivate :2806-2900 iterates pinstances; the failure detector's
 * checkRunForCoordinator pass likewise) and test each one; with millions of groups resident the test belongs where the
 * state is.  gpx_select_groups returns the live groups of `lane` whose flag byte -- exactly what gpx_get_group_flags
 * reports: GPX_GF_OVERFLOW_BIT | GPX_GF_NEEDS_SYNC_BIT | GPX_GF_NOT_CAUGHT_UP_BIT -- satisfies
 * (flags & mask) == value and whose acceptor is ACTIVE: mask = value = GPX_GF_NEEDS_SYNC_BIT lists the groups to sync
 * (PISM.syncLongDecisionGaps :1550), mask = GPX_GF_NOT_CAUGHT_UP_BIT, value = 0 the pause candidates
 * (PISM.tryPause :2004).  out_gids[0 .. min(*n_found, cap)) in ascending order; *n_found is the number that matched
 * (when it exceeds cap, which `cap` of them were returned is unspecified: ask again with a larger buffer). */
int gpx_select_groups(gpx_engine* e, uint32_t lane, uint32_t mask, uint32_t value, uint32_t* out_gids, uint32_t cap,
                      uint32_t* n_found);

/* What a listed group is missing: PISM.requestMissingDecisions :2292-2320 at `lane` for a batch of groups --
 * PaxosAcceptor.getMaxCommittedSlot :425-438 (the highest committed slot held, slot - 1 when there is none or the acceptor
 * is stopped), getMissingCommittedSlots(sizeLimit) :405-423 (from the next slot to execute up to the highest committed one:
 * no commit there, or a value-less commit without its accept) -- [slot] itself when nothing else is missing (:2297-2298) --
 * and isMissingTooMuch :2367-2370 = shouldSync(maxCommittedSlot, too_much_gap) :2341-2361 in its default mode (the
 * reference passes getMaxSyncDecisionsGap()).  These are the fields of the SYNC_DECISIONS_REQUEST the host sends
 * (SyncDecisionsPacket); whom to ask (:2305-2312) stays with the host.  With the bounded window a commit further than W
 * slots ahead is not held (it was dropped and flagged NEEDS_SYNC), so at most W - 1 slots are listed.
 * n_missing == 0: stopped / no live instance -- no request (getMissingCommittedSlots returns null). */
typedef struct gpx_missing_rec { /* 48 B */
  uint32_t gid;
  int32_t slot;               /* paxosState.getSlot(): the next slot to execute */
  int32_t max_decision_slot;  /* getMaxCommittedSlot() */
  uint16_t n_missing;
  uint8_t missing_too_much;
  uint8_t flags;              /* the group's flag byte (GPX_GF_*) */
  int32_t missing[GPX_MAX_WINDOW];
} gpx_missing_rec;
int gpx_missing_decisions(gpx_engine* e, uint32_t lane, uint32_t n, const uint32_t* gids, int32_t size_limit,
                          int32_t too_much_gap, gpx_missing_rec* out);

/* The OVERFLOW / NEEDS_SYNC bits are sticky: they stay until the host has dealt with the group (caught it up by a sync or
 * a checkpoint transfer) and says so -- out of the slow-path list.  Clears `mask` (of those two bits) at `lane` for
 * every gid given. */
int gpx_clear_group_flags(gpx_engine* e, uint32_t lane, uint32_t n, const uint32_t* gids, uint32_t mask);

/* ---- batched pause: the deactivation sweep (PaxosManager.Deactivator :2951 -> syncAndDeactivate :2806-2900 ->
 * pause(Map, dequeue) :2327-2366, PAUSE_BATCH_SIZE PaxosConfig.java:715) as one launch.  For every gid of the batch,
 * PISM.tryPause :2004-2035 at every local lane that hosts a replica: the group is paused only if it is live, every such
 * acceptor is ACTIVE and every lane is caught up (GPX_GF_NOT_CAUGHT_UP_BIT clear).  Then out_rows[i * n_lanes + lane]
 * = the HotRestoreInfo field set of every lane (what gpx_dump_rows returns; the caller turns them into the pause
 * table's strings, SQLPaxosLogger.pause) and the gid is free as after gpx_destroy_groups (forceStop + softCrash
 * :2284-2300).  out_paused[i] = 1 / 0; a group that does not pause is not touched and its rows are not written.
 * No gid may appear twice (GPX_EINVAL).  Unpause (PaxosManager.unpause :2370, PISM.hotRestore :677-690) =
 * gpx_load_rows. */
int gpx_pause_groups(gpx_engine* e, uint32_t n, const uint32_t* gids, gpx_row* out_rows, uint8_t* out_paused);
/* `active.<name>=host:port` entries (PaxosConfig.getActives :156-170) of the last
 * gpx_config_from_properties call, as "name=host:port\n" lines */
int gpx_properties_actives(char* out, size_t cap);

/* ---- device-resident API (bench `value`, multi-GPU shards): all pointers are device
 * pointers owned by the caller, `stream` is a cudaStream_t ------------------------------ */
typedef struct gpx_dev_round_bufs {
  const gpx_request_rec* reqs; /* [n] device */
  const uint8_t* payload;      /* device */
  uint64_t payload_bytes;
  uint32_t n;
  int32_t* status;             /* [n] device */
  gpx_exec_rec* exec;          /* [n * n_lanes] device */
} gpx_dev_round_bufs;
int gpx_round_device(gpx_engine* e, const gpx_dev_round_bufs* b, void* stream);        /* fused */
/* Form of the fused round.  0 / 1 (default): k_round_slow -- the general code for runs that are not the plain in-order
 * case -- is launched from the device, as a tail launch, by the first team that leaves a run over: a round without
 * such runs is ONE kernel on the stream.  2: the host launches k_round_slow behind every k_round (tuning / fallback).
 * The in-order kernel is k_round_g (one thread per group) for n_lanes <= 3 and k_round (a team of n_lanes threads per
 * group) above that; 3 and 4 are 0 and 2 with k_round at every n_lanes, to time the two against each other and to test
 * that they compute the same round. */
int gpx_set_round_mode(gpx_engine* e, int mode);
int gpx_round_device_phases(gpx_engine* e, const gpx_dev_round_bufs* b, void* stream); /* phase by phase */
/* gpx_propose + gpx_handle_accepts_fused on device buffers: ACCEPTs compacted at the front (exec[k * n_lanes + lane]
 * belongs to the k-th ACCEPT of the batch; the count is gpx_counters.proposals' increment), no per-request holes in
 * the log segments -- the form for batches in which many requests share a slot (RequestBatcher.java:198-219) */
int gpx_round_device_compact(gpx_engine* e, const gpx_dev_round_bufs* b, void* stream);
/* ---- device-resident phase calls: replicas of a group in DIFFERENT engines (spread placement:
 * one engine per GPU hosts one node; ACCEPT / ACCEPT_REPLY / DECISION records travel between engines
 * over NVLink).  Everything is asynchronous on `stream`; all pointers are device pointers unless
 * noted.  `ctl` is a caller-owned device block the kernels count into (the caller zeroes it). ---- */
typedef struct gpx_dev_ctl {
  uint32_t n_accepts;   /* gpx_propose_device: ACCEPTs written */
  uint32_t n_decisions; /* gpx_replies_device: DECISIONs appended (accumulates over calls) */
  uint32_t n_extra;     /* EXEC records appended to the extra queue */
  uint32_t any_batched;
  uint64_t blob1_used;  /* bytes of constructed (batched) blobs behind the payload arena */
  uint32_t n_todo;
  uint32_t pad;
} gpx_dev_ctl;
/* RequestBatcher + PISM.handleProposal / PCS.propose: out_accepts[<= n] (grouped by gid, dst_mask = all
 * members), payload_off relative to [payload arena | engine-owned batched blobs] */
int gpx_propose_device(gpx_engine* e, const gpx_request_rec* reqs, const uint8_t* payload, uint64_t payload_bytes,
                       uint32_t n, int32_t* status, gpx_accept_rec* out_accepts, gpx_dev_ctl* ctl, void* stream);
/* PaxosPacketBatcher per-destination grouping + PaxosManager.send unicast split (:2098-2128): bucket the
 * records of one kind (GPX_F_ACCEPT, GPX_F_DECISION, 0 = ACCEPT_REPLY) by destination node.
 * dest_nodes[n_dest <= 8] (host) lists the nodes served, the local one included (loopback).
 * out_recs[n_dest][cap], out_counts[n_dest] (zeroed by the caller); ACCEPTs also re-pack their blobs:
 * out_blob[n_dest][blob_cap], out_blob_units[n_dest] = bytes / 16.  Records of a group stay adjacent
 * and ordered inside a bucket.  *dropped counts records without a served destination / over capacity. */
int gpx_route_device(gpx_engine* e, uint32_t kind, const void* recs, const uint32_t* n_ptr, uint32_t n_max,
                     const uint8_t* payload, uint64_t payload_bytes, uint32_t n_dest, const int32_t* dest_nodes,
                     void* out_recs, uint32_t cap, uint32_t* out_counts, uint8_t* out_blob, uint64_t blob_cap,
                     uint32_t* out_blob_units, uint32_t* dropped, void* stream);
/* PISM.handleAccept at the local lanes for n received ACCEPTs = n_chunks concatenated buckets (chunk c ends
 * at record chunk_rec_end[c], its blob starts at chunk_blob_base[c] of `blob`; host arrays); payload_off of
 * the records is rebased in place.  out_replies[n * n_lanes]; executions released by
 * reconstructDecision go to out_extra[ctl->n_extra++]. */
int gpx_accepts_device(gpx_engine* e, gpx_accept_rec* recs, uint32_t n, const uint8_t* blob, uint64_t blob_bytes,
                       uint32_t n_chunks, const uint32_t* chunk_rec_end, const uint64_t* chunk_blob_base,
                       gpx_accept_reply_rec* out_replies, gpx_exec_rec* out_extra, uint32_t extra_cap,
                       gpx_dev_ctl* ctl, void* stream);
/* PaxosCoordinator.handleAcceptReply for n replies grouped by gid (one bucket of one acceptor at a time keeps
 * the replies of a group in one run); DECISIONs are appended at out_decisions[ctl->n_decisions++] */
int gpx_replies_device(gpx_engine* e, const gpx_accept_reply_rec* replies, uint32_t n,
                       gpx_decision_rec* out_decisions, gpx_dev_ctl* ctl, void* stream);
/* PISM.handleBatchedCommit + extractExecuteAndCheckpoint: out_exec[n * n_lanes], further executions in
 * out_extra[ctl->n_extra++].  (Received ACCEPT / DECISION records get their dst_mask -- a LOCAL lane mask --
 * rewritten in place to this engine's member lanes.) */
int gpx_decisions_device(gpx_engine* e, gpx_decision_rec* decisions, uint32_t n, gpx_exec_rec* out_exec,
                         gpx_exec_rec* out_extra, uint32_t extra_cap, gpx_dev_ctl* ctl, void* stream);

/* ---- SPREAD placement behind the C ABI (SURVEY.md 8e): the replicas of a group live in DIFFERENT engines -- one
 * single-lane engine per node, one node per GPU, replica j of a group on node (home + j) mod N
 * (PISM.roundRobinCoordinator :2251-2256) -- and the three inter-replica packet types of a round (ACCEPT,
 * ACCEPT_REPLY, DECISION; unicast fan-out paxosutil/PaxosMessenger.java:175-182, PaxosManager.send :2098-2128,
 * per-destination batching PaxosPacketBatcher.java:270-303) cross GPUs as fixed-capacity buckets whose record
 * count travels in-band: no host ever reads a count, a whole round is one asynchronous enqueue (optionally one
 * CUDA-graph launch) of  k_propose -> k_sp_route -> [exchange] -> k_sp_accept -> [exchange] -> k_sp_tally ->
 * [exchange] -> k_sp_commit.  The exchange is one ncclGroupStart / ncclSend + ncclRecv per peer / ncclGroupEnd per
 * packet type over NVLink (one process per GPU; libnccl.so.2 is loaded at run time), or plain device copies
 * when all nodes are engines of one process ("local" mode: tests on a single GPU).
 *
 * A Java PaxosManager would create one engine + one spread handle per GPU process, hand every batch of client
 * requests for the groups it coordinates to gpx_spread_round and apply the EXEC records it gets back; every
 * process of the spread group calls gpx_spread_round once per round (an empty batch still takes part in the
 * exchanges). */
#define GPX_SPREAD_MAX_NODES 8
#define GPX_SPREAD_GRAPH 1u /* capture a round into a CUDA graph per distinct io block and replay it */
#define GPX_SPREAD_P2P 2u   /* peer-memory transport: a node's send buckets ARE its peers' receive buckets (CUDA IPC between
                             * the per-GPU processes): k_sp_route / k_sp_accept / k_sp_tally store over NVLink, the exchange
                             * is a flag (k_sp_signal / k_sp_wait).  NCCL is then used once, to hand the IPC handles around */
typedef struct gpx_spread gpx_spread;
typedef struct gpx_spread_config {
  uint32_t n_nodes;                                         /* engines (nodes) of the spread group */
  int32_t node_ids[GPX_SPREAD_MAX_NODES];                   /* node id served by engine i (its lane 0) */
  uint32_t cap[GPX_SPREAD_MAX_NODES][GPX_SPREAD_MAX_NODES]; /* cap[s][d]: ACCEPTs node s may send node d in one round
                                                             * (>= groups s coordinates that d is a member of, times the
                                                             * slots a round may open per group); cap[s][s] is the
                                                             * loop-back bucket; 0 = the pair never exchanges.  The same
                                                             * matrix on every node. */
  uint32_t blob_per_rec; /* blob bytes a bucket reserves per record slot (multiple of 16): request bodies travel
                          * with their ACCEPT (AcceptPacket carries the RequestPacket, AcceptPacket.java:95-138) */
  uint32_t max_reqs;     /* requests one node submits per round (<= the engine's max_batch_recs) */
  uint32_t flags;        /* GPX_SPREAD_GRAPH | GPX_SPREAD_P2P */
  uint32_t reserved[8];
} gpx_spread_config;
/* what one node's buffers look like: byte offsets into its bucket arena, transfer sizes (0 = no transfer with that
 * peer), and the virtual index space of its receive side.  kind 0 = ACCEPT, 1 = ACCEPT_REPLY, 2 = DECISION.
 * Pure host arithmetic: send_bytes[k][d] of node s equals recv_bytes[k][s] of node d. */
typedef struct gpx_spread_plan {
  uint32_t n_nodes, rank;
  uint64_t send_off[3][GPX_SPREAD_MAX_NODES], send_bytes[3][GPX_SPREAD_MAX_NODES];
  uint64_t recv_off[3][GPX_SPREAD_MAX_NODES], recv_bytes[3][GPX_SPREAD_MAX_NODES];
  uint32_t vbase[GPX_SPREAD_MAX_NODES]; /* first virtual record index of the bucket received from node s */
  uint32_t vtotal;                      /* EXEC slots / log image slots per round at this node */
  uint64_t blob_off[GPX_SPREAD_MAX_NODES];
  uint64_t blob_vtotal;
  uint64_t arena_bytes;
} gpx_spread_plan;
int gpx_spread_plan_node(const gpx_spread_config* cfg, uint32_t rank, gpx_spread_plan* out);
/* per node and round: device pointers owned by the caller */
typedef struct gpx_spread_io {
  const gpx_request_rec* reqs; /* [n] requests for groups this node coordinates, grouped by gid (entry lane 0) */
  const uint8_t* payload;
  uint64_t payload_bytes;
  uint32_t n;
  uint32_t reserved;
  int32_t* status;    /* [n] */
  gpx_exec_rec* exec; /* [plan.vtotal]: EXEC record of the DECISION at that virtual index, VOID holes elsewhere */
  gpx_exec_rec* extra;
  uint32_t extra_cap;
  uint32_t reserved2;
  gpx_dev_ctl* ctl;   /* zeroed by the round; n_accepts / n_extra when it is done */
} gpx_spread_io;
/* 128-byte NCCL unique id (ncclGetUniqueId): made by one process, handed to the others by the host's own channel */
int gpx_spread_unique_id(void* out_id128);
/* one process per node: `e` is node `rank` of cfg->n_nodes; collective over the spread group (ncclCommInitRank) */
int gpx_spread_create_nccl(gpx_engine* e, const gpx_spread_config* cfg, uint32_t rank, const void* id128,
                           gpx_spread** out);
/* all cfg->n_nodes nodes are engines of this process (same device): the exchange is a set of device copies */
int gpx_spread_create_local(gpx_engine* const* engines, const gpx_spread_config* cfg, gpx_spread** out);
void gpx_spread_destroy(gpx_spread* sp);
/* one round, asynchronous on `stream`.  io[k] belongs to the k-th local node (NCCL mode: one; local mode: n_nodes) */
int gpx_spread_round(gpx_spread* sp, const gpx_spread_io* io, void* stream);
/* records k_sp_route could not place since creation (bucket too small / member node not in the spread group);
 * synchronises the device */
int gpx_spread_dropped(gpx_spread* sp, uint32_t local_index, uint32_t* out);

/* per-kernel CUDA-event timing of the last gpx_round_device calls (ms, accumulated) */
typedef struct gpx_kernel_times {
  double propose_ms, accept_ms, tally_ms, commit_ms;
  uint64_t launches;
} gpx_kernel_times;
int gpx_enable_kernel_timing(gpx_engine* e, int on);
int gpx_get_kernel_times(gpx_engine* e, gpx_kernel_times* out, int reset);

/* ---- phase-2 wire packets on the device: replicas of a group on other hosts ---------------------------------------
 * A group's replicas on other machines exchange ACCEPT, ACCEPT_REPLY and DECISION as the reference's bytes:
 * AcceptPacket, BatchedAcceptReply and BatchedCommit (layouts in gpx_wire.h).  These calls turn a batch of received
 * packets into engine records and the engine's reply / decision records into packets, on the device; gpx_wire_* in
 * gpx_wire.h is the host codec of one packet per call.
 *
 * Names.  A packet names its group by (paxosID, version) (PaxosPacket.java:459-476).  gpx_set_group_names gives gids
 * their paxosID (names[name_off[k] .. + name_len[k]), ISO-8859-1 bytes, at most GPX_WIRE_MAX_ID) and stores the
 * version the group was created or loaded with.  The first call allocates the name state: 128 B per gid, a 4-byte
 * version and slot per gid, and an open-addressing table of 8-byte cells (at least 2 per gid); an engine that never
 * calls it has none.  A name held by another live gid, the same name twice or the same gid twice in one call is
 * GPX_EINVAL and changes nothing.  gpx_destroy_groups, gpx_pause_groups (for the groups that pause), gpx_create_groups
 * and gpx_load_rows remove the names of the gids they touch: after a re-create or an unpause the caller sets the name
 * again. */
int gpx_set_group_names(gpx_engine* e, uint32_t n, const uint32_t* gids, const uint8_t* names, const uint32_t* name_off,
                        const uint32_t* name_len);

/* one packet in a byte arena: input of the decoders (gid ignored; node ignored except by
 * gpx_wire_decode_requests_device: the receiving node), output of the encoders, 16 B */
typedef struct gpx_wire_ref {
  uint32_t off;  /* byte offset in the arena */
  uint32_t len;
  uint32_t gid;  /* encoders: the packet's group */
  int32_t node;  /* encoders: the destination node id */
} gpx_wire_ref;

/* per-packet status of gpx_wire_decode_batch (never fatal, gpx.h conventions) */
enum {
  GPX_WS_OK = 0,
  GPX_WS_UNKNOWN_NAME = 1, /* no live gid has this paxosID: the host may unpause it (PaxosManager.getInstance), resubmit */
  GPX_WS_VERSION = 2,      /* version differs from the group's: dropped (PISM :441-447) */
  GPX_WS_MALFORMED = 3,    /* truncated, bad magic, idLen out of range, trailing bytes, negative length, a latched
                            * request with latched requests of its own, an acceptor or coordinator outside the group */
  GPX_WS_UNHANDLED = 4,    /* JSON packets and every type but ACCEPT / BATCHED_ACCEPT_REPLY / BATCHED_COMMIT: host */
  GPX_WS_NOT_LOCAL = 5     /* no local lane is addressed (ACCEPT / commit: none is a member; reply: the ballot's
                            * coordinator is not served by a local lane) */
};

/* Decode a batch of received packets.  bytes[0 .. n_bytes) is host memory, pkts[k] = {off, len} of packet k.
 * Outputs, each grouped by gid and, within a group, in packet order and then in the packet's slot order -- the order
 * gpx_handle_accepts, gpx_handle_accept_replies and gpx_handle_decisions require:
 *   accepts[*n_accepts]    one gpx_accept_rec per ACCEPT, dst_mask = the group's local lanes; the request body goes to
 *                          blob (payload_off into it, every body 16-byte aligned): the requestValue, or for a batched
 *                          RequestPacket nreq x gpx_batch_ent then the values (gpx_propose's form).  Entry-lane bits of
 *                          gpx_batch_ent.flags: the lane serving entryReplica, 0xf when it is not a local lane.
 *   replies[*n_replies]    one gpx_accept_reply_rec per slot of a BATCHED_ACCEPT_REPLY: who = (member index of the
 *                          acceptor, member index of the ballot's coordinator, 0); max_cp from the packet header.
 *   decisions[*n_decisions] one gpx_decision_rec per slot of a BATCHED_COMMIT (flags GPX_F_DECISION, req_id 0: the
 *                          value is the accept the acceptor holds).
 *   status[n]              GPX_WS_* per packet; only GPX_WS_OK packets produce records.
 * The four counts are in/out: capacities in, sizes out.  When an output is too small the call returns GPX_ERANGE,
 * writes no record and reports the sizes needed.  Without gpx_set_group_names every packet is GPX_WS_UNKNOWN_NAME
 * (or malformed / unhandled). */
int gpx_wire_decode_batch(gpx_engine* e, uint32_t n, const uint8_t* bytes, uint64_t n_bytes, const gpx_wire_ref* pkts,
                          int32_t* status, gpx_accept_rec* accepts, uint32_t* n_accepts, uint8_t* blob,
                          uint64_t* blob_bytes, gpx_accept_reply_rec* replies, uint32_t* n_replies,
                          gpx_decision_rec* decisions, uint32_t* n_decisions);

/* per-record outcome of the encoders */
enum {
  GPX_WE_SENT = 0,    /* in a packet */
  GPX_WE_VOID = 1,    /* a hole (GPX_F_VOID), or a group that is not live */
  GPX_WE_LOCAL = 2,   /* loop-back: reply to a local lane / decision of a group with no remote member (SHORT_CIRCUIT_LOCAL) */
  GPX_WE_NACK = 3,    /* not coalesced (PaxosPacketBatcher.allPositiveAcceptReplies :423-430): the host sends it alone */
  GPX_WE_NO_NAME = 4  /* the group has no name (gpx_set_group_names) */
};

/* Encode accept replies, in the layout gpx_handle_accepts returns (record i * n_lanes + lane), the way one
 * PaxosPacketBatcher per lane coalesces them: one BatchedAcceptReply per (lane, gid, ballot), its header taken from the
 * first reply (BatchedAcceptReply(AcceptReplyPacket) :53-58), slot -> requestID of every reply added
 * (addAcceptReply :179-184) and written in ascending slot order.  n = number of records (a multiple of n_lanes).
 * out[0 .. *out_bytes) receives the packets, refs[*n_refs] one {off, len, gid, node = the coordinator} per packet, in
 * (lane, gid) order; rstatus[n] GPX_WE_* per record.  *out_bytes and *n_refs are capacities in, sizes out;
 * GPX_ERANGE as for the decoder. */
int gpx_wire_encode_replies(gpx_engine* e, uint32_t n, const gpx_accept_reply_rec* replies, uint8_t* rstatus,
                            uint8_t* out, uint64_t* out_bytes, gpx_wire_ref* refs, uint32_t* n_refs);
/* Encode decisions, as gpx_handle_accept_replies returns them (any order): one BatchedCommit per (gid, ballot),
 * medianCheckpointedSlot the wrap-aware maximum (gpx_wire_fuse_commits), slots ascending, the group's member node ids
 * as its group list.  The packet is stored once and indexed once per member node that no local lane serves, in gid
 * order. */
int gpx_wire_encode_decisions(gpx_engine* e, uint32_t n, const gpx_decision_rec* decisions, uint8_t* rstatus,
                              uint8_t* out, uint64_t* out_bytes, gpx_wire_ref* refs, uint32_t* n_refs);

/* Device-buffer forms of the three calls above: a remote replica's packets go from bytes to records, through the
 * device phase calls (gpx_accepts_device, gpx_replies_device, gpx_decisions_device) and back to packets without
 * leaving HBM.  They are the implementation: the host-buffer forms stage their inputs on the device, run them into
 * engine-owned buffers and copy the outputs out.  The wire calls of one engine share its scratch, so a call on one
 * stream waits for the previous call's work on another. */

/* gpx_wire_decode_batch on device buffers.  bytes, pkts, status, accepts, blob, replies, decisions are device
 * pointers; the four counts are HOST pointers, capacities in / sizes out, with GPX_ERANGE exactly as in the host form
 * (sizes reported, no record written).  Stream-ordered on `stream` (NULL = the engine's stream); the call returns
 * after the one synchronisation that reads the totals.  Outputs, order and statuses are byte-identical to
 * gpx_wire_decode_batch, and feed gpx_accepts_device (n_chunks = 0), gpx_replies_device and gpx_decisions_device
 * as they are. */
int gpx_wire_decode_batch_device(gpx_engine* e, uint32_t n, const uint8_t* bytes, uint64_t n_bytes,
                                 const gpx_wire_ref* pkts, int32_t* status, gpx_accept_rec* accepts,
                                 uint32_t* n_accepts, uint8_t* blob, uint64_t* blob_bytes,
                                 gpx_accept_reply_rec* replies, uint32_t* n_replies,
                                 gpx_decision_rec* decisions, uint32_t* n_decisions, void* stream);

/* gpx_wire_encode_replies on device buffers (replies, rstatus, out, refs device; out_bytes / n_refs host,
 * capacities in / sizes out).  n = n_lanes x the ACCEPTs handled, which the caller always knows on the host. */
int gpx_wire_encode_replies_device(gpx_engine* e, uint32_t n, const gpx_accept_reply_rec* replies, uint8_t* rstatus,
                                   uint8_t* out, uint64_t* out_bytes, gpx_wire_ref* refs, uint32_t* n_refs,
                                   void* stream);

/* gpx_wire_encode_decisions on device buffers.  The number of records is read on the device from *n_ptr (device;
 * e.g. &ctl->n_decisions after gpx_replies_device), at most n_max; NULL n_ptr = n_max.  Records at and beyond
 * *n_ptr are neither read as input nor given an rstatus. */
int gpx_wire_encode_decisions_device(gpx_engine* e, const gpx_decision_rec* decisions, const uint32_t* n_ptr,
                                     uint32_t n_max, uint8_t* rstatus, uint8_t* out, uint64_t* out_bytes,
                                     gpx_wire_ref* refs, uint32_t* n_refs, void* stream);

/* ---- the JSON form of replies and commits -------------------------------------------------------------------------
 * A Java peer sends a BatchedAcceptReply or BatchedCommit as bytes only when it travels alone.  Under load its batcher
 * wraps a sweep's packets in a BATCHED_PAXOS_PACKET (type 37, PaxosPacketBatcher.process :270-277), which is a JSON
 * string {"type":90,"PT":37,"V":-1,"PP":[...]} whose members are the JSON objects of the BatchedAcceptReplies (34) and
 * BatchedCommits (35) (BatchedPaxosPacket.toJSONSmartImpl :87-99); a wrapper is at most 4 MiB.  A NACK is a singleton
 * ACCEPT_REPLY (8), always JSON.  gpx_wire_decode_json_device decodes these into the records gpx_wire_decode_batch
 * makes from the byte forms.
 *
 * Schema (the keys of PaxosPacket.toJSONObject :478-494 and of the subclasses' toJSONSmartImpl):
 *   every packet and member  "type" = 90 and "PT", both int; a member also "ID" (string; absent for PT 37) and "V" (int)
 *   8  ACCEPT_REPLY          "SNDR", "B", "S", "CP_S", "QID", and optionally "NACK" (bool)
 *   34 BATCHED_ACCEPT_REPLY  the keys of 8 and "SLOTS" = [slot, requestID, slot, requestID, ...] (an odd length is
 *                            malformed)
 *   35 BATCHED_COMMIT        "B", "GC_S", "GROUP" (int array), "SLOTS" (int array)
 *   37 BATCHED_PAXOS_PACKET  "PP", an array of objects; no "ID", "V" = -1
 * Strictness:
 *   - Key order is free, unknown keys are skipped whatever their value, a duplicated key takes its last value (the
 *     objects are hash maps), and any JSON whitespace may stand between tokens.
 *   - Strings take every JSON escape (\uXXXX and \/ included); a raw byte 0x80-0xff is that ISO-8859-1 character (a
 *     Java node writes String.getBytes("ISO-8859-1")); a raw control character is malformed.  "ID" is unescaped before
 *     the lookup; one with a character above U+00FF or longer than GPX_WIRE_MAX_ID characters is GPX_WS_UNKNOWN_NAME
 *     (no gid can have that name: the host decides).  "B" is "<int32>:<int32>", each part with an optional '-'.
 *   - int fields are JSON integers within int32; "QID" and the requestIDs of SLOTS within int64.  A fraction, an
 *     exponent, a leading zero or a leading '+' is malformed.  The reference would truncate some of these through
 *     Number.intValue(); no Java sender writes them, and input from outside the process is rejected rather than
 *     guessed at.
 *   - A skipped value nested deeper than 64 levels is malformed.
 *
 * The one deliberate difference between the forms: a singleton ACCEPT_REPLY's "QID" is read as the reference reads it,
 * with getInt (AcceptReplyPacket(JSONObject) :115), so req_id keeps its low 32 bits, sign-extended; the requestIDs of a
 * BatchedAcceptReply's SLOTS are read with getLong (BatchedAcceptReply(JSONObject) :71), as the byte form carries
 * them.  No state and no tally reads a reply's req_id (gpx_replies_device and gpx_handle_accept_replies use slot,
 * ballot, max_cp and who), so the difference reaches no state; gpx_wire_encode_replies copies it into the bytes it
 * writes.
 *
 * Scratch: the call sizes its working buffers from bounds known before its one synchronisation -- about 7 bytes of
 * engine-owned HBM per arena byte (chunk summaries, the two event lists at half the covered bytes each, member slots
 * at one per GPX_JSON_MIN_MEMBER bytes) plus about 1 KiB per packet -- and keeps them for the engine's next wire call,
 * as the other wire calls keep theirs. */
typedef struct gpx_wire_member { /* 16 B */
  uint32_t pkt;   /* index of the packet it came from */
  uint32_t off;   /* byte range of the member's JSON object in the arena (the whole packet for a bare one) */
  uint32_t len;
  int32_t status; /* GPX_WS_* */
} gpx_wire_member;

/* Decode JSON packets: BATCHED_PAXOS_PACKET wrappers and bare ACCEPT_REPLY / BATCHED_ACCEPT_REPLY / BATCHED_COMMIT
 * packets.  bytes, pkts, status, members, replies, decisions are device pointers; the three counts are HOST pointers,
 * capacities in / sizes out, and GPX_ERANGE reports the sizes and writes no output.  pkts[k].node is the node that
 * received packet k (gid ignored).  The packets' lengths must add up to at most n_bytes (refs that do not overlap
 * always do), else GPX_EINVAL and nothing is written.  Stream-ordered on `stream` (NULL = the engine's stream) with the
 * other wire calls' scratch; one synchronisation reads the totals.
 *   status[n]   GPX_WS_OK: well-formed JSON of type 37, or of type 8, 34 or 35 (one member, the whole packet); an
 *               empty PP is OK without members.  GPX_WS_MALFORMED: invalid JSON anywhere in the packet, a schema
 *               failure in it or in any member (no member of it is listed or gives records: the reference loses the
 *               whole container when its constructor throws), or a ref past n_bytes.  GPX_WS_UNHANDLED: not JSON (the
 *               first byte that is not whitespace is not '{': gpx_wire_decode_batch_device's), or JSON of another type.
 *   members[*n_members]  the members of the OK packets, in packet order and in PP order within one.  Member status:
 *               GPX_WS_UNKNOWN_NAME, GPX_WS_VERSION, GPX_WS_NOT_LOCAL, GPX_WS_OK as gpx_wire_decode_batch judges a
 *               byte packet, and GPX_WS_MALFORMED for an acceptor or coordinator outside the group; GPX_WS_UNHANDLED
 *               for other types (REQUEST, DECISION, BATCHED_ACCEPT, a nested 37) and an ACCEPT_REPLY with
 *               "NACK":true (digest mode's undigestRequest): the host takes those from off / len.  An
 *               GPX_WS_UNKNOWN_NAME member may be resubmitted alone, as a bare packet, once the host unpauses its group.
 *   replies[*n_replies]  34: one per SLOTS pair, byte-identical to what gpx_wire_decode_batch makes of the byte form
 *               (who = (member index of SNDR, member index of the ballot's coordinator, 0), max_cp = CP_S; S and QID
 *               validated, not used).  8: one reply, slot = S, max_cp = CP_S, ballot = B, req_id = QID (see above);
 *               its destination is the receiving node, not the ballot's coordinator -- a NACK carries the acceptor's
 *               higher ballot, whose coordinator is another node -- and GPX_WS_NOT_LOCAL when that node is not a
 *               member or no local lane serves it.
 *   decisions[*n_decisions]  35: one per SLOTS entry, median_cp = GC_S, flags GPX_F_DECISION, dst_mask = the group's
 *               local lanes, req_id 0; byte-identical to the byte form's.  GROUP is validated, not used.
 * Records are grouped by gid and, within a group, in (packet, member, slot) order: gpx_replies_device's and
 * gpx_decisions_device's input form. */
int gpx_wire_decode_json_device(gpx_engine* e, uint32_t n, const uint8_t* bytes, uint64_t n_bytes,
                                const gpx_wire_ref* pkts, int32_t* status, gpx_wire_member* members,
                                uint32_t* n_members, gpx_accept_reply_rec* replies, uint32_t* n_replies,
                                gpx_decision_rec* decisions, uint32_t* n_decisions, void* stream);

/* The sending side: a node's replies and commits as a loaded Java node sends them.
 *   GPX_JSON_WRAP_BYTES     a wrapper's default and largest size (4 MiB)
 *   GPX_JSON_WRAP_OVERHEAD  the bytes of a wrapper that are not its members or the commas between them:
 *                           {"type":90,"PT":37,"V":-1,"PP":[ and ]}
 *   GPX_JSON_MAX_MEMBER     the largest member object the call writes; a BatchedAcceptReply of up to 1,800 distinct
 *                           slots, or a BatchedCommit of up to 5,000, is always below it */
#define GPX_JSON_WRAP_BYTES 4194304u
#define GPX_JSON_WRAP_OVERHEAD 34u
#define GPX_JSON_MAX_MEMBER 65536u

/* Encode replies (gpx_handle_accepts' layout, record i * n_lanes + lane, n_replies a multiple of n_lanes) and
 * decisions (n_dec_ptr: a device count, at most n_dec_max, as in gpx_wire_encode_decisions_device; NULL = n_dec_max)
 * as the JSON a loaded Java node sends: BATCHED_PAXOS_PACKET wrappers (PaxosPacketBatcher.batch :280-303) of
 * BatchedAcceptReply and BatchedCommit objects, and each NACK as a bare ACCEPT_REPLY.  Either input may be empty.
 * The caller sends a sweep of at most MIN_PP_BATCH_SIZE (3) packets unwrapped (PaxosPacketBatcher.process :270-277),
 * with gpx_wire_encode_replies_device and gpx_wire_encode_decisions_device; this call always wraps.
 *   rstatus_replies[n_replies], rstatus_decisions[below the count]  the byte encoders' GPX_WE_* from the same rules,
 *     except for a reply with GPX_F_NACK: GPX_WE_NACK when it is written here as a bare ACCEPT_REPLY (its destination
 *     is a member no local lane serves, the group is live and named), else GPX_WE_LOCAL, GPX_WE_VOID or
 *     GPX_WE_NO_NAME as a positive reply would be.  NACKs are never wrapped (PaxosPacketBatcher.coalesce :345-387).
 *   Members: one BatchedAcceptReply per (lane, gid, ballot) run of GPX_WE_SENT replies, with the byte encoder's header
 *     (the run's first reply) and SLOTS = [slot, requestID, ...] ascending, the last put of a slot winning; one
 *     BatchedCommit per (gid, ballot) run of GPX_WE_SENT decisions with the wrap-aware maximum GC_S, GROUP = every
 *     member node in the member-set order, SLOTS ascending and distinct.  Each object, and each bare ACCEPT_REPLY
 *     (SNDR = the member node of WHO_ACC, S, CP_S and QID from the record), is byte-identical to packets_json's
 *     batched_accept_reply_json / batched_commit_json / accept_reply_json: keys in their order, "," and ":" with no
 *     spaces, strings escaped as json.dumps escapes them (\" \\ \b \f \n \r \t; every other byte below 0x20 and
 *     every byte from 0x7f up as \u00xx, lowercase).
 *   Sender and recipients: a reply is sent from lane i % n_lanes to the node of WHO_DST; a commit from the lane serving
 *     its ballot coordinator (else the group's lowest local lane, lane 0 when it has none) to every member node no
 *     local lane serves.  Recipient sets are compared as sets of node ids.
 *   Wrappers: each lane, ascending, sweeps its reply members in (gid, run) order, then its commit members in gid
 *     order (PaxosPacketBatcher.dequeueImpl :182-209).  Its members are grouped by recipient set in order of first
 *     appearance (the LinkedHashMap of batch :281-296), sweep order within a group.  A group is cut in parallel: with
 *     start_j the offset of member j in the group's comma-joined member stream and T = wrap_bytes -
 *     GPX_JSON_WRAP_OVERHEAD - GPX_JSON_MAX_MEMBER, member j opens a new wrapper iff floor(start_j / T) differs from
 *     its predecessor's, so no wrapper exceeds wrap_bytes.  A wrapper is {"type":90,"PT":37,"V":-1,"PP":[...]}.
 *     wrap_bytes = 0 means GPX_JSON_WRAP_BYTES; a value above it or at most GPX_JSON_WRAP_OVERHEAD +
 *     GPX_JSON_MAX_MEMBER is GPX_EINVAL.
 *   out[*out_bytes]  every packet once: the bare ACCEPT_REPLYs in record order, then the wrappers in (lane, first-seen
 *     recipient set, cut) order.
 *   refs[*n_refs]  one {off, len, gid, node} per (packet, recipient node), nodes ascending within a packet, in the
 *     order of out.  gid is the group for a bare ACCEPT_REPLY and the SENDING LANE for a wrapper.
 * replies, decisions, n_dec_ptr, rstatus_*, out and refs are device pointers; *out_bytes and *n_refs are HOST pointers,
 * capacities in / sizes out, and GPX_ERANGE reports the sizes and writes no packet.  A member larger than
 * GPX_JSON_MAX_MEMBER makes the call GPX_EINVAL with no packet written.  Stream-ordered on `stream` (NULL = the
 * engine's stream) with the other wire calls' scratch; one synchronisation reads the totals. */
int gpx_wire_encode_json_device(gpx_engine* e, uint32_t n_replies, const gpx_accept_reply_rec* replies,
                                const gpx_decision_rec* decisions, const uint32_t* n_dec_ptr, uint32_t n_dec_max,
                                uint8_t* rstatus_replies, uint8_t* rstatus_decisions, uint64_t wrap_bytes,
                                uint8_t* out, uint64_t* out_bytes, gpx_wire_ref* refs, uint32_t* n_refs, void* stream);

/* ---- the coordinator's side: REQUEST packets in, ACCEPT packets out ---------------------------------------------
 * A RequestPacket reaches the coordinator as REQUEST bytes (PaxosPacket type 1), from a client or forwarded by another
 * replica (PISM.handleProposal :854-885), and leaves inside the coordinator's AcceptPacket, which carries the whole
 * RequestPacket (AcceptPacket.java:95-138, RequestPacket.toBytes :819-949).  gpx_request_rec keeps what the engine
 * needs; gpx_wire_req_meta keeps the rest of the wire fields, so that the ACCEPT can be written again byte for byte.
 * Callers keep it parallel to the request array: meta[q] belongs to reqs[q].
 *
 * Requests that carry a digest (digest mode, PISM :842-843) or a non-empty responseValue stay on the host: the decoder
 * reports their packets as GPX_WS_UNHANDLED and the encoder always writes both as empty. */
#define GPX_RM_RETURN_VALUE 1u /* RequestPacket.shouldReturnRequestValue */
#define GPX_RM_BROADCASTED 2u  /* RequestPacket.broadcasted */
typedef struct gpx_wire_req_meta { /* 32 B */
  uint8_t client_ip[4];   /* clientAddress (zeros when client_port is 0) */
  uint16_t client_port;   /* 0 = no client address */
  uint16_t listen_port;   /* 0 = no listen address */
  uint8_t listen_ip[4];   /* listenAddress */
  int32_t forward_count;  /* RequestPacket.forwardCount */
  int64_t entry_time;     /* RequestPacket.entryTime (ms) */
  uint32_t flags;         /* GPX_RM_* */
  uint32_t pad;
} gpx_wire_req_meta;

/* Decode a batch of REQUEST packets into proposals.  bytes, pkts, status, reqs, meta and payload are device pointers;
 * pkts[k].node names the node that received packet k (gid ignored).  Outputs:
 *   reqs[*n_reqs], meta[*n_reqs]  grouped by gid, packet order within a group; a batched RequestPacket unrolls into
 *                          its outer request and then its `batched` entries in order -- gpx_propose_device's input form.
 *                          flags = STOP | the lane serving the receiving node << 8; client = packet index; an unset
 *                          entryReplica (IntegerMap.NULL_INT_NODE, -1) becomes the receiving node with entry_time =
 *                          now_ms (RequestPacket.setEntryReplica :393-403), otherwise both are the packet's.
 *   payload[*payload_bytes] every requestValue at a 16-byte aligned offset (payload_off).
 *   status[n]              GPX_WS_* per packet: GPX_WS_MALFORMED as gpx_wire_decode_batch judges an ACCEPT's request
 *                          part; GPX_WS_UNHANDLED for JSON, every type but REQUEST, and a digest or a responseValue in
 *                          any of its requests; GPX_WS_UNKNOWN_NAME / GPX_WS_VERSION from the name table;
 *                          GPX_WS_NOT_LOCAL when no local lane serves the receiving node or it is not a member.
 * *n_reqs and *payload_bytes are HOST pointers, capacities in / sizes out; GPX_ERANGE reports the sizes and writes
 * nothing else.  Stream-ordered on `stream` (NULL = the engine's stream); one synchronisation reads the totals. */
int gpx_wire_decode_requests_device(gpx_engine* e, uint32_t n, const uint8_t* bytes, uint64_t n_bytes,
                                    const gpx_wire_ref* pkts, int64_t now_ms, int32_t* status, gpx_request_rec* reqs,
                                    gpx_wire_req_meta* meta, uint32_t* n_reqs, uint8_t* payload,
                                    uint64_t* payload_bytes, void* stream);

/* gpx_propose_device, and out_head[n] (device): for each ACCEPT k below ctl->n_accepts, the index of the request that
 * starts its slot -- its nreq requests are [out_head[k], out_head[k] + nreq) -- or 0xffffffff for a VOID filler.
 * Every other output is byte-identical to gpx_propose_device's. */
int gpx_propose_device_heads(gpx_engine* e, const gpx_request_rec* reqs, const uint8_t* payload, uint64_t payload_bytes,
                             uint32_t n, int32_t* status, gpx_accept_rec* out_accepts, uint32_t* out_head,
                             gpx_dev_ctl* ctl, void* stream);

#define GPX_WE_BAD_HEAD 5 /* encode_accepts: head out of range, head + nreq > n_reqs, or reqs[head] of another gid */

/* Encode ACCEPTs as AcceptPackets, byte-identical to gpx_wire_encode_accept: the outer RequestPacket is request
 * heads[k] (header type ACCEPT), `batched` its next nreq - 1 requests as REQUEST packets, then slot, ballot,
 * recovery 0, median_cp, noCoalesce 0 and sender.  Request bodies are read at reqs[q].payload_off of `payload` (the
 * arena gpx_propose_device was given), never from the engine's constructed blobs.  The count of ACCEPTs is read on the
 * device from *n_ptr (e.g. &ctl->n_accepts), at most n_max; NULL = n_max.  Each packet is stored once and indexed once
 * per member node that no local lane serves, in gid order.  rstatus[k] (below the count): GPX_WE_SENT, GPX_WE_VOID,
 * GPX_WE_LOCAL (no remote member), GPX_WE_NO_NAME or GPX_WE_BAD_HEAD.  All pointers but out_bytes / n_refs (host,
 * capacities in / sizes out, GPX_ERANGE as above) are device pointers. */
int gpx_wire_encode_accepts_device(gpx_engine* e, const gpx_accept_rec* accepts, const uint32_t* n_ptr, uint32_t n_max,
                                   const uint32_t* heads, const gpx_request_rec* reqs, const gpx_wire_req_meta* meta,
                                   uint32_t n_reqs, const uint8_t* payload, uint8_t* rstatus, uint8_t* out,
                                   uint64_t* out_bytes, gpx_wire_ref* refs, uint32_t* n_refs, void* stream);

/* ---- forwarding: a non-coordinator's REQUEST packets to the coordinator -------------------------------------------
 * Clients send to any replica, and the coordinators are spread over the members, so most requests enter at a node that
 * does not coordinate their group; that node forwards them (PISM.handleProposal :854-885).  gpx_propose_device gives
 * them GPX_RS_FORWARD.  gpx_wire_encode_forwards_device writes the REQUEST packets the entry node sends, and the
 * coordinator decodes them with gpx_wire_decode_requests_device -- or, when a Java peer sent them as JSON members of a
 * BATCHED_PAXOS_PACKET, with gpx_wire_decode_json_requests_device. */
#define GPX_WE_ELECT 6 /* encode_forwards: the host runs for coordinator (PISM.checkRunForCoordinator) instead */

/* Encode the forwarded requests of a gpx_propose_device call as REQUEST packets.  reqs, meta (parallel to reqs, as in
 * gpx_wire_encode_accepts_device), status and payload are that call's request array, its gpx_wire_req_meta, its
 * statuses and its payload arena; run it after gpx_propose_device and before any call that changes the engine's state.
 *   Which requests: status GPX_RS_FORWARD, and propose_run's routing on the current rows still says FORWARD for the
 *     gid's run (the entry lane of the run's first request has no usable coordinator, and no local lane serves the
 *     acceptor's ballot coordinator).  Proposing changes neither the acceptor rows nor whether a coordinator exists, so
 *     this is k_propose's answer; it tells a forwarded request from one whose wrapped slot equals -2.  A broadcasted
 *     request (GPX_RM_BROADCASTED) reached every replica already and is not forwarded (:854).
 *   Packets: consecutive forwarded requests of one gid are cut as k_propose cuts a batch (BATCHING_ENABLED,
 *     MAX_BATCH_SIZE, the byte bound with the size estimate).  A cut is one REQUEST packet, byte-identical to
 *     gpx_wire_encode_request: the outer request is the cut's first with forwardCount + 1 (setForwarderID :437-441),
 *     the others its `batched` REQUEST packets with their own meta, unchanged.
 *   Destination: the ballot coordinator of the run's entry lane; when it is in down_nodes[n_down] (host, the nodes the
 *     host takes for down: PaxosManager.isNodeUp), the next member after it in sorted order (getNextCoordinator
 *     :2232-2241).
 *   GPX_WE_ELECT for every request of the cut, and no packet, when the destination is a node a local lane serves
 *     (coordinator == getMyID(), :869), the outer request ping-pongs after the increment (forwardCount > 3,
 *     RequestPacket.isPingPonging :508), or the ballot coordinator is not a member.
 * out[*out_bytes] receives the packets, refs[*n_refs] one {off, len, gid, node = destination} per packet in request
 * order; rstatus[n]: GPX_WE_SENT for every request inside a packet, GPX_WE_VOID for one that is not forwarded,
 * GPX_WE_ELECT, GPX_WE_NO_NAME.  *out_bytes and *n_refs are HOST pointers, capacities in / sizes out; GPX_ERANGE reports
 * the sizes and writes nothing else.  All other pointers but down_nodes are device pointers.  Stream-ordered on `stream`
 * (NULL = the engine's stream) with the other wire calls' scratch; one synchronisation reads the sizes. */
int gpx_wire_encode_forwards_device(gpx_engine* e, const gpx_request_rec* reqs, const gpx_wire_req_meta* meta,
                                    uint32_t n, const int32_t* status, const uint8_t* payload, uint32_t n_down,
                                    const int32_t* down_nodes, uint8_t* rstatus, uint8_t* out, uint64_t* out_bytes,
                                    gpx_wire_ref* refs, uint32_t* n_refs, void* stream);

/* Decode the REQUEST members of JSON packets (a Java peer's forwards, BATCHED_PAXOS_PACKET members) into proposals.
 * The input is what gpx_wire_decode_json_device returned for the same arena and refs: members[n_members], whose
 * wrappers are not read again.  bytes, pkts, members, status, reqs, meta and payload are device pointers.
 *   Which members: only those listed GPX_WS_UNHANDLED are examined; every other status is copied to status[i].  An
 *     object with "PT":1 is decoded; any other type stays GPX_WS_UNHANDLED.
 *   Schema (RequestPacket(net.minidev.json.JSONObject) :584-649, toJSONSmartImpl :697-742): "type" = 90, "PT", "ID"
 *     (string) and "V" (int) as for every member; "QID" (int64), "QV" (string), "ET" (int64) and "E" (int32) required;
 *     "NFWDS" (int32), "STOP", "QF", "BC" (bool), "CA", "LA" (string) and "BATCH" (an array of request objects, with
 *     the same request keys, one level) optional; "FWDR", "DBG" and unknown keys are skipped.  The strictness rules are
 *     gpx_wire_decode_json_device's.
 *   status[i]: GPX_WS_MALFORMED for a schema failure, a BATCH entry with a BATCH of its own, or a member ref past
 *     n_bytes or pkt past n_pkts.  GPX_WS_UNHANDLED when "RV" or "DIG" is present (as in the byte decoder), a "QV" has a
 *     character above U+00FF, or a "CA" / "LA" is not [anything/]a.b.c.d:port with a port of 1-65535 -- that is
 *     Util.getInetSocketAddressFromString :278-287 restricted to literal IPv4 addresses; a hostname needs a lookup and
 *     port 0 means "no address" in the byte form, so the host decides both.  GPX_WS_UNKNOWN_NAME, GPX_WS_VERSION and
 *     GPX_WS_NOT_LOCAL as gpx_wire_decode_requests_device judges them, the receiving node being pkts[members[i].pkt].node.
 *   reqs, meta, payload: gpx_wire_decode_requests_device's outputs with client = the member index, byte-identical for
 *     the same RequestPacket: an "E" of -1 becomes the receiving node and now_ms, an absent address is all zeros, "QV"
 *     is unescaped into payload at 16-byte aligned offsets.  Grouped by gid, member order within a gid, a request's
 *     BATCH after it: gpx_propose_device's input form.
 * One thread handles one member, its BATCH included, so a very long "QV" is copied by one thread.  *n_reqs and
 * *payload_bytes are HOST pointers, capacities in / sizes out, with GPX_ERANGE as above; stream-ordered, one
 * synchronisation. */
int gpx_wire_decode_json_requests_device(gpx_engine* e, uint32_t n_members, const uint8_t* bytes, uint64_t n_bytes,
                                         const gpx_wire_ref* pkts, uint32_t n_pkts, const gpx_wire_member* members,
                                         int64_t now_ms, int32_t* status, gpx_request_rec* reqs,
                                         gpx_wire_req_meta* meta, uint32_t* n_reqs, uint8_t* payload,
                                         uint64_t* payload_bytes, void* stream);

/* ---- a client's own requests: bare JSON REQUEST packets, addressed by the connection they came in on ------------
 * A gigapaxos client sends each RequestPacket as a bare JSON object, PaxosPacket.toJSONObject :478-494 ("type", "PT",
 * "ID", "V") over toJSONObjectImpl :652-694, neither as bytes nor inside a BATCHED_PAXOS_PACKET
 * (PaxosClientAsync.sendRequest :165-172).  Its clientAddress is null, so it carries no "CA": the reference takes the
 * client address from the connection.  On receipt MessageExtractor.stampAddressIntoJSONObject :348-376 adds
 * "_SNDR_ADDRESS" and "_RCVR_ADDRESS" (the socket's remote and local address) unless the keys are there already, and
 * RequestPacket(JSONObject) :530-536 uses "CA" if present, else the sender stamp; "LA" likewise with the receiver's.
 * The host's socket layer knows those two addresses for every packet it hands to the device: gpx_wire_peer. */
typedef struct gpx_wire_peer { /* 16 B */
  uint8_t sender_ip[4];   /* the connection's remote address (IPv4) */
  uint16_t sender_port;   /* 0 = unknown: no fallback address */
  uint16_t receiver_port; /* the local listen address the packet came in on; 0 = unknown */
  uint8_t receiver_ip[4];
  uint32_t pad;
} gpx_wire_peer;

/* Decode n bare JSON REQUEST packets from clients into proposals.  pkts[k] is packet k in the arena, pkts[k].node the
 * node that received it, peers[k] its connection.  bytes, pkts, peers, status, reqs, meta and payload are device
 * pointers; peers may be NULL (no fallback address: an absent one is all zeros, as in
 * gpx_wire_decode_json_requests_device).
 *   Which packets: a packet whose first byte after leading whitespace is '{' and whose object is "type":90, "PT":1.
 *     A byteified packet, and JSON of any other type or PT, is GPX_WS_UNHANDLED, so a node that receives both forms
 *     calls this and gpx_wire_decode_requests_device over the same arena.
 *   Schema, strictness, BATCH and the GPX_WS_* rules: gpx_wire_decode_json_requests_device's for a member, in the
 *     org.json form a client writes and the json-smart form alike, with the receiving node pkts[k].node.  A packet
 *     that is not one JSON object with an int "type", or whose "type" 90 comes without an int "PT", is
 *     GPX_WS_MALFORMED.
 *   Addresses, in the reference's order: client address = "CA" if the key is present, else "_SNDR_ADDRESS" if present,
 *     else peers[k].sender_*; listen address = "LA", else "_RCVR_ADDRESS", else peers[k].receiver_*.  A stamp is read
 *     in both forms the reference writes: "a.b.c.d:port" (org.json) and "[host]/a.b.c.d:port" (json-smart).  A present
 *     string that is not a literal IPv4 address with a port of 1-65535, or a fallback whose port is 0, makes the packet
 *     GPX_WS_UNHANDLED: the host decides (IPv6 and hostnames need a lookup).  A BATCH entry takes its own "CA" / "LA",
 *     else its own stamps, else no address (all zeros): RequestPacket(JSONObject) :541-552 builds each entry from its
 *     own object, which the receiver never stamps.
 *   reqs, meta, payload: byte-identical to gpx_wire_decode_json_requests_device's for the same RequestPacket with the
 *     resolved "CA" / "LA" written out, client = the packet index; an "E" of -1 becomes the receiving node and now_ms.
 *     Grouped by gid, packet order within a gid: the input of gpx_response_cache_match_device and gpx_propose_device.
 * One thread handles one packet, its BATCH included.  *n_reqs and *payload_bytes are HOST pointers, capacities in /
 * sizes out; GPX_ERANGE reports the sizes and writes nothing else.  Stream-ordered on `stream` (NULL = the engine's
 * stream) with the other wire calls' scratch; one synchronisation reads the totals. */
int gpx_wire_decode_client_requests_device(gpx_engine* e, uint32_t n, const uint8_t* bytes, uint64_t n_bytes,
                                           const gpx_wire_ref* pkts, const gpx_wire_peer* peers, int64_t now_ms,
                                           int32_t* status, gpx_request_rec* reqs, gpx_wire_req_meta* meta,
                                           uint32_t* n_reqs, uint8_t* payload, uint64_t* payload_bytes, void* stream);

/* Encode a node's whole non-digest sweep as a loaded Java node sends it: gpx_wire_encode_json_device's replies and
 * decisions, and the requests gpx_wire_encode_forwards_device forwards, as REQUEST members of the same
 * BATCHED_PAXOS_PACKET wrappers (BATCHED_REQUESTS and BATCH_ACROSS_GROUPS, both on by default: PaxosPacketBatcher
 * coalesces a forwarded RequestPacket without batched requests, allCoalescableRequests :447-454).  The replies'
 * and decisions' arguments are gpx_wire_encode_json_device's; reqs, meta, n_reqs, status, payload, n_down and
 * down_nodes are gpx_wire_encode_forwards_device's, with the same conditions.  With n_reqs == 0 every output, size and
 * return code is gpx_wire_encode_json_device's.
 *   rstatus_reqs[n_reqs]  byte for byte gpx_wire_encode_forwards_device's rstatus for the same inputs (GPX_WE_SENT,
 *     GPX_WE_VOID, GPX_WE_ELECT, GPX_WE_NO_NAME): the same routing, cuts, destinations and rules.
 *   Wrapped or alone: a GPX_WE_SENT cut of exactly one request is a REQUEST member, byte-identical to packets_json's
 *     request_json of that request with forwardCount + 1: "type", "PT", "ID", "V", "QID", "QV", "ET", "NFWDS" (when
 *     forwardCount + 1 > 0), "STOP" (when true), "E", "CA" and "LA" ("/a.b.c.d:port", when the port is nonzero), "QF"
 *     (when true), strings escaped as for gpx_wire_encode_json_device's names.  A cut of two or more requests -- a
 *     RequestPacket with batched requests, which the reference does not coalesce but sends byteified
 *     (PaxosMessenger.toJSONSmartObject :126-132) -- is written alone, byte-identical to the REQUEST packet
 *     gpx_wire_encode_forwards_device writes for it.  So is a one-request member larger than GPX_JSON_MAX_MEMBER: a
 *     deliberate difference, where a Java node would wrap it, so that a very large client value does not fail the
 *     whole sweep.  Both are GPX_WE_SENT.  An oversized reply or commit member stays GPX_EINVAL.
 *   Sender and recipients: a forward member is sent from the entry lane of its run's first request ((flags >> 8) &
 *     0xf, the lane propose_route routes from) to the singleton {destination}.  So a forward to node X shares a wrapper
 *     with that lane's replies to X and its commits whose only remote member is X.
 *   Sweep: each lane sweeps its replies, then its commits, then its forward members in request order
 *     (PaxosPacketBatcher.dequeueImpl :182-209); grouping by recipient set and the cut rule are
 *     gpx_wire_encode_json_device's.
 *   out[*out_bytes]  the bare ACCEPT_REPLYs in record order, then the lone REQUEST packets in request order, then the
 *     wrappers.  refs[*n_refs] in that order: a lone packet's ref is {off, len, gid, node = destination}, as
 *     gpx_wire_encode_forwards_device writes it; a wrapper's gid is the sending lane.
 * n_replies + n_dec_max + n_reqs above 2^31 - 1 is GPX_ERANGE.  Pointers, capacities, GPX_ERANGE, GPX_EINVAL, the
 * stream and the one synchronisation are gpx_wire_encode_json_device's; down_nodes is a HOST pointer.  As there, the
 * caller decides whether a sweep of at most MIN_PP_BATCH_SIZE packets goes unwrapped. */
int gpx_wire_encode_json_sweep_device(gpx_engine* e, uint32_t n_replies, const gpx_accept_reply_rec* replies,
                                      const gpx_decision_rec* decisions, const uint32_t* n_dec_ptr, uint32_t n_dec_max,
                                      const gpx_request_rec* reqs, const gpx_wire_req_meta* meta, uint32_t n_reqs,
                                      const int32_t* status, const uint8_t* payload, uint32_t n_down,
                                      const int32_t* down_nodes, uint8_t* rstatus_replies,
                                      uint8_t* rstatus_decisions, uint8_t* rstatus_reqs, uint64_t wrap_bytes,
                                      uint8_t* out, uint64_t* out_bytes, gpx_wire_ref* refs, uint32_t* n_refs,
                                      void* stream);

/* ---- response cache: a client's retransmitted request is answered from the cache, not proposed again -------------
 * PaxosManager.handleIncomingPacket :1084 checks every incoming REQUEST against the response cache before it is
 * batched (ENABLE_RESPONSE_CACHING, on by default); retransmittedRequest :332-349 answers a hit from the cached
 * response and drops the request; executed :311-330 puts every executed ClientRequest's response at every replica;
 * entries expire REQUEST_TIMEOUT after they are put.  On the device path the requests are decoded on the device, so
 * the check runs there: the engine keeps a key table in HBM, and the responses stay with the host app, which names
 * each one by a `handle` of its choosing.  A Java adapter calls gpx_response_cache_put after Replicable.execute and
 * gpx_response_cache_match between the request decoders and gpx_propose_device.
 *
 * Key identity: (gid, generation, req_id, client address) -- RequestPacket.equals :1489-1510 within one group.  The
 * generation of a gid starts at 0 and rises by one each time gpx_set_group_names names it (0 for every gid of an
 * engine that has no name state).  So an entry stops matching once its group is destroyed, paused, re-created or
 * loaded and then named again, where the reference would answer from it until it expires: a deliberate difference, a
 * response belongs to the group state that produced it.  client_port 0 means "no address" and equals only another
 * port 0 (Java's null == null); client_ip is then not read.
 *
 * Table: n_buckets buckets of 8 cells; a key's bucket is the low bits of
 *   splitmix64(req_id ^ splitmix64((uint64)gid << 32 | generation) ^ splitmix64((uint64)ip_be32 << 16 | port))
 * and a key never moves to another bucket.  A cell is expired when now_ms - put_ms >= timeout_ms.  A full bucket
 * costs only missed hits: a miss is proposed as it would be without the cache. */
typedef struct gpx_rc_key { /* 24 B: one executed client request */
  uint32_t gid;
  int32_t handle;         /* >= 0: the host's name for the cached response */
  int64_t req_id;
  uint8_t client_ip[4];   /* as gpx_wire_req_meta */
  uint16_t client_port;   /* 0 = no client address */
  uint16_t pad;
} gpx_rc_key;

/* Allocate the table: n_buckets (a power of two, at most 2^24; anything else is GPX_EINVAL) and timeout_ms (>= 0, the
 * host's REQUEST_TIMEOUT * 1000).  Calling it again clears the table.  gpx_response_cache_put and _match before it are
 * GPX_EINVAL. */
int gpx_response_cache_init(gpx_engine* e, uint32_t n_buckets, int64_t timeout_ms);

/* outstanding.responses.put of executed :318-322 for keys[n] (device), at now_ms.  Keys apply in input order; in its
 * bucket a key replaces the lowest live cell with the same key, else takes the lowest free or expired cell, else
 * evicts the cell with the smallest put time (the lowest such cell).  A negative handle or a gid >= max_groups is
 * GPX_EINVAL, and nothing is written.  Stream-ordered on `stream` (NULL = the engine's stream) with the wire calls;
 * one synchronisation reads the check. */
int gpx_response_cache_put_device(gpx_engine* e, uint32_t n, const gpx_rc_key* keys, int64_t now_ms, void* stream);

/* handleIncomingPacket :1084 + retransmittedRequest :332 for reqs[n] and meta[n] (device; a request decoder's output).
 * reqs[q] is a hit when no other request of the call has the same `client` value (the request decoders set it to the
 * packet or member index, so a request unrolled from a batched RequestPacket is never a hit), its gid has a name or
 * the engine has no name state, and a live cell holds its key, the address read from meta[q].
 *   hit[n] (device): the cell's handle for a hit, -1 for a miss.
 *   out_reqs, out_meta (device, room for n each): the misses in input order, so gpx_propose_device can take them as
 *     they are; *n_out (a HOST pointer) receives their count.
 * The table is read as it was before the call (a retransmission in the batch of its original is a miss); match never
 * inserts.  Stream-ordered as put; one synchronisation reads *n_out. */
int gpx_response_cache_match_device(gpx_engine* e, uint32_t n, const gpx_request_rec* reqs,
                                    const gpx_wire_req_meta* meta, int64_t now_ms, int32_t* hit,
                                    gpx_request_rec* out_reqs, gpx_wire_req_meta* out_meta, uint32_t* n_out,
                                    void* stream);

/* ---- helpers shared with the reference semantics ---------------------------------- */
int32_t gpx_java_string_hash(const char* s, size_t len); /* String.hashCode() */
/* PISM.roundRobinCoordinator :2251-2256 on sorted members */
int32_t gpx_round_robin_coordinator(int32_t name_hash, const int32_t* sorted_members, int32_t n,
                                    int32_t ballotnum);
/* PISM.getCPI :2694-2697 */
int32_t gpx_get_cpi(int32_t cpi, double noise, int32_t name_hash);

#ifdef __cplusplus
}
#endif
#endif /* GPX_H */
