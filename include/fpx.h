/*
 * fpx.h -- C ABI of the H100 quorum-vote engine (libfpx.so).
 *
 * This is the drop-in boundary for the FrankenPaxos quorum-vote hot path.  The
 * reference (mwhittaker/frankenpaxos, Scala) has no FFI; its extension surface
 * is the Actor/Transport/Chan traits.  A JVM actor (GpuProxyLeader/GpuAcceptor,
 * see INTEGRATION.md) batches the messages the transport delivers to it and
 * hands each batch, in delivery order, to one of the entry points below.  Every
 * entry point cites the reference handler it replaces.  Paths are relative to
 * the reference root; S/ = shared/src/main/scala/frankenpaxos/.
 *
 * Conventions
 *   - plain C, no CUDA / torch types in any signature;
 *   - all integers are int32 little-endian (the JVM's Int), records are 16-byte
 *     (or 8-byte) PODs that map 1:1 onto the protobuf fields of the reference;
 *   - host entry points (`fpx_x`) take HOST pointers, copy in, run, copy out
 *     and return when the results are in the caller's buffers;
 *   - device entry points (`fpx_x_dev`) take DEVICE pointers, enqueue on the
 *     engine's stream and return immediately; call fpx_sync() to collect the
 *     error status and the output counts;
 *   - a handle is not thread safe: the reference's contract is one
 *     single-threaded event loop per actor (S/Transport.scala:37-39);
 *   - return value 0 = ok, negative = fpx_status.  The reference has no error
 *     codes: handlers call logger.fatal (process exit / AssertionError under
 *     FakeLogger, S/FakeLogger.scala:11-14) or `require` (IllegalArgument).  A
 *     negative status is that event; *err_index receives the index, within the
 *     batch, of the FIRST offending record in delivery order (or -1).
 */
#ifndef FPX_H_
#define FPX_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FPX_ABI_VERSION 1

/* ---- records ------------------------------------------------------------ */

/* Phase2a as delivered to a proxy leader (arm) or to an acceptor (vote).
 * S/multipaxos/MultiPaxos.proto:273-280 {slot, round, command_batch_or_noop}.
 * value_id is a caller-owned 32-bit handle for the command batch bytes (the
 * bytes themselves never influence the path).  dst = group<<16 | acceptor is
 * the recipient the transport delivered this copy to; it is ignored by
 * fpx_proxyleader_arm. */
typedef struct { int32_t slot, round, value_id, dst; } fpx_p2a;

/* Phase2b == the four required int32 fields of
 * S/multipaxos/MultiPaxos.proto:282-290, in field order. */
typedef struct { int32_t group, acceptor, slot, round; } fpx_p2b;

/* Chosen{slot, value} S/multipaxos/MultiPaxos.proto (Chosen).  One record per
 * chosen (slot, round); the reference sends it to every replica in config
 * order (S/multipaxos/ProxyLeader.scala:246-253) -- that fan-out is the
 * caller's. */
typedef struct { int32_t slot, value_id; } fpx_chosen;

/* Nack{round} to leaders(phase2a.round % numLeaders)
 * (S/multipaxos/Acceptor.scala:192-199). */
typedef struct { int32_t leader, round; } fpx_nack;

/* value_id of CommandBatchOrNoop().withNoop(Noop()): what the range fills below write. */
#define FPX_VALUE_NOOP INT32_MIN

/* S/mencius/Mencius.proto Phase2aNoopRange{slotStartInclusive, slotEndExclusive, round}
 * as delivered to a proxy leader (dst ignored) or to acceptor dst = group<<16 | acceptor,
 * group = leader_group * num_acceptor_groups + acceptor_group. */
typedef struct { int32_t slot_start, slot_end, round, dst; } fpx_p2a_range;
/* Phase2bNoopRange{acceptorGroupIndex, acceptorIndex, slotStartInclusive,
 * slotEndExclusive, round}; the voter is packed in dst like above. */
typedef struct { int32_t dst, slot_start, slot_end, round; } fpx_p2b_range;
/* ChosenNoopRange{slotStartInclusive, slotEndExclusive}. */
typedef struct { int32_t slot_start, slot_end; } fpx_chosen_range;
/* S/vanillamencius Skip{serverIndex, startSlotInclusive, stopSlotExclusive} applied to
 * server `server`'s log; own = 1: the fill advanceWithSkips does at the skipping server. */
typedef struct { int32_t server, slot_start, slot_stop, own; } fpx_vm_skip_rec;
#define FPX_MAX_RANGE_BATCH 65535   /* records per range call */

/* ---- status ------------------------------------------------------------- */

typedef enum {
  FPX_OK = 0,
  FPX_ERR_INVALID_ARG = -1,        /* null pointer, n < 0, n > max_batch ...           */
  FPX_ERR_CONFIG = -2,             /* Config.checkValid() would `require`-fail          */
  FPX_ERR_CUDA = -3,               /* CUDA runtime error (fpx_last_error has the text)  */
  FPX_ERR_UNKNOWN_SLOT_ROUND = -4, /* Phase2b for a (slot,round) never armed:
                                      logger.fatal, S/multipaxos/ProxyLeader.scala:220-225 */
  FPX_ERR_BAD_ACCEPTOR = -5,       /* (group,acceptor) not a member of the quorum system:
                                      Grid.isWriteQuorum `require`, S/quorums/Grid.scala:44-47;
                                      also: group != slot % numAcceptorGroups (non-flexible)  */
  FPX_ERR_SLOT_RANGE = -6,         /* slot < 0, >= capacity, or not in this shard       */
  FPX_ERR_ROUND_RANGE = -7,        /* round < 0 or > FPX_MAX_ROUND                      */
  FPX_ERR_OVERFLOW_FULL = -8,      /* more concurrent secondary (slot,round) keys than
                                      config.overflow_capacity                           */
  FPX_ERR_CONFLICT = -9,           /* same key delivered twice with different values, and
                                      the in-batch order could not be resolved exactly   */
  FPX_ERR_NO_DEVICE = -10,
  FPX_ERR_UNSUPPORTED = -11,
  FPX_ERR_BATCH_ORDER = -12,       /* EPaxos batch contract E1/E2 violated (two messages of
                                      one instance / one (instance, replica) in one call):
                                      split the batch at err_index and resubmit           */
  FPX_ERR_CHECK_FAILED = -14,      /* a logger.check of the reference failed (vanilla Mencius
                                      advanceWithSkips: a slot to skip is not vacant)   */
  FPX_ERR_WIRE = -15,              /* malformed protobuf bytes: what parseFrom rejects with
                                      InvalidProtocolBufferException                    */
  FPX_ERR_EXCHANGE_TIMEOUT = -16,  /* fpx_global_watermark: a shard did not publish in time */
  FPX_ERR_EPAXOS_STATE = -13       /* transitionToPreAcceptPhase on a committed instance or
                                      with a regressing ballot: logger.fatal / checkLe,
                                      S/epaxos/Replica.scala:663-681                       */
} fpx_status;

#define FPX_MAX_ROUND 0x7ffffff0
#define FPX_MAX_ACCEPTORS 32       /* total acceptors (groups*per_group) per engine     */
#define FPX_MAX_VOTERS_PER_SLOT 30 /* acceptors that can vote on one slot               */

/* ---- configuration ------------------------------------------------------ */

typedef enum {
  FPX_MULTIPAXOS = 0,       /* S/multipaxos: ProxyLeader + Acceptor                      */
  FPX_MENCIUS = 1,          /* S/mencius: same handlers, quorum f+1 of the slot's group  */
  FPX_VANILLA_MENCIUS = 2   /* S/vanillamencius/Server.scala: per-slot round, self vote  */
} fpx_protocol;

/* Mirrors the fields of S/multipaxos/Config.scala:6-31 that the path reads.
 * Validity rules are those of Config.checkValid (S/multipaxos/Config.scala:32-147):
 *   f >= 1; num_leaders >= f+1; num_replicas >= f+1;
 *   !flexible: every group has exactly 2f+1 acceptors;
 *    flexible: groups = grid rows, acceptors_per_group = grid columns,
 *              min(rows, cols) - 1 >= f. */
typedef struct {
  int32_t struct_size;          /* = sizeof(fpx_config), ABI guard                      */
  int32_t protocol;             /* fpx_protocol                                          */
  int32_t f;
  int32_t num_acceptor_groups;  /* non-flexible: G; flexible: grid rows                  */
  int32_t acceptors_per_group;  /* non-flexible: 2f+1; flexible: grid columns            */
  int32_t flexible;             /* 0 / 1                                                 */
  int32_t num_leaders;
  int32_t num_replicas;
  int32_t slot_capacity;        /* GLOBAL slots [0, slot_capacity) the log can hold      */
  int32_t overflow_capacity;    /* secondary (slot, round) keys (two live rounds of one
                                   slot after a leader change); power of two or 0        */
  int32_t max_batch;            /* largest n of any one call                             */
  int32_t device;               /* CUDA ordinal                                          */
  int32_t shard_index;          /* this engine owns slots with slot % shard_count ==     */
  int32_t shard_count;          /*   shard_index (1 GPU: 0 / 1)                          */
  int32_t num_leader_groups;    /* FPX_MENCIUS: leader groups; slot s belongs to leader
                                   group s % num_leader_groups and, inside it, to acceptor
                                   group (s / num_leader_groups) % num_acceptor_groups
                                   (S/mencius/ProxyLeader.scala:169-176,231-234);
                                   num_acceptor_groups is then PER LEADER GROUP, num_leaders
                                   the leaders per group, and a record's group id is
                                   leader_group * num_acceptor_groups + acceptor_group.
                                   Nack.leader = leader_group * num_leaders + round %
                                   num_leaders (S/mencius/Acceptor.scala:215-219).  Other
                                   protocols: 0 or 1.                                    */
} fpx_config;

typedef struct fpx_engine fpx_engine; /* opaque */

/* ---- life cycle --------------------------------------------------------- */

int fpx_abi_version(void);
const char* fpx_strerror(int status);
const char* fpx_last_error(const fpx_engine* e); /* text of the last CUDA failure     */

/* Actor constructors of the reference: `new ProxyLeader(address, transport,
 * logger, config, ...)` S/multipaxos/ProxyLeader.scala:67-75 and `new
 * Acceptor(...)` S/multipaxos/Acceptor.scala:59-66 both start with
 * config.checkValid(); so does this.  One engine holds the state of every
 * acceptor of the config plus one proxy leader plus one replica log. */
int fpx_create(fpx_engine** out, const fpx_config* cfg);
void fpx_destroy(fpx_engine* e);
int fpx_reset(fpx_engine* e); /* back to the freshly constructed state */

/* ---- host-pointer entry points (the reference-facing calls) ------------- */

/* ProxyLeader.handlePhase2a, S/multipaxos/ProxyLeader.scala:175-215.
 * For each record in delivery order: if (slot, round) is unknown create
 * Pending(value, {}) (:213); a duplicate (slot, round) is ignored (:177-183).
 * Recipient choice (:190-196) uses the JVM's global RNG and is NOT reproduced:
 * the caller forwards the Phase2a copies and the acceptor batch carries the
 * recipients actually chosen. */
int fpx_proxyleader_arm(fpx_engine* e, const fpx_p2a* in, int32_t n, int64_t* err_index);

/* Acceptor.handlePhase2a, S/multipaxos/Acceptor.scala:184-220, for the
 * interleaved delivery stream of ALL acceptors of the config (record i goes to
 * acceptor in[i].dst).  Per acceptor, in delivery order: round_msg < round ->
 * Nack(round) to leaders(round_msg % numLeaders) (:192-199); else round =
 * round_msg, states(slot) = (round, value), maxVotedSlot = max(..) (:204-209),
 * reply Phase2b(group, index, slot, round) (:211-219).
 * out_p2b / out_nack receive the replies in delivery order of the messages
 * that caused them; capacity n each. */
int fpx_acceptor_phase2a(fpx_engine* e, const fpx_p2a* in, int32_t n,
                         fpx_p2b* out_p2b, int32_t* n_p2b,
                         fpx_nack* out_nack, int32_t* n_nack, int64_t* err_index);

/* ProxyLeader.handlePhase2b, S/multipaxos/ProxyLeader.scala:217-258, with the
 * quorum test of :238-243: non-flexible `phase2bs.size < f+1`, flexible
 * Grid.isWriteQuorum (S/quorums/Grid.scala:43-50).  Unknown (slot, round) is
 * fatal (:220-225) -> FPX_ERR_UNKNOWN_SLOT_ROUND; Done is ignored (:227-232);
 * the vote map assignment is idempotent per acceptor (:237).  out receives one
 * Chosen per (slot, round) whose quorum completes in this batch, ORDERED BY THE
 * INDEX OF THE COMPLETING VOTE (the order the reference's sends happen in);
 * capacity n. */
int fpx_proxyleader_phase2b(fpx_engine* e, const fpx_p2b* in, int32_t n,
                            fpx_chosen* out, int32_t* n_out, int64_t* err_index);

/* Replica.handleChosen, S/multipaxos/Replica.scala:572-627: first Chosen per
 * slot wins (:580-588); later ones are redundant.  Then the executable prefix
 * (executeLog stops at the first hole, :394-402). */
int fpx_replica_chosen(fpx_engine* e, const fpx_chosen* in, int32_t n, int64_t* err_index);

/* First GLOBAL slot of this shard's residue class that is not yet chosen, as
 * a global slot number (shard_count==1: the replica's executedWatermark had it
 * executed everything it could). */
int fpx_chosen_watermark(fpx_engine* e, int32_t* out);

/* Batched quorum predicates over member bitmasks (bit g*per_group+a set <=>
 * acceptor (g,a) in the set; bit 31 set <=> the set contains a non-member):
 * which: 0 isReadQuorum 1 isWriteQuorum 2 isSuperSetOfReadQuorum
 * 3 isSuperSetOfWriteQuorum; flexible -> Grid (S/quorums/Grid.scala:35-56),
 * else SimpleMajority over all acceptors of group 0
 * (S/quorums/SimpleMajority.scala:41-55).  out[i] = 0/1, or 2 where the
 * reference `require` would throw (non-member passed to is{Read,Write}Quorum). */
int fpx_quorum_eval(fpx_engine* e, int32_t which, const uint32_t* masks, int32_t n, uint8_t* out);

/* ---- state read-back (Phase1b / parity) --------------------------------- */

/* Acceptor (group, acceptor): scalars `round` (S/multipaxos/Acceptor.scala:95)
 * and `maxVotedSlot` (:104), and for the n_slots GLOBAL slots starting at
 * first_slot (only slots of this shard are written; others get -1) the vote
 * (voteRound, voteValue) of `states` (:98); voteRound = -1 where no vote. */
int fpx_snapshot_acceptor(fpx_engine* e, int32_t group, int32_t acceptor,
                          int32_t* round, int32_t* max_voted_slot,
                          int32_t first_slot, int32_t n_slots,
                          int32_t* vote_round, int32_t* vote_value);

/* Replica log read-back: value_id per global slot, -1 = hole. */
int fpx_snapshot_log(fpx_engine* e, int32_t first_slot, int32_t n_slots, int32_t* value_id);




/* ---- Phase 1 reads of the same state (SURVEY.md 8(f) rank 2) --------------
 * Acceptor.handlePhase1a, S/multipaxos/Acceptor.scala:148-182: phase1a.round <
 * round -> Nack(round): *nack_round = the acceptor's round, state unchanged;
 * else round = phase1a.round, *nack_round = -1, and the Phase1b's `info` is the
 * acceptor's votes from chosenWatermark on (:171-179), i.e. fpx_snapshot_acceptor
 * over [chosen_watermark, maxVotedSlot] with the voteRound = -1 slots dropped.
 * Not batched with Phase2a traffic: SURVEY 8(g) rule 2 makes it a batch boundary. */
int fpx_acceptor_phase1a(fpx_engine* e, int32_t group, int32_t acceptor, int32_t round, int32_t* nack_round);

/* Leader.handlePhase1b's fill-in, S/multipaxos/Leader.scala:318-329,536-562: for the
 * n_slots slots from first_slot, the vote with the highest voteRound among the
 * acceptors that answered Phase 1 (responders: bit group*acceptors_per_group+index)
 * and may vote on the slot -- safeValue -- or vote_round = -1 / value_id = -1 where
 * none voted (Noop is safe).  *max_slot = the largest slot with a vote among the
 * responders (maxPhase1bSlot, :303-312), -1 if none.
 * Flexible grids: the reference's fill-in literally reads phase1bs(slot % numAcceptorGroups)
 * (:553), i.e. ONE grid row per slot, although every acceptor of the grid may hold a vote
 * for the slot; this call takes the maximum over ALL responders (never a lower round than
 * the reference's answer; identical whenever that row holds the responders' highest vote). */
int fpx_leader_safe_values(fpx_engine* e, uint32_t responders, int32_t first_slot, int32_t n_slots,
                           int32_t* vote_round, int32_t* value_id, int32_t* max_slot);

/* ---- Vanilla Mencius (S/vanillamencius/Server.scala), protocol FPX_VANILLA_MENCIUS ----
 * n = 2f+1 servers (acceptors_per_group = n, num_acceptor_groups = 1), every
 * server is proposer + acceptor, server s coordinates the slots with slot % n ==
 * s.  One engine holds the log entries of all n servers (vote cells [slot][server])
 * and the coordinators' `phase2s`.  Skips, revocation and Phase 1 are control
 * path and out of scope (SURVEY.md 8(a) row a9).  Batch contract (checked, ->
 * FPX_ERR_BATCH_ORDER): at most one Phase2a per (slot, server) per call, because
 * the round compare is per log entry (:1016-1042), not per acceptor.          */

/* Server.handleClientRequest, state part (:767-829): the coordinator in.dst (which
 * must own in.slot) votes for its own command -- log(slot) = PendingEntry(0, 0,
 * value) (:779) -- and opens phase2s(slot) with its own Phase2b (:818-825). */
int fpx_vm_client_request(fpx_engine* e, const fpx_p2a* in, int32_t n, int64_t* err_index);

/* Server.handlePhase2a (:1001-1082) at server in.dst.  DENSE replies, reply[i]
 * answers in[i]: {group = kind, acceptor = server, slot, round}:
 *   kind 0  Phase2b(server, slot, round)                 (:1077-1081)
 *   kind 1  Phase2Nack(slot, round = the entry's round)  (:1044-1051)
 *   kind 2  Chosen(slot, value in `round`)               (:1018-1027, entry already chosen) */
int fpx_vm_phase2a(fpx_engine* e, const fpx_p2a* in, int32_t n, fpx_p2b* reply, int64_t* err_index);
/* device-pointer forms (asynchronous on the engine's stream, errors surface at fpx_sync) */
int fpx_vm_client_request_dev(fpx_engine* e, const fpx_p2a* d_in, int32_t n);
int fpx_vm_phase2a_dev(fpx_engine* e, const fpx_p2a* d_in, int32_t n, fpx_p2b* d_reply);

/* Server.handlePhase2b (:1084-1142) is fpx_proxyleader_phase2b with this protocol's
 * rules: no Phase 2 running for the slot -> ignored (:1099-1106), stale round ->
 * ignored (:1109-1112), larger round -> checkEq fails (FPX_ERR_UNKNOWN_SLOT_ROUND,
 * :1116), quorum f+1 INCLUDING the coordinator's own vote (:1119-1122); on completion
 * the coordinator's own entry becomes ChosenEntry (choose, :622-625). */

/* Server.handleChosen -> choose (:1170-1197, :622-640): server in.acceptor learns
 * that in.slot is chosen with value in.round: its entry becomes ChosenEntry; if it
 * coordinates the slot, phase2s(slot) is dropped. */
int fpx_vm_learn_chosen(fpx_engine* e, const fpx_p2b* in, int32_t n, int64_t* err_index);

/* Skips.  own = 1: the log fill of advanceWithSkips (:577-620) at the skipping server --
 * its own slots slot_start, slot_start + n, ... < slot_stop become ChosenEntry(Noop); each
 * must be vacant (logger.check(!log.contains) / check(!phase2s.contains), :613-614 ->
 * FPX_ERR_CHECK_FAILED); nextSlot and skipSlots stay the caller's scalars.  own = 0:
 * handleSkip (:1144-1168) at `server`: choose(slot, Noop) for the coordinator's slots of
 * the range (log.put unconditionally, phase2s.remove, :622-625).  n <= FPX_MAX_RANGE_BATCH. */
int fpx_vm_skip(fpx_engine* e, const fpx_vm_skip_rec* in, int32_t n, int64_t* err_index);

/* ---- Mencius Phase2aNoopRange path (S/mencius), protocol FPX_MENCIUS ---------------
 * A lagging leader group closes its gap with ONE message standing for the strided run
 * of Noop slots {s in [start, end) : s = start (mod numLeaderGroups)} (Leader.scala:
 * 742-764).  The four handlers below are the range forms of arm / acceptor_phase2a /
 * proxyleader_phase2b / replica_chosen and share their state (the acceptors' rounds and
 * vote cells, the replica log).  Deliver ranges and single-slot messages in separate
 * calls, each a batch in delivery order; n <= FPX_MAX_RANGE_BATCH.  Preconditions the
 * reference does not state (it would loop or index out of bounds): 0 <= start <= end <=
 * slot_capacity (FPX_ERR_SLOT_RANGE), round as for Phase2a, dst an acceptor of leader
 * group start % numLeaderGroups (FPX_ERR_BAD_ACCEPTOR).
 *
 * ProxyLeader.handlePhase2aNoopRange (S/mencius/ProxyLeader.scala:255-303): key
 * SlotRound(start, end, round) present -> ignored, else PendingPhase2aNoopRange.  The
 * key space is shared with Phase2a (slot, slot+1, round) (:217-219): a one-slot range and
 * that slot's Phase2a exclude each other, first one wins (both directions checked here
 * and in fpx_proxyleader_arm).  Table of overflow_capacity (>= 1024) keys
 * (FPX_ERR_OVERFLOW_FULL).  [A Phase2b for a key held by a one-slot RANGE would be
 * ignored by the reference (:319-332) and is FPX_ERR_UNKNOWN_SLOT_ROUND here; no
 * execution produces it, the proxy leader never forwarded that Phase2a.] */
int fpx_mencius_arm_range(fpx_engine* e, const fpx_p2a_range* in, int32_t n, int64_t* err_index);
/* Acceptor.handlePhase2aNoopRange (S/mencius/Acceptor.scala:237-291): round < the
 * acceptor's round -> Nack(round) to leaders(start % LG)(round % leadersPerGroup); else
 * round = msg.round, the acceptor group's slots of the range get State(round, Noop)
 * (first such slot, then stride numLeaderGroups * numAcceptorGroups, :263-277), reply
 * Phase2bNoopRange.  Outputs compacted in delivery order like fpx_acceptor_phase2a. */
int fpx_mencius_acceptor_noop_range(fpx_engine* e, const fpx_p2a_range* in, int32_t n, fpx_p2b_range* out,
                                    int32_t* n_out, fpx_nack* out_nack, int32_t* n_nack, int64_t* err_index);
/* ProxyLeader.handlePhase2bNoopRange (S/mencius/ProxyLeader.scala:355-412): unknown key ->
 * logger.fatal (FPX_ERR_UNKNOWN_SLOT_ROUND), Done -> ignored, else record the vote and wait
 * until EVERY acceptor group of the leader group has f+1 votes (:394-396); the completing
 * delivery emits ChosenNoopRange(start, end), in delivery order. */
int fpx_mencius_range_phase2b(fpx_engine* e, const fpx_p2b_range* in, int32_t n, fpx_chosen_range* out,
                              int32_t* n_out, int64_t* err_index);
/* Replica.handleChosenNoopRange (S/mencius/Replica.scala:464-486): slots start, start+LG,
 * ... < end are put as Noop UNTIL THE FIRST ONE ALREADY IN THE LOG, where the reference's
 * handler returns (:476-480).  Batch contract (FPX_ERR_BATCH_ORDER): two records of one
 * call must not cover a common slot.  With shard_count > 1 "already in the log" is judged
 * on this shard's slots only (use the _first / _fill pair below for the reference's result).  fpx_chosen_watermark afterwards is the first hole, i.e.
 * where executeLog stops when it next runs. */
int fpx_mencius_replica_chosen_range(fpx_engine* e, const fpx_chosen_range* in, int32_t n, int64_t* err_index);
/* The two halves of the call above for a log sharded by slot residue, where "the first slot already in the log"
 * (:476-480) may live on another shard: _first reports, per record, this shard's first slot of the range that is
 * in its log (FPX_RANGE_NO_HIT if none) and changes nothing; the caller takes the minimum over the shards (one
 * integer per record: sharding.replica_chosen_range all-reduces it) and hands it to _fill, which puts Noop into
 * this shard's slots of [start, min(end, first[i])).  With the minimum over all shards the union of the shards'
 * logs is the reference's log. */
#define FPX_RANGE_NO_HIT 0x7f7f7f7f
int fpx_mencius_replica_range_first(fpx_engine* e, const fpx_chosen_range* in, int32_t n, int32_t* first_out,
                                    int64_t* err_index);
int fpx_mencius_replica_range_fill(fpx_engine* e, const fpx_chosen_range* in, int32_t n, const int32_t* first,
                                   int64_t* err_index);

/* ---- Wire codec: the reference's protobuf bytes <-> the records above ---------------
 * Every actor's inbound serializer is ProtoSerializer (S/ProtoSerializer.scala:3-11:
 * scalapb toByteArray / parseFrom), and parsing + serialising dominate a handler's time in
 * the reference.  These entry points take a BATCH of received messages as one byte buffer
 * plus offsets[n+1] (message i = bytes[offsets[i] .. offsets[i+1])) and decode it on the
 * GPU, and encode a batch of reply records into the same layout.  Shapes from
 * S/multipaxos/MultiPaxos.proto: Phase2a :273-280, Phase2b :282-290, Chosen :292-298, Nack
 * :455-460, LeaderInbound.nack = 6 :525-539, ProxyLeaderInbound {phase2a = 1, phase2b = 2}
 * :541-549, AcceptorInbound {phase2a = 2} :551-561, ReplicaInbound.chosen = 1 :563-576.
 * Parsing follows protobuf-java's CodedInputStream as scalapb drives it: varints of at most
 * 10 bytes, int32 = low 32 bits, unknown fields skipped by wire type, oneof = last member on
 * the wire, a missing required field or malformed bytes -> FPX_ERR_WIRE with the message's
 * index (group wire types and a repeated command_batch_or_noop, which no serializer emits,
 * are FPX_ERR_WIRE too).  Encoders emit the canonical form (fields in number order, minimal
 * varints, negative int32 as 10 bytes), which is what toByteArray produces.  Buffers: bytes
 * and out 16-byte aligned for the *_dev forms; total size below 2^31. */
enum { FPX_WIRE_PROXYLEADER_INBOUND = 0, FPX_WIRE_ACCEPTOR_INBOUND = 1,
       /* S/mencius/Mencius.proto (protocol FPX_MENCIUS): ProxyLeaderInbound :339-350 {phase2a = 2,
        * phase2a_noop_range = 3, phase2b = 4, phase2b_noop_range = 5}, AcceptorInbound :352-361 */
       FPX_WIRE_MENCIUS_PROXYLEADER_INBOUND = 2, FPX_WIRE_MENCIUS_ACCEPTOR_INBOUND = 3 };
/* One decoded message.  kind[i] = field number of the `request` oneof member that is set
 * (0: none).  Phase2b -> {group, acceptor, slot, round} (an fpx_p2b; mencius' Phase2b :169-176
 * has no group index: 0); Phase2a -> {slot, round, value_off, value_len}: the
 * CommandBatchOrNoop is bytes[value_off .. +value_len), never read; mencius
 * Phase2aNoopRange :160-167 -> {slot_start, slot_end, round, 0}; Phase2bNoopRange :178-187 ->
 * an fpx_p2b_range (dst built from acceptor_group_index and the leader group of slot_start;
 * -1 if out of range); any other member -> {0, 0, body_off, body_len} for the host. */
typedef struct { int32_t a, b, c, d; } fpx_wire_rec;

int fpx_wire_decode_inbound(fpx_engine* e, int32_t inbound, const uint8_t* bytes, const int32_t* offsets, int32_t n,
                            int32_t* kind, fpx_wire_rec* out, int64_t* err_index);
int fpx_wire_decode_inbound_dev(fpx_engine* e, int32_t inbound, const uint8_t* d_bytes, const int32_t* d_offsets,
                                int32_t n, int32_t* d_kind, fpx_wire_rec* d_out);
/* ProxyLeaderInbound{phase2b}: the acceptor's replies, ready for transport.send.  offsets[n+1]
 * is written; the bytes must fit out_capacity (FPX_ERR_INVALID_ARG otherwise).  With protocol
 * FPX_MENCIUS the mencius shape is written ({acceptor_index, slot, round} under field 4). */
int fpx_wire_encode_phase2b(fpx_engine* e, const fpx_p2b* in, int32_t n, uint8_t* out, int32_t out_capacity,
                            int32_t* offsets, int64_t* err_index);
int fpx_wire_encode_phase2b_dev(fpx_engine* e, const fpx_p2b* d_in, int32_t n, uint8_t* d_out, int32_t out_capacity,
                                int32_t* d_offsets);
/* LeaderInbound{nack{round}}; in[i].leader selects the destination and is not on the wire. */
int fpx_wire_encode_nack(fpx_engine* e, const fpx_nack* in, int32_t n, uint8_t* out, int32_t out_capacity,
                         int32_t* offsets, int64_t* err_index);
/* ReplicaInbound{chosen{slot, command_batch_or_noop}}: the value bytes of value_id v are
 * arena[value_offsets[v] .. value_offsets[v+1]) (e.g. the Phase2a payloads the proxy leader
 * kept); value_id out of [0, num_values) -> FPX_ERR_INVALID_ARG with the record's index. */
int fpx_wire_encode_chosen(fpx_engine* e, const fpx_chosen* in, int32_t n, const uint8_t* arena,
                           const int32_t* value_offsets, int32_t num_values, uint8_t* out, int32_t out_capacity,
                           int32_t* offsets, int64_t* err_index);

/* ---- EPaxos replica (S/epaxos/Replica.scala) ------------------------------
 * One fpx_epaxos handle = one replica's cmdLog (:298-330) and leaderStates
 * (:347-386) for n = 2f+1 replicas, instances (replicaIndex, instanceNumber <
 * instances_per_replica).  Messages are rows of int32 of fixed width (n = 2f+1);
 * dependency sets are DENSE watermark vectors of n ints (InstancePrefixSet with
 * empty `values`, the topKDependencies = 1 default, Replica.scala:95); general
 * sets go through fpx_depset_union.  Ballot = (ordering, replicaIndex), tuple
 * order (S/epaxos/BallotHelpers.scala:11-21).  Replies / events are DENSE: row i
 * of the output belongs to message i of the input (kind 0 = nothing to send).
 * Batch contract, checked on the device (FPX_ERR_BATCH_ORDER + first index):
 *   E1 lead / preaccept / accept: at most one message per instance per call;
 *   E2 preacceptok / acceptok: at most one message per (instance, replica) per
 *      call; a PreAcceptOk that replaces an earlier response of its replica with
 *      DIFFERENT content must be the only message of its instance in the call.
 * What the conflict index would compute (computeSequenceNumberAndDependencies,
 * :569-600) is an INPUT: `local_deps` of a PreAccept, `deps` of lead.        */
typedef struct fpx_epaxos fpx_epaxos;
typedef struct {
  int32_t struct_size;
  int32_t f;                      /* n = 2f+1 <= 7; fast quorum n-1, slow f+1 (S/epaxos/Config.scala:8-9) */
  int32_t replica_index;          /* this replica                                                       */
  int32_t instances_per_replica;
  int32_t max_batch;
  int32_t device;
} fpx_epaxos_config;

enum { FPX_EP_REPLY_NONE = 0, FPX_EP_REPLY_OK = 1, FPX_EP_REPLY_NACK = 2, FPX_EP_REPLY_COMMIT = 3 };
enum { FPX_EP_EV_NONE = 0, FPX_EP_EV_FAST_COMMIT = 1, FPX_EP_EV_SLOW_ACCEPT = 2, FPX_EP_EV_TIMER = 3,
       FPX_EP_EV_COMMIT = 4 };

int fpx_epaxos_create(fpx_epaxos** out, const fpx_epaxos_config* cfg);
void fpx_epaxos_destroy(fpx_epaxos* e);

/* transitionToPreAcceptPhase, Replica.scala:633-729 (the leader's own cmdLog entry
 * + PreAccepting state with its own response).  in rows of 8+n ints:
 * {inst_replica, inst_number, ballot_ord, ballot_rep, value_id, seq, avoid_fast_path, 0, deps[n]} */
int fpx_epaxos_lead(fpx_epaxos* e, const int32_t* in, int32_t n_rec, int64_t* err_index);
/* handlePreAccept, Replica.scala:1159-1289.  in rows of 6+2n ints: {inst_replica,
 * inst_number, ballot_ord, ballot_rep, value_id, seq, local_deps[n], msg_deps[n]};
 * reply rows of 4+n ints: {kind, ballot_ord, ballot_rep, seq, deps[n]} -- PreAcceptOk
 * (kind OK), Nack(largestBallot) (kind NACK), Commit resend (kind COMMIT). */
int fpx_epaxos_preaccept(fpx_epaxos* e, const int32_t* in, int32_t n_rec, int32_t* reply, int64_t* err_index);
/* handleAccept, Replica.scala:1421-1512.  in rows of 6+n ints: {inst_replica,
 * inst_number, ballot_ord, ballot_rep, value_id, seq, deps[n]}; reply as above (OK = AcceptOk). */
int fpx_epaxos_accept(fpx_epaxos* e, const int32_t* in, int32_t n_rec, int32_t* reply, int64_t* err_index);
/* handlePreAcceptOk, Replica.scala:1291-1419 incl. the fast-path equality vote
 * (Util.popularItems, S/Util.scala:19-21, threshold n-2) and preAcceptingSlowPath
 * (:796-813, dep-set union of all responses).  in rows of 6+n ints: {inst_replica,
 * inst_number, ballot_ord, ballot_rep, from_replica, seq, deps[n]}; event rows of
 * 2+n ints: {kind, seq, deps[n]}. */
int fpx_epaxos_preacceptok(fpx_epaxos* e, const int32_t* in, int32_t n_rec, int32_t* event, int64_t* err_index);
/* handleAcceptOk, Replica.scala:1514-1565.  in rows of 6 ints: {inst_replica,
 * inst_number, ballot_ord, ballot_rep, from_replica, 0}; event rows as above (COMMIT). */
int fpx_epaxos_acceptok(fpx_epaxos* e, const int32_t* in, int32_t n_rec, int32_t* event, int64_t* err_index);
/* The same handlers on DEVICE-resident rows, asynchronous on the handle's stream (fpx_epaxos_stream, a
 * cudaStream_t); status and first offending index are collected by fpx_epaxos_sync. */
void* fpx_epaxos_stream(fpx_epaxos* e);
int fpx_epaxos_sync(fpx_epaxos* e, int64_t* err_index);
int fpx_epaxos_lead_dev(fpx_epaxos* e, const int32_t* d_in, int32_t n_rec);
int fpx_epaxos_preaccept_dev(fpx_epaxos* e, const int32_t* d_in, int32_t n_rec, int32_t* d_reply);
int fpx_epaxos_accept_dev(fpx_epaxos* e, const int32_t* d_in, int32_t n_rec, int32_t* d_reply);
int fpx_epaxos_preacceptok_dev(fpx_epaxos* e, const int32_t* d_in, int32_t n_rec, int32_t* d_event);
int fpx_epaxos_acceptok_dev(fpx_epaxos* e, const int32_t* d_in, int32_t n_rec, int32_t* d_event);
/* handlePreAccept for callers whose dependency sets may be SPARSE (IntPrefixSet with overflow `values`,
 * S/compact/IntPrefixSet.scala:388-398, created by subtractOne below the watermark / top-k > 1):
 * overflow_count[i] = number of overflow values in message i's local + message sets.  This handle computes with
 * dense watermark vectors only: a message with overflow values is FPX_ERR_UNSUPPORTED (err_index = that message,
 * nothing of the batch is applied); union such sets with fpx_depset_union on the side. */
int fpx_epaxos_preaccept_sets(fpx_epaxos* e, const int32_t* in, int32_t n_rec, const int32_t* overflow_count,
                              int32_t* reply, int64_t* err_index);
/* read-back: out[7+n] = {kind, b_ord, b_rep, vb_ord, vb_rep, value_id, seq, deps[n]},
 * kind 0 none 1 NoCommand 2 PreAccepted 3 Accepted 4 Committed; *leader_kind 0 none 1
 * PreAccepting 2 Accepting; largest_ballot[2] */
/* device time (ms, CUDA events on the handle's stream) of the kernels of the last
 * fpx_epaxos_* call, without its host<->device copies */
float fpx_epaxos_last_kernel_ms(fpx_epaxos* e);
int fpx_epaxos_entry(fpx_epaxos* e, int32_t inst_replica, int32_t inst_number, int32_t* out,
                     int32_t* leader_kind, int32_t* largest_ballot);

/* Batched IntPrefixSet union (S/compact/IntPrefixSet.scala:253-259 == repeated
 * addAll :317-351, then compact :426-431).  Sets in CSR form: watermark[j] and
 * values[off[j] .. off[j+1]) (canonical: every value > its watermark); group q
 * unions sets [group_off[q], group_off[q+1]).  Output: out_watermark[q],
 * out_count[q] and the sorted overflow values at out_values[off[group_off[q]] ..).
 * `device` = CUDA ordinal. */
int fpx_depset_union(int32_t device, const int32_t* watermark, const int32_t* off, const int32_t* values,
                     int32_t n_sets, const int32_t* group_off, int32_t n_groups, int32_t* out_watermark,
                     int32_t* out_count, int32_t* out_values);

/* Dense batched dep-set union, DEVICE pointers (BASELINE cfg4's "dep-set union kernel"):
 * out[q][k] = max_r in[q][r][k] for q < n_groups, r < sets_per_group, k < n_replicas --
 * InstancePrefixSet.addAll over sets whose `values` are empty (IntPrefixSet.scala:320-321),
 * e.g. preAcceptingSlowPath's union of the R responses of an instance (Replica.scala:804-807).
 * Asynchronous on `stream` (a cudaStream_t, 0 = default stream). */
int fpx_depset_union_dense_dev(int32_t device, const int32_t* d_in, int32_t n_groups, int32_t sets_per_group,
                               int32_t n_replicas, int32_t* d_out, void* stream);

/* ---- device-pointer entry points (inputs already resident in HBM) ------- */

/* Same semantics, DEVICE pointers, asynchronous on fpx_stream(e).  Output
 * counts and the error status are collected by fpx_sync. */
int fpx_proxyleader_arm_dev(fpx_engine* e, const fpx_p2a* d_in, int32_t n);
int fpx_acceptor_phase2a_dev(fpx_engine* e, const fpx_p2a* d_in, int32_t n,
                             fpx_p2b* d_out_p2b, fpx_nack* d_out_nack);
int fpx_proxyleader_phase2b_dev(fpx_engine* e, const fpx_p2b* d_in, int32_t n,
                                fpx_chosen* d_out);
int fpx_replica_chosen_dev(fpx_engine* e, const fpx_chosen* d_in, int32_t n);
/* as fpx_replica_chosen_dev, but n is read on the device from the count the
 * last fpx_proxyleader_phase2b_dev produced (no host round trip) */
int fpx_replica_chosen_last_dev(fpx_engine* e, const fpx_chosen* d_in);
int fpx_chosen_watermark_dev(fpx_engine* e, int32_t* d_out);

typedef struct {
  int32_t status;        /* first (lowest record index) error of any call since last sync */
  int32_t reserved;
  int64_t err_index;
  int32_t n_p2b, n_nack; /* of the last fpx_acceptor_phase2a_dev                         */
  int32_t n_chosen;      /* of the last fpx_proxyleader_phase2b_dev                      */
  int32_t watermark;     /* of the last fpx_chosen_watermark_dev                         */
} fpx_sync_result;

int fpx_sync(fpx_engine* e, fpx_sync_result* out);

/* One pipeline step of co-located roles on device-resident buffers, issued from one C call, with the same
 * results as fpx_proxyleader_arm_dev, fpx_acceptor_phase2a_dev, fpx_proxyleader_phase2b_dev,
 * fpx_replica_chosen_last_dev, fpx_chosen_watermark_dev in that order -- in three launches: the acceptor
 * batch, the arm batch (disjoint state, so the order of those two is free; the rows armed last are still
 * L2-resident when the votes are tallied), and the tally with the replica's handleChosen and the watermark
 * scan (+ the multi-GPU exchange store) riding in the same cooperative kernel.
 * ring_slot >= 0 additionally records CUDA events on the engine's stream before and after the
 * acceptor and the tally kernel; fpx_step_kernel_ms(ring_slot) returns their durations once the
 * step has run (a ring of 1024 steps). */
int fpx_step_dev(fpx_engine* e, const fpx_p2a* d_arm, int32_t n_arm, const fpx_p2a* d_p2a, int32_t n_p2a,
                 fpx_p2b* d_out_p2b, fpx_nack* d_out_nack, const fpx_p2b* d_p2b, int32_t n_p2b, fpx_chosen* d_out_chosen,
                 int32_t* d_watermark, int32_t ring_slot);
/* The vanilla Mencius form (protocol FPX_VANILLA_MENCIUS; S/vanillamencius/Server.scala): one step of the n
 * co-located servers on device-resident buffers, with the same results as fpx_vm_client_request_dev (:767-829),
 * fpx_vm_phase2a_dev (:1001-1082), fpx_proxyleader_phase2b_dev (:1084-1142), fpx_replica_chosen_last_dev and
 * fpx_chosen_watermark_dev in that order -- in three launches: the client requests at the owners (arm + own
 * vote), the Phase2a batch at the other servers (dense replies), and the tally with the servers' shared log
 * (executeLog's prefix, :641-690) and the watermark (+ the exchange store) riding in the same kernel. */
int fpx_vm_step_dev(fpx_engine* e, const fpx_p2a* d_req, int32_t n_req, const fpx_p2a* d_p2a, int32_t n_p2a,
                    fpx_p2b* d_reply, const fpx_p2b* d_p2b, int32_t n_p2b, fpx_chosen* d_out_chosen, int32_t* d_watermark);
int fpx_step_kernel_ms(fpx_engine* e, int32_t ring_slot, float* acceptor_ms, float* tally_ms);
int fpx_step_arm_ms(fpx_engine* e, int32_t ring_slot, float* arm_ms);   /* the arm kernel of the same step */

/* ---- EPaxos, the execution side (SURVEY.md 8(f) rank 4) ----------------------------------------------
 * Top-1 conflict index: KeyValueStore.typedTopKConflictIndex(k = 1), S/statemachine/KeyValueStore.scala:219-302,
 * consulted by epaxos.Replica.computeSequenceNumberAndDependencies (S/epaxos/Replica.scala:569-600).  Keys are
 * caller-assigned int32 ids of the reference's string keys (INT32_MIN is reserved).  One batch = commands in
 * delivery order; command i is instance (leader[i], id[i]), a set (is_set[i] != 0) or a get, on the keys
 * keys[key_off[i] .. key_off[i+1]).  mode 0: for every command getTopOneConflicts (it sees every earlier
 * command of the batch and every earlier batch), then put (:1252, :1274); mode 1: put only; mode 2: query only.
 * deps_out[i * num_leaders + L] = the TopOne watermark of leader column L (largest conflicting id + 1, 0 = none);
 * a command without keys conflicts with the snapshots only.  FPX_ERR_OVERFLOW_FULL: more distinct keys than
 * key_capacity (a power of two).  num_leaders <= 8. */
typedef struct fpx_conflict_index fpx_conflict_index;
int fpx_conflict_index_create(fpx_conflict_index** out, int32_t num_leaders, int32_t key_capacity, int32_t max_commands,
                              int32_t max_keys, int32_t device);
void fpx_conflict_index_destroy(fpx_conflict_index* c);
int fpx_conflict_index_put_snapshot(fpx_conflict_index* c, int32_t leader, int32_t id);
int fpx_conflict_index_batch(fpx_conflict_index* c, const int32_t* leader, const int32_t* id, const uint8_t* is_set,
                             const int32_t* key_off, const int32_t* keys, int32_t n_cmd, int32_t mode, int32_t* deps_out,
                             int64_t* err_index);
/* Dependency graph: depgraph.TarjanDependencyGraph, S/depgraph/TarjanDependencyGraph.scala:225-451.  Keys are
 * int32 in [0, key_capacity).  commit: a batch of (key, sequenceNumber, dependencies) in delivery order, CSR
 * dependencies deps[dep_off[i] .. dep_off[i+1]); a key that is already committed or executed is ignored (:230-234).
 * execute = executeByComponent(None): the executable keys (everything they transitively depend on is committed or
 * executed), as components in dependency order (a component after every component it depends on), each sorted by
 * (sequenceNumber, key); out_component_head[p] = 1 where a component starts.  The order among INDEPENDENT
 * components is (level, root key) -- the reference's is a hash map's iteration order (:343), its tests accept any.
 * blockers (optional, key_capacity bytes): 1 for every uncommitted key a committed one waits for. */
typedef struct fpx_depgraph fpx_depgraph;
int fpx_depgraph_create(fpx_depgraph** out, int32_t key_capacity, int32_t dep_pool_capacity, int32_t max_batch, int32_t device);
void fpx_depgraph_destroy(fpx_depgraph* g);
int fpx_depgraph_commit(fpx_depgraph* g, const int32_t* keys, const int32_t* seqs, const int32_t* dep_off, const int32_t* deps,
                        int32_t n, int64_t* err_index);
int fpx_depgraph_update_executed(fpx_depgraph* g, const int32_t* keys, int32_t n, int64_t* err_index);
int fpx_depgraph_execute(fpx_depgraph* g, int32_t* out_keys, uint8_t* out_component_head, int32_t* n_out, uint8_t* blockers);

/* One pipeline step from HOST buffers, asynchronous and double-buffered, for co-located roles on one GPU
 * (pinned host memory recommended).  fpx_step_submit enqueues: H2D of the Phase2a batch and of the Phase2b
 * batch on a copy stream; the acceptor batch; the arm batch -- arm == NULL arms from the Phase2a batch itself
 * (ProxyLeader.handlePhase2a ignores a key it already holds, S/multipaxos/ProxyLeader.scala:177-183, so arming
 * with every forwarded copy leaves the same state as arming once per slot); the tally with the replica's
 * handleChosen and the watermark; D2H of the Phase2b replies on a second copy stream while the tally runs.
 * fpx_step_wait completes the OLDEST submitted step: counts, watermark, error status, and the Chosen
 * stream's D2H (its length is known only then).  At most 2 steps may be in flight, so the H2D of step k+1
 * overlaps the kernels and the D2H of step k (full-duplex PCIe).  The output buffers of a step must stay
 * valid until its fpx_step_wait returns.  Same semantics and errors as the five separate host calls. */
int fpx_step_submit(fpx_engine* e, const fpx_p2a* arm, int32_t n_arm, const fpx_p2a* p2a, int32_t n_p2a,
                    const fpx_p2b* p2b, int32_t n_p2b, fpx_p2b* out_p2b, fpx_nack* out_nack, fpx_chosen* out_chosen);
int fpx_step_wait(fpx_engine* e, int32_t* n_out_p2b, int32_t* n_out_nack, int32_t* n_out_chosen, int32_t* watermark,
                  int64_t* err_index);

/* ---- the exchange of a sharded log (SURVEY.md 8(e)) -------------------------------------------------
 * P engines, one per GPU (one process per GPU, or several engines in one process), shard_index g of
 * shard_count P, each hold one residue class of ONE global log.  Replicas execute in slot order and stop
 * at the first hole (S/multipaxos/Replica.scala:397-402; S/mencius/Replica.scala:334-370), so the global
 * executable prefix is the minimum over the shards of each shard's first unchosen GLOBAL slot.  Every
 * engine owns a frontier table {epoch, frontier}[P] in its device memory.  Once a peer's table is
 * attached, the kernel that publishes this engine's watermark (fpx_chosen_watermark[_dev], fpx_step_dev)
 * also stores {epoch, watermark} into entry g of that table over NVLink: peer-mapped stores from inside
 * the kernel, an all-gather without a collective launch.  epoch = number of this engine's watermark
 * publications since fpx_create / fpx_reset (every shard publishes once per step).
 *   fpx_exchange_export   the IPC handle (cudaIpcMemHandle_t, FPX_EXCHANGE_HANDLE_BYTES) of this engine's table
 *   fpx_exchange_attach   open shard `shard`'s table from its exported handle (other process, other GPU)
 *   fpx_exchange_attach_local  same, for an engine of this process
 *   fpx_global_watermark[_dev]  waits on the device (bounded: FPX_ERR_EXCHANGE_TIMEOUT after timeout_ms)
 *                         until every shard's entry carries an epoch >= `epoch`, then returns the minimum;
 *                         frontiers (optional, [P]) receives every shard's entry. */
#define FPX_EXCHANGE_HANDLE_BYTES 64
#define FPX_MAX_SHARDS 64
int fpx_exchange_export(fpx_engine* e, void* handle);
int fpx_exchange_attach(fpx_engine* e, int32_t shard, const void* handle);
int fpx_exchange_attach_local(fpx_engine* e, int32_t shard, fpx_engine* peer);
uint32_t fpx_exchange_epoch(const fpx_engine* e);
int fpx_global_watermark_dev(fpx_engine* e, uint32_t epoch, int32_t timeout_ms, int32_t* d_out, int32_t* d_frontiers);
int fpx_global_watermark(fpx_engine* e, uint32_t epoch, int32_t timeout_ms, int32_t* out, int32_t* frontiers);

/* State is a ring of slot_capacity slots (per shard: its residue class).  fpx_retire_below slides the live
 * window [base, base + slot_capacity): every slot below `slot` must be chosen and executed (slot <= the last
 * published watermark, else FPX_ERR_INVALID_ARG); its proxy-leader row, vote cells and log entry are recycled
 * for the slots slot_capacity ahead, so a long-lived engine is bounded by the number of slots IN FLIGHT, not
 * by the length of the log (the reference's maps grow with the log; Replica's BufferMap.garbageCollect,
 * S/util/BufferMap.scala:94-115, is the same idea).  Afterwards a message for a retired slot meets what the
 * reference's would: an arm / vote / Chosen finds the key Done or the entry present and is ignored; a Phase2a
 * is answered (round compare, Phase2b or Nack) but the vote is not recorded -- Phase1b never reads below the
 * chosen watermark (Acceptor.scala:171-179).  Slots at or beyond base + slot_capacity are FPX_ERR_SLOT_RANGE.
 * Secondary (slot, round) keys of retired slots stay in the overflow table until fpx_reset.  Not offered for
 * FPX_VANILLA_MENCIUS (a retired ChosenEntry would have to answer with its value). */
int fpx_retire_below(fpx_engine* e, int32_t slot);

/* The engine's CUDA stream (a cudaStream_t) so a caller can order its own work
 * (events, NCCL collectives) with the engine's. */
void* fpx_stream(fpx_engine* e);
/* Several engines (slot-residue shards) may share one GPU, each on its own stream.  The
 * acceptor and tally kernels are persistent cooperative launches sized to fill the GPU
 * (SMs x resident CTAs), and a cooperative launch waits until its whole grid fits; capping
 * an engine at ctas_per_sm resident CTAs per SM lets the kernels of different engines run
 * side by side instead of one after the other.  0 restores the full grid. */
int fpx_set_coop_ctas_per_sm(fpx_engine* e, int32_t ctas_per_sm);
/* Kernels launched by this handle since creation (bench.py's gpu_launches). */
int64_t fpx_launch_count(const fpx_engine* e);

#ifdef __cplusplus
}
#endif
#endif /* FPX_H_ */
