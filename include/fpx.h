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
/* One message of the Mencius replica's mixed stream (fpx_mencius_replica_inbound): the slots
 * slot_start, slot_start + num_leader_groups, ... < slot_end get value_id.  Chosen(slot, v) is
 * {slot, slot + 1, v}, ChosenNoopRange(s, e) is {s, e, FPX_VALUE_NOOP}; reserved is ignored. */
typedef struct { int32_t slot_start, slot_end, value_id, reserved; } fpx_mencius_chosen;
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
  FPX_ERR_BATCH_ORDER = -12,       /* fpx_epaxos_*: batch contract E1/E2 violated (two messages
                                      of one instance / one (instance, replica) in one call).
                                      NOTHING of the call is applied (outputs unspecified):
                                      resubmit rows [0, err_index) and [err_index, n) as two
                                      calls.  fpx_vm_phase2a, fpx_mencius_replica_chosen_range:
                                      their batch contract violated; the call is HALF APPLIED,
                                      fatal like every other status (fpx_reset)           */
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
                                   slot after a leader change); power of two or 0.  The
                                   table is held twice (fpx_retire_below rebuilds it into
                                   the spare copy): 2 x capacity x (8 + 4 x row words)
                                   bytes; FPX_MENCIUS also holds its noop-range table
                                   of max(1024, capacity) keys twice                     */
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
 * and the coordinators' `phase2s`.  Skips are below; the servers' side of a
 * revocation's Phase 1 is the block after them.  Batch contract (checked, ->
 * FPX_ERR_BATCH_ORDER): at most one Phase2a per (slot, server) per call, because
 * the round compare is per log entry (:1016-1042), not per acceptor.  The key is
 * in the message, so a caller can always flush ahead of a repeat; a call that
 * returns the status is half applied and fatal like every other (fpx_reset).  */

/* Server.handleClientRequest, state part (:767-829): the coordinator in.dst (which
 * must own in.slot) votes for its own command -- log(slot) = PendingEntry(0, 0,
 * value) (:779) -- and opens phase2s(slot) with its own Phase2b (:818-825).
 * Value ids here and in fpx_vm_phase2a must not be FPX_VALUE_RAISED (INT32_MIN + 1), which marks
 * an entry raised by a revocation's Phase1a (fpx_vm_phase1a_wire); the hot path does not check it. */
int fpx_vm_client_request(fpx_engine* e, const fpx_p2a* in, int32_t n, int64_t* err_index);

/* Server.handlePhase2a (:1001-1082) at server in.dst.  DENSE replies, reply[i]
 * answers in[i]: {group = kind, acceptor = server, slot, round}:
 *   kind 0  Phase2b(server, slot, round)                 (:1077-1081)
 *   kind 1  Phase2Nack(slot, round = the entry's round)  (:1044-1051)
 *   kind 2  Chosen(slot, value in `round`)               (:1018-1027, entry already chosen)
 *   kind 3  {3, server, slot, 0}: the slot was retired by fpx_retire_below.  The reference answers
 *           Chosen(slot, value) (:1016-1025), but the engine no longer holds the value: it is the
 *           shared log's executed entry of the slot, which the caller holds.  This is the one reply
 *           that differs from the reference's; a server that had not learned the slot before it was
 *           retired would have answered Phase2b or Phase2Nack there, and gets kind 3 here as well.
 *   kind 4  Chosen(slot, value in `round`, isRevocation = true): the entry was chosen by a revocation
 *           (fpx_vm_choose with is_revocation = 1).  Without revocation, kind 4 never occurs. */
enum { FPX_VM_REPLY_PHASE2B = 0, FPX_VM_REPLY_NACK = 1, FPX_VM_REPLY_CHOSEN = 2, FPX_VM_REPLY_CHOSEN_RETIRED = 3,
       FPX_VM_REPLY_CHOSEN_REVOCATION = 4 };
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

/* ---- Vanilla Mencius revocation, the servers' side (protocol FPX_VANILLA_MENCIUS, shard_count 1; any other:
 * FPX_ERR_UNSUPPORTED) ----
 * Revocation keeps Mencius live after a server fails: another server (the revoker, round % n of a round >= n)
 * runs Phase 1 over the failed server's slots [start, stop) and fills them in.  Besides PendingEntry and
 * ChosenEntry an entry can now be VotelessEntry(round) or a PendingEntry whose round was raised above its
 * voteRound, and a ChosenEntry carries isRevocation.  FPX_VALUE_RAISED is a value id the engine reserves for
 * raised entries: a Phase2a must not carry it.  The revoker's fill-in and its Phase 2 are the caller's. */
#define FPX_VALUE_RAISED (INT32_MIN + 1)

/* Server.handleChosen -> choose(slot, value, isRevocation) (:1170-1197, :622-640) at server in.acceptor.  Record
 * fields: group = is_revocation (nonzero: true), acceptor = the learning server, slot, round = the value id.  A
 * decoder kind-7 row {slot, is_revocation, value_off, value_len} becomes {b, server, a, the caller's value id for
 * the span}.  fpx_vm_learn_chosen is this call with is_revocation = 0 (it does not read group).  A ChosenEntry learned both with and without
 * isRevocation keeps isRevocation = true (the reference keeps the last delivered; the value is the same). */
int fpx_vm_choose(fpx_engine* e, const fpx_p2b* in, int32_t n, int64_t* err_index);
int fpx_vm_choose_dev(fpx_engine* e, const fpx_p2b* d_in, int32_t n);

/* Read-only snapshot of server `server`'s entries at slots [first_slot, first_slot + n_slots), all live
 * (FPX_ERR_SLOT_RANGE otherwise): out[5 * k ..] = {kind (0 none, 1 VotelessEntry, 2 PendingEntry, 3 ChosenEntry),
 * round, voteRound (-1 for none and Voteless), value (Pending and Chosen), isRevocation (Chosen)}; 0 where a
 * kind has no such field. */
int fpx_vm_entries(fpx_engine* e, int32_t server, int32_t first_slot, int32_t n_slots, int32_t* out);

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
 * call must not cover a common slot (the call is then half applied: fatal, fpx_reset).  With shard_count > 1 "already in the log" is judged
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
/* Replica.handleChosen (S/mencius/Replica.scala:402-420) and handleChosenNoopRange (:464-486) for ONE batch of both,
 * in delivery order (fpx_mencius_chosen records, e.g. from fpx_wire_decode_mencius_replica_inbound).  Records
 * [0, *split) are applied exactly as the reference applies those messages one at a time: each record puts its value
 * into its slots until the first slot already in the log -- put before the call, retired by fpx_retire_below, or put
 * by an earlier record of the call -- and stops there.  A record of one slot is therefore handleChosen's
 * put-if-absent (the first Chosen of a slot wins), a record covering no slot changes nothing.  Records of two or more
 * slots ("ranges") are where the order matters, so *split is the smallest of
 *   (a) the index of the first range that shares a slot with an earlier range of the call (judged on the full
 *       extents: its stop would depend on how far the earlier one got),
 *   (b) the index of the first range past FPX_MAX_RANGE_BATCH,
 * and n.  Nothing at or past *split is applied: continue with in + *split (no refusal, nothing half applied).  A
 * range re-proposed after a leader change is what makes two ranges of one batch overlap, so a split is rare.
 * Statuses of the records before the split: FPX_ERR_SLOT_RANGE for 0 <= slot_start <= slot_end <= slot_capacity
 * broken (the lowest such index in *err_index; the other records are applied).  FPX_ERR_UNSUPPORTED unless
 * protocol == FPX_MENCIUS and shard_count == 1 (a sharded log keeps the _first / MIN / _fill path above).
 * n <= max_batch.  fpx_chosen_watermark afterwards is the first hole.  The _dev form runs on the engine's stream and
 * writes the split to d_split; its status is collected by fpx_sync. */
int fpx_mencius_replica_inbound(fpx_engine* e, const fpx_mencius_chosen* in, int32_t n, int32_t* split,
                                int64_t* err_index);
int fpx_mencius_replica_inbound_dev(fpx_engine* e, const fpx_mencius_chosen* d_in, int32_t n, int32_t* d_split);

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
 * FPX_MENCIUS the mencius shape is written ({acceptor_index, slot, round} under field 4).
 * out_capacity, for every encoder of this header: output that does not fit is refused with
 * FPX_ERR_INVALID_ARG at index 0.  Then nothing at or past out[out_capacity] is written, the host
 * forms leave the caller's out untouched, and the contents of a _dev form's d_out below
 * out_capacity are unspecified (the small-record encoders write the tiles that fit, the others
 * nothing).  The refusal latches nothing: the handle's next call runs as usual. */
int fpx_wire_encode_phase2b(fpx_engine* e, const fpx_p2b* in, int32_t n, uint8_t* out, int32_t out_capacity,
                            int32_t* offsets, int64_t* err_index);
int fpx_wire_encode_phase2b_dev(fpx_engine* e, const fpx_p2b* d_in, int32_t n, uint8_t* d_out, int32_t out_capacity,
                                int32_t* d_offsets);
/* LeaderInbound{nack{round}}; in[i].leader selects the destination and is not on the wire.  The member is
 * nack = 6 (S/multipaxos/MultiPaxos.proto:525-539), with protocol FPX_MENCIUS nack = 7
 * (S/mencius/Mencius.proto:322-337, where field 6 is leader_info_request_batcher). */
int fpx_wire_encode_nack(fpx_engine* e, const fpx_nack* in, int32_t n, uint8_t* out, int32_t out_capacity,
                         int32_t* offsets, int64_t* err_index);
/* ReplicaInbound{chosen{slot, command_batch_or_noop}}: the value bytes of value_id v are
 * arena[value_offsets[v] .. value_offsets[v+1]) (e.g. the Phase2a payloads the proxy leader
 * kept); value_id out of [0, num_values) -> FPX_ERR_INVALID_ARG with the record's index. */
int fpx_wire_encode_chosen(fpx_engine* e, const fpx_chosen* in, int32_t n, const uint8_t* arena,
                           const int32_t* value_offsets, int32_t num_values, uint8_t* out, int32_t out_capacity,
                           int32_t* offsets, int64_t* err_index);

/* ---- Wire codec of vanilla Mencius (protocol FPX_VANILLA_MENCIUS; any other: FPX_ERR_UNSUPPORTED) ----
 * S/vanillamencius/VanillaMencius.proto: ServerInbound :227-241 {client_request = 1, phase1a = 2, phase1b = 3,
 * phase2a = 4, phase2b = 5, skip = 6, chosen = 7, phase1_nack = 8, phase2_nack = 9}, CommandOrNoop :84-93
 * {command = 1, noop = 2}, ClientRequest :95-100, Phase2a :154-162, Skip :164-172, Phase2b :174-181, Chosen
 * :183-190 (isRevocation is a required bool), Phase2Nack :209-215.  Parsing rules, buffers, offsets[n+1] and
 * out_capacity as for the calls above; n (servers) = acceptors_per_group.
 *
 * Decode: kind[i] = the oneof member's field number (0: none); sender[i] = the message's server field
 * (Phase2a.sending_server, which handlePhase2a :1055 compares with the slot's owner; Phase2b / Skip
 * server_index), -1 for the other members.  out[i] per kind:
 *   1 client_request  {0, 0, value_off, value_len}: the whole `command` field, tag and length included.
 *                     Those bytes are CommandOrNoop().withCommand(command) (both carry Command as field 1):
 *                     the arena entry of the Phase2a the coordinator sends.
 *   4 phase2a         {slot, round, value_off, value_len}: the CommandOrNoop, never read
 *   5 phase2b         {0, server_index, slot, round}: the fpx_p2b fpx_proxyleader_phase2b takes
 *   6 skip            {server_index, start, stop, 0}: an fpx_vm_skip_rec once the caller sets server and own
 *   7 chosen          {slot, is_revocation (0 / 1), value_off, value_len}
 *   9 phase2_nack     {slot, round, 0, 0}
 *   2, 3, 8 and unknown members: {0, 0, body_off, body_len} for the host.
 * A missing required field (isRevocation and command_or_noop included), a second command_or_noop or
 * `command`, or a group wire type is FPX_ERR_WIRE at the message's index. */
int fpx_wire_decode_vm_server_inbound(fpx_engine* e, const uint8_t* bytes, const int32_t* offsets, int32_t n,
                                      int32_t* kind, fpx_wire_rec* out, int32_t* sender, int64_t* err_index);
int fpx_wire_decode_vm_server_inbound_dev(fpx_engine* e, const uint8_t* d_bytes, const int32_t* d_offsets, int32_t n,
                                          int32_t* d_kind, fpx_wire_rec* d_out, int32_t* d_sender);
/* Encoders: canonical ServerInbound bytes, one message per record.  Values: value_id v is the CommandOrNoop
 * arena[value_offsets[v] .. value_offsets[v+1]); FPX_VALUE_NOOP is CommandOrNoop{noop {}} (bytes 12 00); any
 * other value_id outside [0, num_values) is FPX_ERR_INVALID_ARG at that record.  isRevocation is written false
 * (18 00) except for reply kind 4.
 * _vm_replies: the dense reply stream of fpx_vm_phase2a[_dev] / fpx_vm_step_dev, by reply kind:
 *   0 phase2b{server_index = acceptor, slot, round}   1 phase2_nack{slot, round}
 *   2 chosen{slot, command_or_noop = the value in `round`, false}
 *   4 (FPX_VM_REPLY_CHOSEN_REVOCATION) chosen{slot, the value in `round`, true}
 *   3 (FPX_VM_REPLY_CHOSEN_RETIRED) a ZERO-LENGTH message: the engine no longer holds the retired slot's value;
 *     the caller, which holds the executed entry, sends that Chosen itself.
 *   Any other kind is FPX_ERR_INVALID_ARG at that record. */
int fpx_wire_encode_vm_replies(fpx_engine* e, const fpx_p2b* in, int32_t n, const uint8_t* arena,
                               const int32_t* value_offsets, int32_t num_values, uint8_t* out, int32_t out_capacity,
                               int32_t* offsets, int64_t* err_index);
int fpx_wire_encode_vm_replies_dev(fpx_engine* e, const fpx_p2b* d_in, int32_t n, const uint8_t* d_arena,
                                   const int32_t* d_value_offsets, int32_t num_values, uint8_t* d_out,
                                   int32_t out_capacity, int32_t* d_offsets);
/* chosen{slot, value, false} per tally output (handlePhase2b :1127-1135 sends it to every other server). */
int fpx_wire_encode_vm_chosen(fpx_engine* e, const fpx_chosen* in, int32_t n, const uint8_t* arena,
                              const int32_t* value_offsets, int32_t num_values, uint8_t* out, int32_t out_capacity,
                              int32_t* offsets, int64_t* err_index);
int fpx_wire_encode_vm_chosen_dev(fpx_engine* e, const fpx_chosen* d_in, int32_t n, const uint8_t* d_arena,
                                  const int32_t* d_value_offsets, int32_t num_values, uint8_t* d_out,
                                  int32_t out_capacity, int32_t* d_offsets);
/* phase2a{sending_server = slot mod n (in [0, n)), slot, round, value} per client-request record
 * (handleClientRequest :806-815); dst is not on the wire. */
int fpx_wire_encode_vm_phase2a(fpx_engine* e, const fpx_p2a* in, int32_t n, const uint8_t* arena,
                               const int32_t* value_offsets, int32_t num_values, uint8_t* out, int32_t out_capacity,
                               int32_t* offsets, int64_t* err_index);
int fpx_wire_encode_vm_phase2a_dev(fpx_engine* e, const fpx_p2a* d_in, int32_t n, const uint8_t* d_arena,
                                   const int32_t* d_value_offsets, int32_t num_values, uint8_t* d_out,
                                   int32_t out_capacity, int32_t* d_offsets);
/* skip{server_index = server, start, stop}; own is not on the wire. */
int fpx_wire_encode_vm_skip(fpx_engine* e, const fpx_vm_skip_rec* in, int32_t n, uint8_t* out, int32_t out_capacity,
                            int32_t* offsets, int64_t* err_index);
int fpx_wire_encode_vm_skip_dev(fpx_engine* e, const fpx_vm_skip_rec* d_in, int32_t n, uint8_t* d_out,
                                int32_t out_capacity, int32_t* d_offsets);

/* The servers' side of a revocation (see fpx_vm_choose above). */
/* Server.handlePhase1a (:831-911) from bytes.  kind[] / in[] are fpx_wire_decode_vm_server_inbound's rows of the
 * ServerInbound batch `bytes` (kind 2: {0, 0, body_off, body_len}) with in[i].a set by the caller to the receiving
 * server.  Values: the caller's CommandOrNoop arena as for the encoders above.  next_slot[n] (in / out) holds
 * every server's nextSlot, as for fpx_vm_skip.  Per server, in delivery order, each Phase1a{round, start, stop}:
 *   - if start mod n is the receiving server, the log fill of advanceWithSkips(stop - 1) first (as an own = 1
 *     fpx_vm_skip, FPX_ERR_CHECK_FAILED where a slot is not vacant); skips[i] = {server, old next_slot, new stop,
 *     1}, the range for the caller's skipSlots (slot_start == slot_stop: none), and next_slot advances;
 *   - the walk over start, start + n, ... < stop: no entry becomes VotelessEntry(round); a Voteless or Pending
 *     entry above the round stops the walk with ServerInbound{phase1_nack = 8 {start, stop, entry's round}} -- the
 *     entries before it stay raised; a PendingEntry adds PendingSlotInfo{voteRound, voteValue} and takes the round;
 *     a ChosenEntry adds ChosenSlotInfo{value, isRevocation};
 *   - otherwise the reply is ServerInbound{phase1b = 3 {server_index, round, start, stop, info...}}.
 * out / offsets[n + 1]: one reply per record, zero-length for any other kind.  Refused with nothing applied:
 * malformed bytes or a missing field (FPX_ERR_WIRE), a server out of range or a next_slot not of its server
 * (FPX_ERR_INVALID_ARG), a round outside [0, FPX_MAX_ROUND] (FPX_ERR_ROUND_RANGE), start < 0, a walked slot or a
 * slot of the fill that is retired or beyond the live window, or a next_slot past INT32_MAX (FPX_ERR_SLOT_RANGE;
 * the caller sizes slot_capacity to cover nextSlot + 2 beta).  Found only after the entries are raised (fatal,
 * like every half-applied call): a value id outside the arena in a reply (FPX_ERR_INVALID_ARG at that record) and
 * replies longer than out_capacity (FPX_ERR_INVALID_ARG at 0). */
int fpx_vm_phase1a_wire(fpx_engine* e, const uint8_t* bytes, int32_t n_bytes, const int32_t* kind,
                        const fpx_wire_rec* in, int32_t n, const uint8_t* arena, const int32_t* value_offsets,
                        int32_t num_values, int32_t* next_slot, uint8_t* out, int32_t out_capacity, int32_t* offsets,
                        fpx_vm_skip_rec* skips, int64_t* err_index);
/* device-pointer form: d_out, d_in and d_skips 16-byte aligned; synchronises once to size its scratch */
int fpx_vm_phase1a_wire_dev(fpx_engine* e, const uint8_t* d_bytes, int32_t n_bytes, const int32_t* d_kind,
                            const fpx_wire_rec* d_in, int32_t n, const uint8_t* d_arena, const int32_t* d_value_offsets,
                            int32_t num_values, int32_t* d_next_slot, uint8_t* d_out, int32_t out_capacity,
                            int32_t* d_offsets, fpx_vm_skip_rec* d_skips);

/* ---- Wire codec of Compartmentalized Mencius' noop ranges and replica (protocol FPX_MENCIUS; any other:
 * FPX_ERR_UNSUPPORTED) ----
 * S/mencius/Mencius.proto: Phase2bNoopRange :178-187, Chosen :189-195, ChosenNoopRange :197-203, ProxyLeaderInbound
 * :339-350, ReplicaInbound :363-371 {chosen = 1, chosen_noop_range = 2}.  Parsing rules, buffers, offsets[n+1] and
 * out_capacity as for the calls above.  The Mencius Chosen has MultiPaxos's shape: fpx_wire_encode_chosen writes it.
 *
 * Decode a batch of ReplicaInbound into the records fpx_mencius_replica_inbound applies, DENSE: row i answers
 * message i.  kind[i] = the member's field number.
 *   1 chosen             {slot, slot + 1, value_id_base + i, 0}; values[2i], values[2i+1] = {off, len} of
 *                        command_batch_or_noop in bytes (located, not parsed; a second one is FPX_ERR_WIRE)
 *   2 chosen_noop_range  {start, end, FPX_VALUE_NOOP, 0}
 *   0 no member          {0, 0, FPX_VALUE_NOOP, 0}, a row that covers no slot.  The reference's replica stops with
 *                        logger.fatal("Empty ReplicaInbound encountered."); that decision is the caller's, by kind.
 * values of the rows of kinds 0 and 2 are {0, 0}; a message that fails (FPX_ERR_WIRE) gets kind 0 and that row. */
int fpx_wire_decode_mencius_replica_inbound(fpx_engine* e, const uint8_t* bytes, const int32_t* offsets, int32_t n,
                                            int32_t value_id_base, int32_t* kind, fpx_mencius_chosen* recs,
                                            int32_t* values, int64_t* err_index);
int fpx_wire_decode_mencius_replica_inbound_dev(fpx_engine* e, const uint8_t* d_bytes, const int32_t* d_offsets,
                                                int32_t n, int32_t value_id_base, int32_t* d_kind,
                                                fpx_mencius_chosen* d_recs, int32_t* d_values);
/* The acceptor's replies of fpx_mencius_acceptor_noop_range: ProxyLeaderInbound{phase2b_noop_range = 5
 * {acceptor_group_index = (dst >> 16) % num_acceptor_groups, acceptor_index = dst & 0xffff, start, end, round}}.
 * Decoding it with FPX_WIRE_MENCIUS_PROXYLEADER_INBOUND gives back the record. */
int fpx_wire_encode_mencius_phase2b_range(fpx_engine* e, const fpx_p2b_range* in, int32_t n, uint8_t* out,
                                          int32_t out_capacity, int32_t* offsets, int64_t* err_index);
int fpx_wire_encode_mencius_phase2b_range_dev(fpx_engine* e, const fpx_p2b_range* d_in, int32_t n, uint8_t* d_out,
                                              int32_t out_capacity, int32_t* d_offsets);
/* The proxy leader's ChosenNoopRange of fpx_mencius_range_phase2b, sent to every replica:
 * ReplicaInbound{chosen_noop_range = 2 {start, end}}. */
int fpx_wire_encode_mencius_chosen_range(fpx_engine* e, const fpx_chosen_range* in, int32_t n, uint8_t* out,
                                         int32_t out_capacity, int32_t* offsets, int64_t* err_index);
int fpx_wire_encode_mencius_chosen_range_dev(fpx_engine* e, const fpx_chosen_range* d_in, int32_t n, uint8_t* d_out,
                                             int32_t out_capacity, int32_t* d_offsets);

/* ---- EPaxos replica (S/epaxos/Replica.scala) ------------------------------
 * One fpx_epaxos handle = one replica's cmdLog (:298-330) and leaderStates
 * (:347-386) for n = 2f+1 replicas, instances (replicaIndex, instanceNumber <
 * instances_per_replica).  Messages are rows of int32 of fixed width (n = 2f+1);
 * dependency sets are DENSE watermark vectors of n ints (InstancePrefixSet with
 * empty `values`, the topKDependencies = 1 default, Replica.scala:95); general
 * sets go through fpx_depset_union.  Ballot = (ordering, replicaIndex), tuple
 * order (S/epaxos/BallotHelpers.scala:11-21).  Replies / events are DENSE: row i
 * of the output belongs to message i of the input (kind 0 = nothing to send).
 * Batch contract, checked on the device AHEAD of the handlers (FPX_ERR_BATCH_ORDER):
 *   E1 lead / preaccept / accept / commit / prepare_phase / prepare /
 *      slow_path_timer: at most one message per instance per call;
 *   E2 preacceptok / acceptok / prepareok: at most one message per (instance,
 *      replica) per call; a PreAcceptOk / PrepareOk that replaces an earlier response
 *      of its replica with DIFFERENT content must be the only message of its instance
 *      in the call.  (Only responses the handler counts take part: the instance is
 *      led in that phase, in the response's ballot.)
 * A batch in any order is legal for the reference, so this status is not fatal: a
 * call that returns it -- or FPX_ERR_SLOT_RANGE / FPX_ERR_ROUND_RANGE -- has applied
 * NOTHING (cmdLog, leader states and largestBallot are as before the call; its
 * outputs are unspecified).  err_index is the later message of the first colliding
 * pair: resubmit rows [0, err_index) and [err_index, n) as two calls (the second may
 * be refused again, further in).  This guarantee holds for fpx_epaxos_* only.
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
enum { FPX_EP_EV_RECOVER_TIMER = 1 };   /* fpx_epaxos_nack */
enum { FPX_EP_EV_RESTART = 1 };         /* fpx_epaxos_prepareok */
enum { FPX_EP_LEADER_NONE = 0, FPX_EP_LEADER_PREACCEPTING = 1, FPX_EP_LEADER_ACCEPTING = 2, FPX_EP_LEADER_PREPARING = 3 };
enum { FPX_EP_STATUS_NOT_SEEN = 0, FPX_EP_STATUS_PRE_ACCEPTED = 1, FPX_EP_STATUS_ACCEPTED = 2 };

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
 * cudaStream_t); status and first offending index are collected by fpx_epaxos_sync.  A refusal (see the batch
 * contract above) stands until it is collected: the calls queued behind the refused one apply nothing either,
 * fpx_epaxos_sync reports the refused call's status and index, and the caller resubmits all of them. */
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

/* Recovery and the timer-driven transitions (Replica.scala:969-1078, 1567-1869).  Same conventions as above:
 * dense replies / events, first offending index, a _dev form asynchronous on fpx_epaxos_stream.  The caller keeps
 * the timers, thrifty recipient choice, the conflict index and execution.  Wherever these calls read
 * largestBallot they read max(largestBallot, (0, replica_index)), the reference's initial value (:458); the
 * stored value starts at (-1, -1), as the existing handlers expect.
 *
 * handleCommit -> commit, :1567-1575, :815-831.  in rows of 4+n ints: {inst_replica, inst_number, value_id, seq,
 * deps[n]}.  Writes CommittedEntry whatever the entry held, even an earlier Committed one, and drops the
 * instance's leader state of any kind.  No reply.  Batch contract E1.  The caller still updates the conflict
 * index (fpx_conflict_index_batch mode PUT) and commits to the dependency graph. */
int fpx_epaxos_commit(fpx_epaxos* e, const int32_t* in, int32_t n_rec, int64_t* err_index);
/* handleNack, :1577-1630.  in rows of 4 ints: {inst_replica, inst_number, lb_ord, lb_rep}; event rows of 1 int:
 * RECOVER_TIMER when this replica leads the instance (any leader kind, Preparing included) in a ballot below the
 * Nack's: (re)arm the recoverInstance timer.  Every Nack raises largestBallot.  No batch contract. */
int fpx_epaxos_nack(fpx_epaxos* e, const int32_t* in, int32_t n_rec, int32_t* event, int64_t* err_index);
/* transitionToPreparePhase, :969-996 (the recoverInstance timer fired).  in rows of 2 ints: {inst_replica,
 * inst_number}; out rows of 2 ints: {b_ord, b_rep}, the ballot of the Prepare to send, to f other replicas and
 * to this one.  Row i gets (L + 1 + i, replica_index), L = the floored largestBallot's ordering at call start;
 * each row raises largestBallot.  The leader state becomes Preparing with no responses; cmdLog is untouched.
 * An ordering past FPX_MAX_ROUND is FPX_ERR_ROUND_RANGE.  Batch contract E1. */
int fpx_epaxos_prepare_phase(fpx_epaxos* e, const int32_t* in, int32_t n_rec, int32_t* ballot, int64_t* err_index);
/* handlePrepare, :1632-1757.  in rows of 4 ints: {inst_replica, inst_number, b_ord, b_rep}; reply rows of 9+n
 * ints: {kind, yielded, b_ord, b_rep, vb_ord, vb_rep, status, value_id, seq, deps[n]}, status 0 NotSeen 1
 * PreAccepted 2 Accepted.  kind OK = PrepareOk in the Prepare's ballot (NotSeen with a (-1, -1) vote ballot and
 * no triple for an absent or NoCommand entry), NACK = Nack(largestBallot) in b, COMMIT = Commit(triple); fields a
 * reply does not carry are (-1, -1) and 0.  Every Prepare raises largestBallot BEFORE the Nack is built (:1637,
 * :1652): the Nack of message i carries the max over the handle's value before the call and messages 0..i.
 * yielded = 1 when the Prepare's ballot exceeded this replica's leader ballot (any kind) and the leader state was
 * dropped -- also for a Nacked Prepare; stop that instance's timers.  Batch contract E1. */
int fpx_epaxos_prepare(fpx_epaxos* e, const int32_t* in, int32_t n_rec, int32_t* reply, int64_t* err_index);
/* handlePrepareOk, :1759-1869.  in rows of 9 ints: {inst_replica, inst_number, b_ord, b_rep, from_replica,
 * vb_ord, vb_rep, status, value_id} (a PrepareOk's seq and deps are not inputs: no reachable branch reads them);
 * event rows of 4 ints: {kind, b_ord, b_rep, value_id}.  Counted only while the leader state is Preparing in
 * that ballot; a larger ballot is FPX_ERR_CHECK_FAILED (logger.checkLt, :1792).  At the delivery that completes
 * f+1 responses: among those with the maximum vote ballot, the PreAccepted one of the lowest replica index gives
 * value_id, else FPX_VALUE_NOOP; kind RESTART, and the instance is led by nobody until the caller runs the
 * conflict index (mode 0) and fpx_epaxos_lead with avoid_fast_path = 1 in {b_ord, b_rep} -- which it must do
 * before its next call that touches these instances (transitionToPreAcceptPhase, :1856-1867).  An Accepted
 * response is never re-accepted and the fast-path candidates are never taken: both branches are unreachable in
 * the reference (:1813, :1836) and stay so.  Batch contract E2. */
int fpx_epaxos_prepareok(fpx_epaxos* e, const int32_t* in, int32_t n_rec, int32_t* event, int64_t* err_index);
/* The defaultToSlowPath timer fired (:1015-1036) -> preAcceptingSlowPath (:796-813).  in rows of 4 ints:
 * {inst_replica, inst_number, b_ord, b_rep} (the ballot the timer was armed in); event rows as PreAcceptOk's:
 * SLOW_ACCEPT {seq, deps} over every answer the leader holds, when it is still PreAccepting in that ballot with the
 * timer armed by an earlier TIMER event; NONE otherwise (the reference would have stopped the timer).  E1. */
int fpx_epaxos_slow_path_timer(fpx_epaxos* e, const int32_t* in, int32_t n_rec, int32_t* event, int64_t* err_index);
int fpx_epaxos_commit_dev(fpx_epaxos* e, const int32_t* d_in, int32_t n_rec);
int fpx_epaxos_nack_dev(fpx_epaxos* e, const int32_t* d_in, int32_t n_rec, int32_t* d_event);
int fpx_epaxos_prepare_phase_dev(fpx_epaxos* e, const int32_t* d_in, int32_t n_rec, int32_t* d_ballot);
int fpx_epaxos_prepare_dev(fpx_epaxos* e, const int32_t* d_in, int32_t n_rec, int32_t* d_reply);
int fpx_epaxos_prepareok_dev(fpx_epaxos* e, const int32_t* d_in, int32_t n_rec, int32_t* d_event);
int fpx_epaxos_slow_path_timer_dev(fpx_epaxos* e, const int32_t* d_in, int32_t n_rec, int32_t* d_event);

/* read-back: out[7+n] = {kind, b_ord, b_rep, vb_ord, vb_rep, value_id, seq, deps[n]},
 * kind 0 none 1 NoCommand 2 PreAccepted 3 Accepted 4 Committed; *leader_kind 0 none 1
 * PreAccepting 2 Accepting 3 Preparing; largest_ballot[2] (as stored: (-1, -1) before any ballot) */
/* device time (ms, CUDA events on the handle's stream) of the kernels of the last
 * fpx_epaxos_* call, without its host<->device copies */
float fpx_epaxos_last_kernel_ms(fpx_epaxos* e);
int fpx_epaxos_entry(fpx_epaxos* e, int32_t inst_replica, int32_t inst_number, int32_t* out,
                     int32_t* leader_kind, int32_t* largest_ballot);

/* ---- Wire codec of EPaxos: ReplicaInbound bytes -> handler rows, on the handle's device and stream ----------
 * S/epaxos/EPaxos.proto: ReplicaInbound :220-235 {client_request = 1, pre_accept = 2, pre_accept_ok = 3, accept = 4,
 * accept_ok = 5, commit = 6, prepare = 7, prepare_ok = 8, nack = 9}; Instance :35-41, Ballot :46-52, Command :61-78,
 * CommandOrNoop :80-88 {command = 1, noop = 2}, CommandStatus :91-95, InstancePrefixSetProto :97-103
 * {numReplicas = 1, repeated int_prefix_set = 2}, S/compact/IntPrefixSet.proto IntPrefixSetProto {watermark = 1,
 * repeated value = 2}.  Batches, offsets[n+1], alignment and the parsing rules as for the codec above, and:
 *   - nested messages are parsed as protobuf-java's mergeFrom builds them: a member, Instance or Ballot given
 *     again merges into the earlier one (a later scalar wins, a field the second copy lacks keeps its value);
 *     another member starts afresh.  `required` is checked at every level of the message that results (Command's
 *     four fields included).  A missing one is FPX_ERR_WIRE at the message's index;
 *   - `value` is accepted packed and unpacked;
 *   - a second command_or_noop (or ClientRequest.command) is FPX_ERR_WIRE, as for vanilla Mencius;
 *   - a dependency set the handle cannot hold -- numReplicas != n, or a count of int_prefix_set entries != n (a
 *     second `dependencies` concatenates its entries) -- and a PrepareOk status outside {0, 1, 2} are
 *     FPX_ERR_UNSUPPORTED at that message: scalapb would parse them.
 * A message that fails stands like a refused batch (see the batch contract above): the fpx_epaxos_*_dev calls
 * queued behind it apply nothing, and fpx_epaxos_sync reports the status and the first failing index.
 *
 * Decode: kind[i] = the member's field number (0: none, or the message failed); rows of 12+n ints
 *   {inst_replica, inst_number, b_ord, b_rep, replica_index, vb_ord, vb_rep, status, value_id, seq, flags,
 *    overflow, deps[n]}
 * Nack's largest_ballot fills b_ord / b_rep.  A pair the message does not carry is (-1, -1), any other column 0
 * (fpx_epaxos_prepare's convention), value_id -1.  value_id = value_id_base + i for a message carrying a Command
 * (a CommandOrNoop whose last member is not noop), FPX_VALUE_NOOP for a noop, -1 without a CommandOrNoop.  flags
 * bit 0: a PrepareOk carries all of its optional command_or_noop, sequence_number and dependencies.  overflow =
 * number of `value` entries over the message's sets; deps = the n watermarks.  values[i] = {off, len}: the
 * CommandOrNoop's bytes in the batch ({0, 0} without one); for a ClientRequest the whole `command` field, tag and
 * length included, which are the bytes of CommandOrNoop().withCommand(command). */
enum { FPX_EP_CALL_LEAD = 0, FPX_EP_CALL_PREACCEPT = 1, FPX_EP_CALL_ACCEPT = 2, FPX_EP_CALL_PREACCEPTOK = 3,
       FPX_EP_CALL_ACCEPTOK = 4, FPX_EP_CALL_COMMIT = 5, FPX_EP_CALL_NACK = 6, FPX_EP_CALL_PREPARE_PHASE = 7,
       FPX_EP_CALL_PREPARE = 8, FPX_EP_CALL_PREPAREOK = 9, FPX_EP_CALL_SLOW_PATH_TIMER = 10 };
int fpx_epaxos_wire_decode(fpx_epaxos* e, const uint8_t* bytes, const int32_t* offsets, int32_t n,
                           int32_t value_id_base, int32_t* kind, int32_t* rows, int32_t* values, int64_t* err_index);
int fpx_epaxos_wire_decode_dev(fpx_epaxos* e, const uint8_t* d_bytes, const int32_t* d_offsets, int32_t n,
                               int32_t value_id_base, int32_t* d_kind, int32_t* d_rows, int32_t* d_values);
/* Pack: decoded rows [first, first+count) of a batch (kind and rows are the whole batch's arrays) -> the input
 * rows of one handler call (FPX_EP_CALL_*): preaccept 6+2n (local_deps, count rows of n ints -- the conflict
 * index's answers -- fill its local columns, zeros if null), accept 6+n, preacceptok 6+n, acceptok 6, commit 4+n,
 * nack 4, prepare 4, prepareok 9 (value_id 0 without the triple, as fpx_epaxos_prepare writes).  A row of another
 * kind is FPX_ERR_INVALID_ARG; a preaccept, accept, preacceptok or commit row with overflow > 0 is
 * FPX_ERR_UNSUPPORTED (fpx_epaxos_preaccept_sets' rule: parse that set on the host, union with fpx_depset_union).
 * Error indices are the batch's (first + j); a failing row refuses like a failing message.  Any other call is
 * FPX_ERR_INVALID_ARG. */
int fpx_epaxos_wire_pack(fpx_epaxos* e, int32_t call, const int32_t* kind, const int32_t* rows, int32_t first,
                         int32_t count, const int32_t* local_deps, int32_t* out, int64_t* err_index);
int fpx_epaxos_wire_pack_dev(fpx_epaxos* e, int32_t call, const int32_t* d_kind, const int32_t* d_rows, int32_t first,
                             int32_t count, const int32_t* d_local_deps, int32_t* d_out);
/* Encode: one canonical ReplicaInbound per record of a handler call -- `in` = the call's input rows, `out_rows` =
 * its replies / events / ballots (unused for lead) -- fields in number order, required fields always, optional ones
 * when present; a record with nothing to send is a ZERO-LENGTH message.  Per call (Replica.scala):
 *   lead              PreAccept{instance, ballot, value, seq, deps} (:697-706)
 *   preaccept         OK PreAcceptOk{instance, reply ballot, replica_index = this replica, seq, deps} (:1279-1288);
 *                     NACK Nack{instance, largest_ballot}; COMMIT Commit{instance, value, seq, deps} (:1226-1233)
 *   accept            OK AcceptOk{instance, ballot, replica_index}; NACK; COMMIT (:1455-1510)
 *   preacceptok,      FAST_COMMIT / COMMIT Commit (:834-845); SLOW_ACCEPT Accept{instance, the row's ballot, value,
 *   slow_path_timer   seq, deps} (:766-774); TIMER / NONE nothing
 *   acceptok          COMMIT Commit
 *   prepare_phase     Prepare{instance, the returned ballot}
 *   prepare           OK PrepareOk{ballot, instance, replica_index, vote_ballot, status, and command_or_noop,
 *                     sequence_number, dependencies only when status != NotSeen} (:1655-1744); NACK; COMMIT (:1748-1755)
 * commit, nack and prepareok send nothing: FPX_ERR_INVALID_ARG.  Values as in the vanilla Mencius encoders (value_id v
 * = arena[value_offsets[v] .. value_offsets[v+1]), FPX_VALUE_NOOP = 12 00, anything else FPX_ERR_INVALID_ARG at the
 * record, as is a reply kind the call does not produce).  Dependency sets are written dense: numReplicas = n and n
 * {watermark} entries (InstancePrefixSet.toProto of an empty-`values` set).  The Commit replies of preaccept and
 * accept and the Commit / Accept of the events carry no value_id in their rows: the encoder reads the instance's
 * value_id from the handle's cmdLog.  So encode BEFORE the next call that rewrites those instances; a _dev encode
 * queued right after its handler on the handle's stream reads that handler's result.  Behind a refused call the
 * _dev encode writes nothing. */
int fpx_epaxos_wire_encode(fpx_epaxos* e, int32_t call, const int32_t* in, const int32_t* out_rows, int32_t n,
                           const uint8_t* arena, const int32_t* value_offsets, int32_t num_values, uint8_t* out,
                           int32_t out_capacity, int32_t* offsets, int64_t* err_index);
int fpx_epaxos_wire_encode_dev(fpx_epaxos* e, int32_t call, const int32_t* d_in, const int32_t* d_out_rows, int32_t n,
                               const uint8_t* d_arena, const int32_t* d_value_offsets, int32_t num_values, uint8_t* d_out,
                               int32_t out_capacity, int32_t* d_offsets);

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
/* The same graph specialised to EPaxos instances with dense InstancePrefixSet dependencies (Replica.scala:864-886):
 * instance (c, j), c < n_replicas <= 7, j < instances_per_replica, depends on every (c', j') with j' < deps[c'],
 * except itself (subtractOne, Replica.scala:582): deps[c] > j is a hole, never a self-dependency.  No edge is
 * materialised; execute runs in O(log(n * instances_per_replica)) launches (DESIGN §6b).
 * commit: rows of 4+n ints, the layout of fpx_epaxos_commit's input: {inst_replica, inst_number, value_id (ignored),
 * seq, deps[n]}.  An instance already committed or executed is ignored; within a batch the first record of an
 * instance wins; an instance outside the handle is FPX_ERR_SLOT_RANGE at its record and nothing of the batch is
 * applied.  A watermark above instances_per_replica names instances that can never be committed: the vertex is
 * never executable.  commit_dev: the same rows in device memory, asynchronous on fpx_epaxos_graph_stream, the
 * error collected by fpx_epaxos_graph_sync.
 * update_executed: updateExecuted of every (c, j < watermark[c]).
 * execute = executeByComponent(None): out rows {inst_replica, inst_number} of the executable instances, as
 * strongly connected components in dependency order, each sorted by (seq, replica, number); out_component_head[p]
 * = 1 where a component starts.  Components are ordered by (sum of the closure vector, ...) (DESIGN §6b).  out
 * holds 2 * n * instances_per_replica ints, out_component_head n * instances_per_replica bytes.  blockers
 * (optional, n * instances_per_replica bytes, index c * instances_per_replica + j): 1 for every absent instance
 * that a committed, unexecuted instance names.  The executables are marked executed. */
typedef struct fpx_epaxos_graph fpx_epaxos_graph;
int fpx_epaxos_graph_create(fpx_epaxos_graph** out, int32_t n_replicas, int32_t instances_per_replica, int32_t max_batch,
                            int32_t device);
void fpx_epaxos_graph_destroy(fpx_epaxos_graph* g);
int fpx_epaxos_graph_commit(fpx_epaxos_graph* g, const int32_t* in, int32_t n_rec, int64_t* err_index);
int fpx_epaxos_graph_commit_dev(fpx_epaxos_graph* g, const int32_t* d_in, int32_t n_rec);
int fpx_epaxos_graph_sync(fpx_epaxos_graph* g, int64_t* err_index);
void* fpx_epaxos_graph_stream(fpx_epaxos_graph* g);
int fpx_epaxos_graph_update_executed(fpx_epaxos_graph* g, const int32_t* watermark);
int fpx_epaxos_graph_execute(fpx_epaxos_graph* g, int32_t* out, uint8_t* out_component_head, int32_t* n_out,
                             uint8_t* blockers);
/* device time (ms, CUDA events) of the kernels of the last commit or execute, without host round trips */
float fpx_epaxos_graph_last_kernel_ms(fpx_epaxos_graph* g);

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
 * Secondary (slot, round) keys of retired slots leave the overflow table, so an engine survives any number of
 * leader changes; the table is rebuilt only while it holds keys, otherwise a retire is one kernel launch.
 * FPX_MENCIUS: a Phase2aNoopRange key leaves its table once the range lies below base_local * shard_count
 * (every slot of the range that this shard holds is retired); a later arm of such a range is ignored and not
 * armed again, a later Phase2bNoopRange is ignored like one for a Done key.  Ranges that reach into the live
 * window keep their key.
 * FPX_VANILLA_MENCIUS: every server's entry of a retired slot counts as a ChosenEntry whose value the engine
 * no longer holds.  A Phase2a gets reply kind 3 (FPX_VM_REPLY_CHOSEN_RETIRED, see fpx_vm_phase2a); a Phase2b,
 * fpx_vm_learn_chosen and an own = 0 skip are ignored; an own = 1 skip is FPX_ERR_CHECK_FAILED (the slot is
 * not vacant); a client request is ignored (the reference's check(!log.contains) drops a duplicate). */
int fpx_retire_below(fpx_engine* e, int32_t slot);

/* ---- MultiPaxos linearizable reads (S/multipaxos/MultiPaxos.proto:36-115) ---------------------------------
 * A read learns a slot from a read quorum of acceptors, then a replica answers it once its log has executed
 * that slot.  One fpx_reads handle holds one of the two read-quorum tallies (the Client's or a ReadBatcher's)
 * and one replica's deferred reads, on the device, stream and quorum geometry of a FPX_MULTIPAXOS engine.  Once
 * that engine is destroyed, fpx_reads_destroy is the only call the handle takes.
 *
 * The acceptor side needs no entry point.  Acceptor.handleMaxSlotRequest / handleBatchMaxSlotRequest
 * (S/multipaxos/Acceptor.scala:222-254) answer {groupIndex, index, maxVotedSlot}; a MaxSlotRequest is a batch
 * boundary of its acceptor's Phase2a stream, and fpx_snapshot_acceptor(..., n_slots = 0) at that boundary
 * returns the maxVotedSlot every request queued there is answered with.
 * Not reproduced: the unsafeReadAtI and unsafeReadAtFirstSlot options (Client.scala:892-898), the
 * state-machine execution of a read (the caller runs the read right after log entry after_slot), and the
 * ReadReplyBatch fan-out to a ProxyReplica (Replica.scala:369-390); all stay with the caller.
 *
 * kind FPX_READS_CLIENT: Client.handleMaxSlotReply (S/multipaxos/Client.scala:851-931).  Replies are keyed
 *   by (group, acceptor) (:877-879); the read completes at f+1 replies (:880), flexible: on Grid.isReadQuorum
 *   (:883-887); slot = max + numAcceptorGroups - 1, flexible: max (:892-898).
 * kind FPX_READS_READ_BATCHER: ReadBatcher.handleBatchMaxSlotReply (S/multipaxos/ReadBatcher.scala:568-623).
 *   Replies are keyed by acceptorIndex only, the group is ignored (:584); the read completes at f+1 replies
 *   even on a flexible config (:585); slot = max + numAcceptorGroups - 1 (:592-598, acceptors :207-211); the
 *   entry is removed on completion (:601).
 * A read is (key, id): key < key_capacity is the caller's handle for a Client pseudonym or a ReadBatcher id
 * slot, id the generation (clientId / readBatcherId).  Memory: key_capacity x (32 + 8 x voters) bytes,
 * voters = numAcceptorGroups x acceptors_per_group (Client) or acceptors_per_group (ReadBatcher). */
typedef struct fpx_reads fpx_reads;
enum { FPX_READS_CLIENT = 0, FPX_READS_READ_BATCHER = 1 };
typedef struct { int32_t key, id; } fpx_read_open;
/* MaxSlotReply / BatchMaxSlotReply (MultiPaxos.proto) with the read's key; voter = group<<16 | acceptor */
typedef struct { int32_t key, id, voter, slot; } fpx_max_slot_reply;
/* a completed read: the slot its ReadRequest carries */
typedef struct { int32_t key, id, slot, reserved; } fpx_read_slot;
/* ReadRequest / SequentialReadRequest {slot}; a *Batch form is one record per command with the batch's slot;
 * EventualReadRequest is slot = -1.  handle is the caller's id of the read. */
typedef struct { int32_t slot, handle; } fpx_read_request;
/* ReadReply.slot = reply_slot; after_slot = the last log entry executed before the read runs */
typedef struct { int32_t handle, reply_slot, after_slot, reserved; } fpx_read_reply;

int fpx_reads_create(fpx_reads** out, fpx_engine* e, int32_t kind, int32_t key_capacity, int32_t pending_capacity,
                     int32_t max_batch);
void fpx_reads_destroy(fpx_reads* r);
/* Client.readImpl (Client.scala:626-660): states(pseudonym) = MaxSlot(id, {}); ReadBatcher (ReadBatcher.scala:472):
 * batchMaxSlotReplies(id) = Map().  Opening an open key again replaces its read; the last record of a key in
 * the batch wins.  key outside [0, key_capacity): FPX_ERR_INVALID_ARG with its index, nothing applied. */
int fpx_reads_open(fpx_reads* r, const fpx_read_open* in, int32_t n, int64_t* err_index);
/* The tally of the handle's kind, replies in delivery order.  A reply whose key is not open, whose read is
 * complete, or whose id differs is ignored (Client.scala:858-874, ReadBatcher.scala:572-580), and so is a key
 * outside [0, key_capacity).  A second reply of a voter overwrites its first; the slot is the maximum over the
 * latest reply of each voter at the completing reply; slot arithmetic wraps like a JVM Int.  out receives
 * one record per read completed in the batch, ORDERED BY THE INDEX OF THE COMPLETING REPLY; capacity n.
 * A counted reply whose voter is no acceptor of the config is FPX_ERR_BAD_ACCEPTOR at its index: with the
 * flexible Client this is Grid.isReadQuorum's `require` (S/quorums/Grid.scala:36-39), elsewhere such a reply
 * cannot arrive.  The handle's read state after an error is unspecified, as the reference's actor has failed. */
int fpx_reads_max_slot_replies(fpx_reads* r, const fpx_max_slot_reply* in, int32_t n, fpx_read_slot* out,
                               int32_t* n_out, int64_t* err_index);
/* Replica.handleReadRequest / handleSequentialReadRequest / handleEventualReadRequest and their *Batch forms
 * (Replica.scala:629-689) -> handleDeferrableRead(s) (:463-529) against the handle's executed watermark W
 * (0 at creation).  slot < W: answered now, in delivery order, reply {handle, W - 1, W - 1, 0} (:521-527);
 * any other read waits in the pending pool (:468-478).  out receives the immediate replies; capacity n.
 * More pending reads than pending_capacity: FPX_ERR_OVERFLOW_FULL at the first deferred read that does not
 * fit, and nothing of the batch is applied (n_out = 0). */
int fpx_reads_replica(fpx_reads* r, const fpx_read_request* in, int32_t n, fpx_read_reply* out, int32_t* n_out,
                      int64_t* err_index);
/* executeLog (Replica.scala:394-413) up to watermark: W = watermark, and every pending read with slot < W
 * leaves, by slot and by arrival within a slot, as {handle, slot - 1, slot, 0}: it runs right after log entry
 * `slot`, and its ReadReply.slot is slot - 1 because processDeferredReads runs before executedWatermark += 1
 * (:405-413) -- a quirk of the reference, kept.  watermark < W: FPX_ERR_INVALID_ARG.  W is
 * fpx_chosen_watermark with one shard, fpx_global_watermark with several.  out capacity pending_capacity. */
int fpx_reads_advance(fpx_reads* r, int32_t watermark, fpx_read_reply* out, int32_t* n_out);
/* The same on DEVICE pointers, asynchronous on the engine's stream (fpx_stream); the status, the first
 * offending index and the output counts are collected by fpx_reads_sync.  fpx_reads_advance_dev reads the
 * watermark from d_watermark on the device, e.g. the one fpx_step_dev writes: no host round trip. */
int fpx_reads_max_slot_replies_dev(fpx_reads* r, const fpx_max_slot_reply* d_in, int32_t n, fpx_read_slot* d_out);
int fpx_reads_replica_dev(fpx_reads* r, const fpx_read_request* d_in, int32_t n, fpx_read_reply* d_out);
int fpx_reads_advance_dev(fpx_reads* r, const int32_t* d_watermark, fpx_read_reply* d_out);
typedef struct {
  int32_t status;       /* first (lowest record index) error of any call since the last sync */
  int32_t watermark;    /* the handle's W                                                     */
  int64_t err_index;
  int32_t n_slots;      /* of the last fpx_reads_max_slot_replies_dev                         */
  int32_t n_replies;    /* of the last fpx_reads_replica_dev                                  */
  int32_t n_released;   /* of the last fpx_reads_advance_dev                                  */
  int32_t n_pending;    /* reads waiting in the pool                                          */
} fpx_reads_sync_result;
int fpx_reads_sync(fpx_reads* r, fpx_reads_sync_result* out);

/* ---- Wire codec of the MultiPaxos replica and read path (S/multipaxos/MultiPaxos.proto) --------------------
 * ClientInbound :489-500, ReadBatcherInbound :513-523, AcceptorInbound :551-561, ReplicaInbound :563-576,
 * CommandId :188-196, Command :198-204, MaxSlotRequest / MaxSlotReply :316-331, BatchMaxSlotRequest /
 * BatchMaxSlotReply :333-349, the read requests :351-396.  Parsing rules, offsets[n+1] batches, 16-byte aligned
 * buffers of the _dev forms and canonical output as for the wire codec above.  A member given more than once,
 * a Command and a CommandId are merged as protobuf-java's mergeFrom builds them (have-bits accumulate, a later
 * scalar wins, a repeated field appends), and `required` is checked on the merged message at every level.  A
 * malformed message or a missing required field is FPX_ERR_WIRE at the message's index.  The _dev forms run on
 * the engine's stream; their status and first index are collected by fpx_sync (engine calls) or fpx_reads_sync
 * (fpx_reads calls).  The fpx_reads calls stage through their engine's buffers.
 *
 * fpx_wire_decode_replica_inbound (protocol FPX_MULTIPAXOS, else FPX_ERR_UNSUPPORTED): kind[i] = the member's
 * field number (0: none, no record).  Records only for the messages [0, split), where split is the index of the
 * first read message (kinds 2..7) that follows a Chosen in the batch, or n:
 *   1 chosen  -> chosen[k] = {slot, value_id_base + i}, dense in delivery order, and chosen_values[2k..2k+1] =
 *                {off, len} of the CommandBatchOrNoop (located, not parsed; a second one is FPX_ERR_WIRE).  The
 *                records go to fpx_replica_chosen[_dev] as they are.
 *   2..7      -> reads[k] = {slot, handle_base + k} per Command, dense in delivery order, a batch's Commands in
 *                wire order; read_commands[2k..2k+1] = {off, len} of the Command message (its body: what
 *                Command.parseFrom takes).  Eventual reads (4, 7) get slot = -1.  A second `command` in a
 *                read_request, sequential_read_request or eventual_read_request is FPX_ERR_WIRE (protobuf would
 *                merge the two Commands).  More records than reads_capacity: FPX_ERR_OVERFLOW_FULL at the first
 *                message whose Commands do not fit.
 * counts = {n_chosen, n_reads, split} (_dev: a device int32[3] written on the stream).  The order of the batch is
 * the reference's when the caller runs fpx_reads_replica(reads), fpx_replica_chosen(chosen), then
 * fpx_reads_advance(the new watermark), and continues with the messages from offsets + split (value_id_base and
 * handle_base advanced by what it has used).  After an error the records and counts are unspecified. */
int fpx_wire_decode_replica_inbound(fpx_engine* e, const uint8_t* bytes, const int32_t* offsets, int32_t n,
                                    int32_t value_id_base, int32_t handle_base, int32_t reads_capacity, int32_t* kind,
                                    fpx_chosen* chosen, int32_t* chosen_values, fpx_read_request* reads,
                                    int32_t* read_commands, int32_t* counts, int64_t* err_index);
int fpx_wire_decode_replica_inbound_dev(fpx_engine* e, const uint8_t* d_bytes, const int32_t* d_offsets, int32_t n,
                                        int32_t value_id_base, int32_t handle_base, int32_t reads_capacity,
                                        int32_t* d_kind, fpx_chosen* d_chosen, int32_t* d_chosen_values,
                                        fpx_read_request* d_reads, int32_t* d_read_commands, int32_t* d_counts);
/* The acceptor's answers (Acceptor.scala:222-254): kind[] and in[] as fpx_wire_decode_inbound(
 * FPX_WIRE_ACCEPTOR_INBOUND) writes them for the request batch bytes[0 .. n_bytes), with a = group << 16 |
 * acceptor and b = maxVotedSlot filled in by the caller (fpx_snapshot_acceptor(..., n_slots = 0) at the request's
 * batch boundary).  One message per record:
 *   3 max_slot_request       -> ClientInbound{max_slot_reply{command_id, group_index, acceptor_index, slot}}; the
 *                               request's CommandId merged and written canonically, client_address copied;
 *   4 batch_max_slot_request -> ReadBatcherInbound{batch_max_slot_reply{read_batcher_index, read_batcher_id,
 *                               acceptor_index, slot}};
 *   any other kind           -> a zero-length message.
 * A body that does not parse or lacks a required field is FPX_ERR_WIRE at its record; a voter that names no
 * acceptor of the config is FPX_ERR_INVALID_ARG. */
int fpx_wire_encode_max_slot_replies(fpx_engine* e, const uint8_t* bytes, int32_t n_bytes, const int32_t* kind,
                                     const fpx_wire_rec* in, int32_t n, uint8_t* out, int32_t out_capacity,
                                     int32_t* offsets, int64_t* err_index);
int fpx_wire_encode_max_slot_replies_dev(fpx_engine* e, const uint8_t* d_bytes, int32_t n_bytes, const int32_t* d_kind,
                                         const fpx_wire_rec* d_in, int32_t n, uint8_t* d_out, int32_t out_capacity,
                                         int32_t* d_offsets);
/* The acceptors' Phase 1 from bytes (Acceptor.handlePhase1a, S/multipaxos/Acceptor.scala:148-182), protocol
 * FPX_MULTIPAXOS with shard_count 1, else FPX_ERR_UNSUPPORTED.  kind[] and in[] as fpx_wire_decode_inbound(
 * FPX_WIRE_ACCEPTOR_INBOUND) writes them for the request batch bytes[0 .. n_bytes), with a = group << 16 | acceptor
 * filled in by the caller; n <= 65535.  One message per record; per acceptor, in delivery order:
 *   1 phase1a, round < the acceptor's round -> LeaderInbound{nack{round = the acceptor's round}};
 *   1 phase1a, otherwise                    -> round = phase1a.round and LeaderInbound{phase1b{group_index,
 *        acceptor_index, round, info*}}: one info {slot, vote_round, vote_value} per voted slot >= chosen_watermark,
 *        ascending; the vote's value_id v is arena[value_offsets[v] .. value_offsets[v+1]) (a CommandBatchOrNoop),
 *        FPX_VALUE_NOOP the Noop (12 00); any other value_id is FPX_ERR_INVALID_ARG at the record;
 *   any other kind                          -> a zero-length message, nothing changed (a Phase1a is a batch boundary
 *        of the Phase2a stream, SURVEY 8(g) rule 2).
 * A body that does not parse or lacks a required field is FPX_ERR_WIRE at its record, a voter that names no acceptor
 * FPX_ERR_INVALID_ARG, a chosen_watermark below the first slot the engine still holds after fpx_retire_below (whose
 * votes it no longer has) FPX_ERR_SLOT_RANGE; with any of these no round changes.  Afterwards the rounds are what
 * fpx_acceptor_phase1a would have left.  out_capacity as for the encoders above.  Both forms read the info count back
 * once (it sizes the encoder): the _dev form synchronises the engine's stream. */
int fpx_acceptor_phase1a_wire(fpx_engine* e, const uint8_t* bytes, int32_t n_bytes, const int32_t* kind,
                              const fpx_wire_rec* in, int32_t n, const uint8_t* arena, const int32_t* value_offsets,
                              int32_t num_values, uint8_t* out, int32_t out_capacity, int32_t* offsets,
                              int64_t* err_index);
int fpx_acceptor_phase1a_wire_dev(fpx_engine* e, const uint8_t* d_bytes, int32_t n_bytes, const int32_t* d_kind,
                                  const fpx_wire_rec* d_in, int32_t n, const uint8_t* d_arena,
                                  const int32_t* d_value_offsets, int32_t num_values, uint8_t* d_out,
                                  int32_t out_capacity, int32_t* d_offsets);
/* ---- The new leader's Phase 1 from bytes (Leader.handlePhase1b, S/multipaxos/Leader.scala:504-577) ---------------
 * Protocol FPX_MULTIPAXOS with shard_count 1, else FPX_ERR_UNSUPPORTED.  The call is stateless: the engine supplies the
 * geometry (f, groups, grid) and its stream, and holds no leader state.  bytes / offsets[n+1]: the LeaderInbound
 * messages (MultiPaxos.proto:525-539; Phase1b :263-271, Phase1bSlotInfo :254-261) received since Phase 1 began, in
 * delivery order; parsing rules as for the wire codec above.  The Phase1b's bodies and its info entries are parsed;
 * the body of any other member is skipped by length, not parsed; a phase1b member given again merges (info appends,
 * a later scalar wins), another member replaces it.  A second vote_value in one info is FPX_ERR_WIRE (protobuf would
 * merge the two CommandBatchOrNoops), like a second command_batch_or_noop above.  Per message, in delivery order:
 *   malformed bytes or a missing required field       -> FPX_ERR_WIRE at the message;
 *   not a phase1b                                      -> skipped;
 *   phase1b.round < round                              -> ignored (:517-525);
 *   phase1b.round > round                              -> FPX_ERR_CHECK_FAILED at the message (logger.checkLt);
 *   group_index / acceptor_index outside the config    -> FPX_ERR_BAD_ACCEPTOR at the message;
 *   else phase1bs(group)(acceptor) = the message (a later Phase1b of an acceptor replaces its earlier one); the quorum
 *   completes when every group holds f+1 acceptors (flexible: Grid.isReadQuorum over the holders).
 * result[0] = complete, the index of the completing message, or -1: then nothing is emitted and the caller calls again
 * with more messages.  Messages after `complete` are not read.  result[1] = max_slot, the largest info slot of the
 * Phase1bs held at completion (maxPhase1bSlot, -1 for none), result[2] = n_out = max(0, max_slot - chosen_watermark +
 * 1).  Record k of out is Phase2a{slot = chosen_watermark + k, round, safeValue(phase1bs(slot % num_acceptor_groups),
 * slot)} as {slot, round, value_id, -1}: value_id = value_id_base + k where a holder voted (spans[2k..2k+1] = {off, len}
 * of its vote_value in bytes), FPX_VALUE_NOOP where none did (spans {0, 0}).  safeValue takes the first info of the
 * slot in each Phase1b (info.find) and the highest vote_round; ties in vote_round, which correct acceptors never
 * produce, go to the lowest acceptor index (DESIGN.md §7, beside the EPaxos recovery tie rule).  The records go
 * to fpx_proxyleader_arm as they are.  More than out_capacity records: FPX_ERR_INVALID_ARG at `complete` and nothing
 * written.  chosen_watermark < 0: FPX_ERR_INVALID_ARG.  Unlike fpx_leader_safe_values this reads the Phase1bs, so on a
 * flexible grid it is the reference's fill-in exactly: one grid row per slot.  The call's device scratch is about
 * 2 x the batch's bytes (one entry per 8 bytes) plus out_capacity x acceptors_per_group x 4 bytes (the info.find
 * window, cleared on every call): out_capacity is best the largest window the caller expects, not a "no limit".
 * _dev: d_bytes holds n_bytes bytes (offsets[n] - offsets[0] beyond them is FPX_ERR_WIRE at the message that reaches
 * past them); d_result is a device int32[3] written on the stream; the status and first index are collected by
 * fpx_sync; d_spans is 8-byte aligned. */
int fpx_leader_phase1b_wire(fpx_engine* e, int32_t round, int32_t chosen_watermark, const uint8_t* bytes,
                            const int32_t* offsets, int32_t n, int32_t value_id_base, fpx_p2a* out, int32_t* spans,
                            int32_t out_capacity, int32_t* result, int64_t* err_index);
int fpx_leader_phase1b_wire_dev(fpx_engine* e, int32_t round, int32_t chosen_watermark, const uint8_t* d_bytes,
                                int32_t n_bytes, const int32_t* d_offsets, int32_t n, int32_t value_id_base,
                                fpx_p2a* d_out, int32_t* d_spans, int32_t out_capacity, int32_t* d_result);
/* ProxyLeaderInbound{phase2a{slot, round, command_batch_or_noop}} per fpx_p2a record (dst is not on the wire):
 * value_id v is bytes[spans[2k] .. spans[2k] + spans[2k+1]) for k = v - value_id_base in [0, num_spans), FPX_VALUE_NOOP
 * is CommandBatchOrNoop{noop {}} (12 00); anything else, or a span outside bytes[0 .. n_bytes), is FPX_ERR_INVALID_ARG
 * at the record.  With fpx_leader_phase1b_wire's output: the Phase1b batch as bytes, its spans and value_id_base.
 * Protocol FPX_MULTIPAXOS with shard_count 1, else FPX_ERR_UNSUPPORTED; out_capacity as for the encoders above. */
int fpx_wire_encode_phase2a(fpx_engine* e, const fpx_p2a* in, int32_t n, const uint8_t* bytes, int32_t n_bytes,
                            const int32_t* spans, int32_t num_spans, int32_t value_id_base, uint8_t* out,
                            int32_t out_capacity, int32_t* offsets, int64_t* err_index);
int fpx_wire_encode_phase2a_dev(fpx_engine* e, const fpx_p2a* d_in, int32_t n, const uint8_t* d_bytes, int32_t n_bytes,
                                const int32_t* d_spans, int32_t num_spans, int32_t value_id_base, uint8_t* d_out,
                                int32_t out_capacity, int32_t* d_offsets);
/* ---- Compartmentalized Mencius leader change from bytes (protocol FPX_MENCIUS, shard_count 1, else
 * FPX_ERR_UNSUPPORTED; the three MultiPaxos calls above refuse FPX_MENCIUS engines).  LG = num_leader_groups, AG =
 * num_acceptor_groups (per leader group); engine group lg * AG + ag is acceptor group ag of leader group lg.
 *
 * fpx_mencius_acceptor_phase1a_wire: Acceptor.handlePhase1a (S/mencius/Acceptor.scala:166-200), arguments and
 * refusals as fpx_acceptor_phase1a_wire.  kind[] and in[] as fpx_wire_decode_inbound(FPX_WIRE_MENCIUS_ACCEPTOR_INBOUND)
 * writes them (kind 1 = phase1a), a = engine_group << 16 | acceptor filled in by the caller.  Per acceptor, in delivery
 * order:
 *   1 phase1a, round < the acceptor's round -> LeaderInbound{nack = 7 {round = the acceptor's round}};
 *   1 phase1a, otherwise                    -> round = phase1a.round and LeaderInbound{phase1b = 1 {group_index =
 *        engine_group % AG, acceptor_index, round, info*}}: one info per voted slot >= chosen_watermark, ascending,
 *        Phase2aNoopRange votes included (states(slot) = State(round, Noop), :263-277);
 *   any other kind                          -> a zero-length message, nothing changed.
 * The acceptor holds the slots s = lg + LG * ag (mod LG * AG) only; they are read from the first one >= chosen_watermark
 * to the end of the live window (noop-range votes do not raise the max_voted_slot of fpx_snapshot_acceptor, so that
 * cannot bound the scan). */
int fpx_mencius_acceptor_phase1a_wire(fpx_engine* e, const uint8_t* bytes, int32_t n_bytes, const int32_t* kind,
                                      const fpx_wire_rec* in, int32_t n, const uint8_t* arena,
                                      const int32_t* value_offsets, int32_t num_values, uint8_t* out,
                                      int32_t out_capacity, int32_t* offsets, int64_t* err_index);
int fpx_mencius_acceptor_phase1a_wire_dev(fpx_engine* e, const uint8_t* d_bytes, int32_t n_bytes, const int32_t* d_kind,
                                          const fpx_wire_rec* d_in, int32_t n, const uint8_t* d_arena,
                                          const int32_t* d_value_offsets, int32_t num_values, uint8_t* d_out,
                                          int32_t out_capacity, int32_t* d_offsets);
/* fpx_mencius_leader_phase1b_wire: Leader.handlePhase1b (S/mencius/Leader.scala:582-659) of leader group
 * leader_group, stateless like fpx_leader_phase1b_wire: the caller passes the group's round, chosenWatermark and
 * recoverSlot (-1: the leader change was not started by a Recover; else the Recover's slot, :845-870) and the
 * LeaderInbound bytes (Mencius.proto:322-338, nine members: a recover or chosen_watermark member after a phase1b
 * replaces it) received since Phase 1 began.  leader_group outside [0, LG), recover_slot < -1 or chosen_watermark < 0:
 * FPX_ERR_INVALID_ARG.  Parsing and the per-message rules as for fpx_leader_phase1b_wire, with group_index in [0, AG)
 * (else FPX_ERR_BAD_ACCEPTOR); the quorum completes when every one of the group's AG acceptor groups holds f+1.
 * result = {complete, max_slot, n_out, next_slot}, {-1, -1, 0, -1} while incomplete.  At completion:
 *   max_slot  = max(maxPhase1bSlot over the held Phase1bs (-1 when empty), recover_slot); an info slot of another
 *               leader group counts here (and fails the check below) but is never re-proposed;
 *   max_slot != -1 and max_slot % LG != leader_group: FPX_ERR_CHECK_FAILED at complete (logger.check), nothing emitted;
 *   s0        = nextClassicRound(leader_group, chosen_watermark - 1), the first slot >= chosen_watermark of the group;
 *   n_out     = max_slot >= s0 ? (max_slot - s0) / LG + 1 : 0;
 *   next_slot = nextClassicRound(leader_group, max_slot) (RoundSystem.scala:66-80), the Leader's new nextSlot (:647);
 *               computed in 64 bits: past INT32_MAX it is FPX_ERR_SLOT_RANGE at complete (the reference's Int would
 *               wrap; DESIGN.md §7);
 *   record k  = {slot = s0 + k * LG, round, value_id_base + k | FPX_VALUE_NOOP, -1} with spans[2k..2k+1] as for
 *               fpx_leader_phase1b_wire; the value is safeValue over the held Phase1bs of acceptor group (slot / LG) % AG
 *               only (acceptorGroupIndexBySlot, :342-345), ties to the lowest acceptor index.
 * n_out > out_capacity: FPX_ERR_INVALID_ARG at complete, nothing written.  The records go to fpx_proxyleader_arm as they
 * are once the caller sets dst = (leader_group * AG + (slot / LG) % AG) << 16 | acceptor.  Scratch as for
 * fpx_leader_phase1b_wire.  _dev: as fpx_leader_phase1b_wire_dev; d_result is a device int32[4]. */
int fpx_mencius_leader_phase1b_wire(fpx_engine* e, int32_t leader_group, int32_t round, int32_t chosen_watermark,
                                    int32_t recover_slot, const uint8_t* bytes, const int32_t* offsets, int32_t n,
                                    int32_t value_id_base, fpx_p2a* out, int32_t* spans, int32_t out_capacity,
                                    int32_t* result, int64_t* err_index);
int fpx_mencius_leader_phase1b_wire_dev(fpx_engine* e, int32_t leader_group, int32_t round, int32_t chosen_watermark,
                                        int32_t recover_slot, const uint8_t* d_bytes, int32_t n_bytes,
                                        const int32_t* d_offsets, int32_t n, int32_t value_id_base, fpx_p2a* d_out,
                                        int32_t* d_spans, int32_t out_capacity, int32_t* d_result);
/* fpx_wire_encode_mencius_phase2a: Mencius' ProxyLeaderInbound{phase2a = 2 {slot, round, command_batch_or_noop}} per
 * fpx_p2a record, otherwise as fpx_wire_encode_phase2a (the span table, FPX_VALUE_NOOP, the refusals).  Decoding the
 * bytes with FPX_WIRE_MENCIUS_PROXYLEADER_INBOUND gives kind 2 and the records back. */
int fpx_wire_encode_mencius_phase2a(fpx_engine* e, const fpx_p2a* in, int32_t n, const uint8_t* bytes, int32_t n_bytes,
                                    const int32_t* spans, int32_t num_spans, int32_t value_id_base, uint8_t* out,
                                    int32_t out_capacity, int32_t* offsets, int64_t* err_index);
int fpx_wire_encode_mencius_phase2a_dev(fpx_engine* e, const fpx_p2a* d_in, int32_t n, const uint8_t* d_bytes,
                                        int32_t n_bytes, const int32_t* d_spans, int32_t num_spans,
                                        int32_t value_id_base, uint8_t* d_out, int32_t out_capacity,
                                        int32_t* d_offsets);
/* The replies a Client or ReadBatcher receives, by the handle's kind; out[] goes to fpx_reads_max_slot_replies[_dev]
 * as it is, spans[2i..2i+1] = {off, len} of the member's body (its last occurrence), {0, 0} for no member.
 *   FPX_READS_CLIENT, ClientInbound: max_slot_reply (4) -> {key = client_pseudonym, id = client_id,
 *     voter = group_index << 16 | acceptor_index, slot} (Client.scala:851-931 keys by pseudonym and checks only the
 *     clientId; client_address is required but not compared).
 *   FPX_READS_READ_BATCHER, ReadBatcherInbound: batch_max_slot_reply (4) -> {key = floorMod(read_batcher_id,
 *     key_capacity), id = read_batcher_id, voter = acceptor_index, slot} (ReadBatcher.scala:568-623;
 *     read_batcher_index is required but not used).  fpx_reads_open must open read_batcher_id under that key
 *     for the replies to find their read; the primer's id -1 is key key_capacity - 1.
 *   A group_index or acceptor_index outside [0, 2^15) gives voter = -1 (FPX_ERR_BAD_ACCEPTOR if counted).
 *   Every other member (replies, read replies, NotLeader, ...) gets key = -1, which the tally ignores, and is
 *   not parsed: the host reads it from its span. */
int fpx_reads_wire_decode(fpx_reads* r, const uint8_t* bytes, const int32_t* offsets, int32_t n, int32_t* kind,
                          fpx_max_slot_reply* out, int32_t* spans, int64_t* err_index);
int fpx_reads_wire_decode_dev(fpx_reads* r, const uint8_t* d_bytes, const int32_t* d_offsets, int32_t n, int32_t* d_kind,
                              fpx_max_slot_reply* d_out, int32_t* d_spans);
/* One canonical ReplicaInbound per completed read (fpx_read_slot of the tally): read_request{slot, command} for the
 * Client (Client.scala:900-911), read_request_batch{slot, command*} for the ReadBatcher (ReadBatcher.scala:613-617).
 * Value id = the record's key: arena[value_offsets[key] .. value_offsets[key+1]) is the message's `command`
 * field or fields, tag and length included (12 len Command, repeated for a batch).  A key outside
 * [0, num_values) is FPX_ERR_INVALID_ARG at its record. */
int fpx_reads_wire_encode_read_requests(fpx_reads* r, const fpx_read_slot* in, int32_t n, const uint8_t* arena,
                                        const int32_t* value_offsets, int32_t num_values, uint8_t* out,
                                        int32_t out_capacity, int32_t* offsets, int64_t* err_index);
int fpx_reads_wire_encode_read_requests_dev(fpx_reads* r, const fpx_read_slot* d_in, int32_t n, const uint8_t* d_arena,
                                            const int32_t* d_value_offsets, int32_t num_values, uint8_t* d_out,
                                            int32_t out_capacity, int32_t* d_offsets);

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
