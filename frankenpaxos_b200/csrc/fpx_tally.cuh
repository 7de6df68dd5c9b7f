// fpx_tally.cuh -- K3: ProxyLeader.handlePhase2b   S/multipaxos/ProxyLeader.scala:217-258
//
//   The reference applies votes one at a time: phase2bs((g,a)) = msg (:237,
//   idempotent per acceptor), then the quorum test (:238-243); the FIRST vote
//   that makes the test pass sends Chosen (:246-253) and flips the key to Done
//   (:256); later votes see Done (:227-232).  Which vote completes depends on
//   delivery order, and the order of Chosen records in the output is the order
//   of their completing votes.
//
//   Every vote gets a sequence number seq_i = seq_base + i (per-engine running
//   counter); a row keeps, per voter, the SMALLEST seq that voter was delivered
//   with (its first delivery).  With those stamps the completing vote of a key has
//   a closed form that needs no per-vote evaluation:
//       non-flexible (:238)   c(key) = the (f+1)-th smallest stamp of the row
//       flexible grid (:241)  c(key) = max over grid rows of (min stamp in the row)
//   (the first moment `phase2bs.size >= f+1` / `isWriteQuorum(phase2bs.keys)` holds).
//   The key emits Chosen in THIS batch iff seq_base <= c(key) < seq_base + n, and
//   the Chosen stream is the keys ordered by c.
//
//   One persistent cooperative kernel, no sort:
//     phase A  stamp[slot][voter] = min(stamp, seq_i): one blind RED per vote, no
//              row load; per-batch statistics (slot window, rounds) on the side
//     barrier
//     phase B  SWEEP (steady state): the window's rows are read once, coalesced
//              (one 32-byte sector per 8 row words, every CTA a contiguous run of rows),
//              c(key) evaluated per row; a key completed by vote i of this batch sets
//              bit i of a bitmap and keeps {i, value} in the CTA's shared memory;
//           or EXACT (fallback): one divergent row load per vote and the reference's
//              test evaluated at that vote ("first delivery of its voter, not a
//              quorum before, a quorum with it"); a completing vote sets bit i and
//              parks its Chosen record at tmp[i]
//     barrier
//     phase C  per 1024-vote chunk: completing votes before each bitmap word, chunk total
//     barrier
//     phase D  rank(i) = number of completing votes before i = chunk prefix + word
//              prefix + popcount below bit i.  SWEEP: every kept {i, value} goes
//              straight to out[rank(i)] (a window too large for shared memory is swept
//              a second time instead).  EXACT: ordered compaction of tmp[].
//
//   When is the sweep sound?  It never looks at a vote, so every property of a vote
//   that the reference checks must be implied by the batch statistics and the rows:
//   (1) all votes of the batch carry ONE round R and every armed row of the window
//   holds exactly that round (else a vote of another round -- which is
//   `logger.fatal`, :220-225, or belongs to a second live round of the slot -- could
//   hide behind an older stamp of its voter), (2) no poisoned row (several live
//   rounds, see fpx_arm.cuh) lies in the window, (3) no touched row is unarmed,
//   (4) every voter is a member of the slot's quorum system, (5) the window is not
//   much larger than the batch.  Any violation flips the WHOLE batch to the exact
//   path, which also produces the reference's error index.  Blind stamping is sound
//   for the same reason as before: a primary row in normal state has exactly ONE
//   armed round.  Vanilla Mencius ignores stale votes instead of failing: its entries are
//   always proposed in round 0, so round-0 votes are stamped blindly too and the sweep runs
//   unconditionally; a vote of another round sends the batch through the checked stamping pass.
#pragma once
#include "fpx_common.cuh"

namespace fpx {

struct TallyParams {
  Geometry g;
  PLState pl;
  const int4* in;
  int32_t n;
  uint32_t seq_base;
  int2* out_chosen;
  uint2* bw;               // [ceil(n/1024)*32] {x: bit i = vote i completes its key, y: completing votes before the word, in its chunk}
  uint32_t* cc;            // [ceil(n/1024)]    completing votes per 1024-vote chunk
  int2* tmp;               // [n] exact path: Chosen record of completing vote i, parked at i
  int32_t first;           // 1: output offset 0, else append at st->n_chosen (sub-launches of one call)
  int32_t path;            // 0: sweep when sound; 2: always the exact per-vote path (tests, A/B); 4: profiling, no REDs
  int32_t keep_cap;        // rows of the window one CTA can keep in shared memory between phases B and D
  unsigned long long* votes;  // vanilla Mencius: the coordinator's log entry turns ChosenEntry on completion
  // fpx_step_dev: the co-located replica's handleChosen (+ executeLog's prefix rule) applied to the Chosen
  // stream as it is emitted (fpx_replica_misc.cuh), instead of two more launches
  unsigned long long* rlog;   // non-null: Replica.handleChosen on every emitted record
  uint32_t rseq_base;         // delivery sequence number of this call's first Chosen record
  int32_t fuse_watermark;     // 1: also the first-hole scan (last sub-launch of a call)
  int32_t* d_watermark;       // optional device copy of the new watermark
  DevExchange* xch;           // multi-GPU: the new watermark also goes to every peer's frontier table
  DevStatus* st;
};

#ifndef FPX_TALLY_UNROLL
#define FPX_TALLY_UNROLL 4
#endif
#ifndef FPX_TT
#define FPX_TT 1024
#endif
constexpr int kTallyUnroll = FPX_TALLY_UNROLL;   // chunks of 32 votes per warp per pipeline stage in phase A
constexpr int kChunkVotes = 1024; // votes per rank chunk (one bitmap word per lane)
constexpr uint32_t kNoVote = 0xffffffffu;
// One CTA of 32 warps per SM: several CTAs per SM spread up to 2x in duration (their loads queue behind
// each other in the SM's L1TEX), and every phase ends at a grid barrier.
constexpr int kTT = FPX_TT;
constexpr int kTW = kTT / 32;

// One proxy-leader row from L2, two 128-bit loads per 8 words (one 32-byte sector; sm_90 has no
// 256-bit load).  Both halves are issued before either is used.
template <int ROWW>
__device__ __forceinline__ void load_row(const uint32_t* p, uint32_t (&w)[ROWW]) {
#pragma unroll
  for (int q = 0; q < ROWW / 4; ++q) {
    asm volatile("ld.global.cg.v4.b32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(w[4 * q]), "=r"(w[4 * q + 1]), "=r"(w[4 * q + 2]), "=r"(w[4 * q + 3])
                 : "l"(p + 4 * q));
  }
}

// ---------------------------------------------------------------------------
// sweep: the completing vote of one row of the window.  Returns false on an anomaly;
// *vote = index (in this batch) of the vote that completes the key, or kNoVote.
// ---------------------------------------------------------------------------
template <int ROWW>
__device__ __forceinline__ bool row_completion(const TallyParams& P, const uint32_t (&w)[ROWW], int R, uint32_t* vote) {
  const Geometry& g = P.g;
  const uint32_t hw = w[0];
  *vote = kNoVote;
  bool touched = false;
#pragma unroll
  for (int v = 0; v < ROWW - 2; ++v)
    if (v < g.voters) touched |= (w[2 + v] - P.seq_base) < (uint32_t)P.n;
  if (g.protocol == FPX_VANILLA_MENCIUS) {
    // the checked phase A only stamped votes the reference counts (right round, Phase 2 running, :1088-1116):
    // every stamp is a vote; a chosen slot emits nothing more
    if (hw == kUnarmed || (hw & kDoneBit) || !touched) return true;
  } else {
    if (hw == kUnarmed) return !touched;                 // a vote for a key that was never armed (:220-225)
    if (hw == kPoison || hw == kBusy) return false;      // several live rounds: its keys live in the table
    if ((int)(hw & ~kDoneBit) != R) return false;        // a vote of round R could hide behind an older stamp
    if (!touched) return true;
  }
  uint32_t c = kStampEmpty;
  if (!g.flexible) {
    // phase2bs.size >= f+1 (:238): the (f+1)-th smallest first-delivery stamp
    const int k = g.quorum - 1;
#pragma unroll
    for (int v = 0; v < ROWW - 2; ++v) {
      if (v >= g.voters) break;
      const uint32_t s = w[2 + v];
      int below = 0;
#pragma unroll
      for (int u = 0; u < ROWW - 2; ++u)
        if (u < g.voters) below += (w[2 + u] < s) || (w[2 + u] == s && u < v);
      if (below == k) c = s;
    }
  } else {
    // Grid.isWriteQuorum: one member of every row (S/quorums/Grid.scala:49)
    c = 0;
    for (int r = 0; r < g.groups; ++r) {
      uint32_t m = kStampEmpty;
#pragma unroll
      for (int v = 0; v < ROWW - 2; ++v) {
        const int lo = r * g.per_group;
        if (v >= lo && v < lo + g.per_group) m = min(m, w[2 + v]);
      }
      c = max(c, m);
    }
  }
  const uint32_t i = c - P.seq_base;
  if (i < (uint32_t)P.n) *vote = i;                    // Chosen is sent by vote i of this batch (:246-253)
  return true;
}

// One record of the Chosen stream at position `pos` of this call's output; with a co-located replica
// also Replica.handleChosen: the first Chosen of a slot wins (S/multipaxos/Replica.scala:580-588)
template <bool kReplica>
__device__ __forceinline__ void emit_chosen(const TallyParams& P, uint32_t pos, int slot, int local, int value, int& mx) {
  st_stream2(P.out_chosen + pos, make_int2(slot, value));
  if (kReplica && P.rlog != nullptr) {
    red_min_u64(&P.rlog[local], ((unsigned long long)(P.rseq_base + pos) << 32) | (uint32_t)value);
    mx = max(mx, P.g.base_local + ring_to_rel(P.g, local));
  }
}

// rank(i): completing votes of the batch before vote i (phase D)
__device__ __forceinline__ uint32_t vote_rank(const TallyParams& P, const uint32_t* s_ccx, uint32_t i) {
  const uint2 wd = __ldcg(&P.bw[i >> 5]);
  return s_ccx[i >> 10] + wd.y + __popc(wd.x & ((1u << (i & 31)) - 1u));
}

// Sweep over the CTA's contiguous run of window rows.  kEmit = false (phase B): mark
// the completing votes, keep {vote, value} in shared memory when it fits.  kEmit = true
// (phase D without kept entries): recompute and emit.
template <int ROWW, bool kEmit>
__device__ __forceinline__ void tally_sweep(const TallyParams& P, int w_lo, int w_hi, int R, int rows_per_cta, bool keep,
                                            uint2* s_keep, const uint32_t* s_ccx, uint32_t out_base, int& mx) {
  constexpr int U = ROWW == 8 ? 2 : 1;   // rows in flight per thread: more spills registers under the 64-register cap
  const Geometry& g = P.g;
  const long long nrows = (long long)w_hi - w_lo + 1;
  const long long r_begin = (long long)blockIdx.x * rows_per_cta;
  const long long r_end = min(nrows, r_begin + rows_per_cta);
  bool ok = true;
  // co-located replica with the watermark riding along: the first row of my run that is NOT in the log after
  // this batch (neither there before nor completed now)
  const bool track_holes = !kEmit && P.rlog != nullptr && P.fuse_watermark;
  long long hole = LLONG_MAX;
  for (long long r0 = r_begin + threadIdx.x; r0 < r_end; r0 += (long long)kTT * U) {
    uint32_t w[U][ROWW];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long r = r0 + u * kTT;
      if (r < r_end) load_row<ROWW>(P.pl.rows + (size_t)rel_to_ring(g, w_lo + r) * ROWW, w[u]);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long r = r0 + u * kTT;
      if (r >= r_end) continue;
      uint32_t i;
      ok &= row_completion<ROWW>(P, w[u], R, &i);
      if (!kEmit) {
        if (track_holes && i == kNoVote && __ldcg(&P.rlog[rel_to_ring(g, w_lo + r)]) == kU64Empty) hole = min(hole, w_lo + r);
        if (i != kNoVote) {
          red_or_u32(&P.bw[i >> 5].x, 1u << (i & 31));
          if (g.protocol == FPX_VANILLA_MENCIUS) {
            // choose(): the coordinator's own entry becomes ChosenEntry, phase2s.remove (Server.scala:622-625)
            const int slot = rel_to_slot(g, w_lo + r), ring = rel_to_ring(g, w_lo + r);
            red_max_u64(&P.votes[cell_index(g, ring, slot % g.per_group)], kCellChosen | w[u][1]);
            red_or_u32(P.pl.rows + (size_t)ring * ROWW, kDoneBit);
          }
          if (P.rlog != nullptr) {
            // co-located replica (Replica.scala:580-588), here rather than at emission: consecutive threads
            // hold consecutive log entries.  Sound in a sweep: one round per batch = at most one Chosen per
            // slot in this call, so only earlier calls can have the slot, and their numbers are smaller.
            red_min_u64(&P.rlog[rel_to_ring(g, w_lo + r)], ((unsigned long long)(P.rseq_base + i) << 32) | w[u][1]);
            mx = max(mx, g.base_local + (int)(w_lo + r));
          }
        }
        if (keep) s_keep[r - r_begin] = make_uint2(i, w[u][1]);
      } else if (i != kNoVote) {
        // Chosen(slot, pending.phase2a.value) (:249-251) at its place in the order of the completing votes
        emit_chosen<false>(P, out_base + vote_rank(P, s_ccx, i), rel_to_slot(g, w_lo + r), rel_to_ring(g, w_lo + r),
                           (int)w[u][1], mx);
      }
    }
  }
  if (!kEmit && __any_sync(0xffffffffu, !ok) && (threadIdx.x & 31) == 0) atomicOr(&P.st->ts_flags, kTsAnomaly);
  if (track_holes) {
    int h = hole == LLONG_MAX ? INT_MAX : g.base_local + (int)hole;      // ordinal
    h = __reduce_min_sync(0xffffffffu, h);
    if ((threadIdx.x & 31) == 0 && h != INT_MAX) atomicMin(&P.st->wm_found, h);
  }
}

// ---------------------------------------------------------------------------
// phase B, exact: the reference's test at every vote of the warp's range.
// kRedo = false: first evaluation; a vote whose slot is poisoned is stamped into its
// table entry and kTsPoison is raised.  kRedo = true: only those votes, against their
// (now fully stamped) table entries.
// ---------------------------------------------------------------------------
template <int ROWW, bool kRedo>
__device__ __forceinline__ void tally_exact(const TallyParams& P, int wlo, int whi, int lane) {
  const Geometry& g = P.g;
  const unsigned full = 0xffffffffu;
  const bool vanilla = g.protocol == FPX_VANILLA_MENCIUS;
  constexpr int kUB = ROWW <= 16 ? 2 : 1;
  for (int base = wlo; base < whi; base += 32 * kUB) {
    int4 rec[kUB];
#pragma unroll
    for (int u = 0; u < kUB; ++u) {
      int i = base + u * 32 + lane;
      rec[u] = (i < whi) ? ld_cg(P.in + i) : make_int4(-1, -1, -1, -1);  // {group, acceptor, slot, round}
    }
    uint32_t w[kUB][ROWW];
    uint32_t* row[kUB];
#pragma unroll
    for (int u = 0; u < kUB; ++u) {
      int i = base + u * 32 + lane;
      row[u] = nullptr;
      if (i < whi) {
        int local = local_slot(g, rec[u].z);
        if (local >= 0) {
          row[u] = P.pl.rows + (size_t)local * g.row_words;
          load_row<ROWW>(row[u], w[u]);
        }
      }
    }
#pragma unroll
    for (int u = 0; u < kUB; ++u) {
      if (base + u * 32 >= whi) break;
      const int i = base + u * 32 + lane;
      bool complete = false;
      int2 out = make_int2(0, 0);
      if (row[u] != nullptr) {
        uint32_t* r = row[u];
        const uint32_t hw = w[u][0];
        bool ok = true;
        if (kRedo && hw != kPoison) {
          ok = false;                                    // judged in the first evaluation
        } else if (vanilla) {
          // Server.handlePhase2b: no Phase 2 for the slot / already chosen -> ignore
          // (:1088-1106); stale round -> ignore (:1109-1112); larger: checkEq (:1116), phase A
          ok = hw != kUnarmed && !(hw & kDoneBit) && rec[u].w == (int)hw;
        } else if (hw == kPoison) {
          // several rounds of this slot were armed: the key lives in the table
          RowRef rr = find_row(g, P.pl, local_slot(g, rec[u].z), rec[u].z, rec[u].w);
          if (rr.p == nullptr) {
            if (!kRedo) report_error(P.st, FPX_ERR_UNKNOWN_SLOT_ROUND, i);            // :220-225
            ok = false;
          } else if (!kRedo) {
            const int v = voter_index(g, rec[u].x, rec[u].y, rec[u].z);
            if (v >= 0) red_min_u32(&rr.p[2 + v], P.seq_base + (uint32_t)i);           // late stamp (:237)
            atomicOr(&P.st->ts_flags, kTsPoison);
            ok = false;
          } else {
            r = rr.p;
            load_row<ROWW>(r, w[u]);
          }
        } else if (hw == kUnarmed || (int)hw != rec[u].w) {
          // the slot has one armed round and it is not this vote's: never armed (:220-225)
          report_error(P.st, FPX_ERR_UNKNOWN_SLOT_ROUND, i);
          ok = false;
        }
        if (ok) {
          const uint32_t seq = P.seq_base + (uint32_t)i;
          uint32_t before = 0;
#pragma unroll
          for (int v = 0; v < ROWW - 2; ++v)
            if (v < g.voters && w[u][2 + v] < seq) before |= 1u << v;
          if (!write_quorum(g, before)) {  // key still Pending when vote i is delivered
            const int v = voter_index(g, rec[u].x, rec[u].y, rec[u].z);
            if (v < 0) {
              // Grid.isWriteQuorum `require(xs subsetOf nodes)` (Grid.scala:44-47)
              report_error(P.st, FPX_ERR_BAD_ACCEPTOR, i);
            } else {
              uint32_t mine = 0;
#pragma unroll
              for (int q = 0; q < ROWW - 2; ++q)
                if (q == v) mine = w[u][2 + q];
              if (mine == seq && write_quorum(g, before | (1u << v))) {
                complete = true;
                out = make_int2(rec[u].z, (int)w[u][1]);  // Chosen(slot, pending.phase2a.value) (:249-251)
                if (vanilla) {
                  // choose(): the coordinator's own entry becomes ChosenEntry, phase2s.remove (:622-625)
                  int owner = rec[u].z % g.per_group;
                  red_max_u64(&P.votes[cell_index(g, local_slot(g, rec[u].z), owner)], kCellChosen | w[u][1]);
                  red_or_u32(r, kDoneBit);
                }
              }
            }
          }
        }
      }
      const unsigned b = __ballot_sync(full, complete);
      if (complete) P.tmp[i] = out;
      if (b != 0 && lane == 0) red_or_u32(&P.bw[(base + u * 32) >> 5].x, b);   // base is a multiple of 32
    }
  }
}

// Vanilla Mencius, checked stamping (fallback when a batch carries a vote of a round other than 0):
// Server.handlePhase2b ignores a vote when there is no Phase 2 for the slot or it is already chosen
// (:1088-1106) or its round is stale (:1109-1112); a larger round fails checkEq (:1116).
__device__ __forceinline__ void tally_stamp_checked(const TallyParams& P, int wlo, int whi, int lane) {
  const Geometry& g = P.g;
  for (int base = wlo; base < whi; base += 32 * kTallyUnroll) {
      int4 rec[kTallyUnroll];
      uint32_t* row[kTallyUnroll];
      uint32_t rw[kTallyUnroll];
#pragma unroll
      for (int u = 0; u < kTallyUnroll; ++u) {
        int i = base + u * 32 + lane;
        rec[u] = (i < whi) ? ld_cg(P.in + i) : make_int4(-1, -1, -1, -1);
      }
#pragma unroll
      for (int u = 0; u < kTallyUnroll; ++u) {
        int i = base + u * 32 + lane;
        row[u] = nullptr;
        rw[u] = kUnarmed;
        if (i < whi) {
          int local = local_slot(g, rec[u].z);
          if (local < 0) {
            if (local != kLocalRetired) report_error(P.st, FPX_ERR_SLOT_RANGE, i);
          } else {
            row[u] = P.pl.rows + (size_t)local * g.row_words;
            rw[u] = __ldcg(row[u]);
          }
        }
      }
#pragma unroll
      for (int u = 0; u < kTallyUnroll; ++u) {
        int i = base + u * 32 + lane;
        if (row[u] == nullptr) continue;
        const uint32_t w = rw[u];
        // Server.handlePhase2b: no Phase 2 for the slot / already chosen -> ignore
        // (:1088-1106); stale round -> ignore (:1109-1112); a larger round fails checkEq (:1116)
        if (w == kUnarmed || (w & kDoneBit) || rec[u].w < (int)w) continue;
        if (rec[u].w > (int)w) { report_error(P.st, FPX_ERR_UNKNOWN_SLOT_ROUND, i); continue; }
        int v = voter_index(g, rec[u].x, rec[u].y, rec[u].z);
        if (v < 0) continue;
        red_min_u32(&row[u][2 + v], P.seq_base + (uint32_t)i);
      }
    }
}

template <int ROWW>
__global__ void __launch_bounds__(kTT, 1024 / kTT) tally_kernel(TallyParams P) {
  const Geometry& g = P.g;
  extern __shared__ uint32_t s_dyn[];  // [nchunks] exclusive scan of the chunk counts, then [keep_cap] kept {vote, value}
  __shared__ int s_red[4][kTW];
  __shared__ uint32_t s_flags;
  __shared__ uint32_t s_scan[kTW];

  const unsigned full = 0xffffffffu;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int total_warps = gridDim.x * kTW;
  const int per = (((P.n + total_warps - 1) / total_warps) + 31) & ~31;   // votes per warp: contiguous ranges
  const int gw = blockIdx.x * kTW + warp;
  const int wlo = (int)min((long long)P.n, (long long)gw * per);
  const int whi = (int)min((long long)P.n, (long long)wlo + per);
  const bool vanilla = g.protocol == FPX_VANILLA_MENCIUS;
  const int nchunks = (P.n + kChunkVotes - 1) / kChunkVotes;
  uint32_t* const s_ccx = s_dyn;
  uint2* const s_keep = (uint2*)(s_dyn + ((nchunks + 1) & ~1));
  const uint32_t out_base = P.first ? 0u : (uint32_t)__ldcg(&P.st->n_chosen);   // rewritten only after the last barrier
  int mx_local = INT_MIN;   // co-located replica: largest local slot this thread put into the log

  // ---- phase A: clear the bitmap, first-delivery stamps, batch statistics
  FPX_MARK(P.st->t_tally, 0);
  if (blockIdx.x == 0 && tid == 0) P.st->wm_need_scan = 0;     // read by every CTA only after the third barrier
  for (int wd = blockIdx.x * kTT + tid; wd < nchunks * 32; wd += gridDim.x * kTT)
    __stcg(&P.bw[wd], make_uint2(0u, 0u));
  int lo = INT_MAX, hi = -1, rmin = INT_MAX, rmax = INT_MIN;
  uint32_t flags = 0;
  {
    // blind: no row header load (see the file comment); phase2bs((g,a)) = msg (:237).
    // Vanilla Mencius too: a coordinator's Phase 2 entries are always in round 0 (Server.handleClientRequest,
    // :779, enforced by fpx_vm_client_request), so a round-0 vote is right for every entry that exists; votes
    // for slots without an entry or with a chosen one are ignored by the reference (:1088-1106) and harmless
    // here (the sweep skips such rows, arming resets the stamps).  A vote of another round raises
    // kTsVanillaRound: nothing is stamped for it and the batch falls back to the checked pass below.
    // Software-pipelined: the records of stage k+1 are in flight while stage k's REDs issue.
    int4 rec[kTallyUnroll], nxt[kTallyUnroll];
#pragma unroll
    for (int u = 0; u < kTallyUnroll; ++u) {
      int i = wlo + u * 32 + lane;
      nxt[u] = (i < whi) ? ld_stream(P.in + i) : make_int4(-1, -1, -1, -1);  // {group, acceptor, slot, round}
    }
    for (int base = wlo; base < whi; base += 32 * kTallyUnroll) {
#pragma unroll
      for (int u = 0; u < kTallyUnroll; ++u) rec[u] = nxt[u];
#pragma unroll
      for (int u = 0; u < kTallyUnroll; ++u) {
        int i = base + 32 * kTallyUnroll + u * 32 + lane;
        nxt[u] = (i < whi) ? ld_stream(P.in + i) : make_int4(-1, -1, -1, -1);
      }
#pragma unroll
      for (int u = 0; u < kTallyUnroll; ++u) {
        int i = base + u * 32 + lane;
        if (i >= whi) continue;
        int local = local_slot(g, rec[u].z);
        if (local < 0) {   // a retired slot was chosen long ago: the vote finds `Done` (:227-232)
          if (local != kLocalRetired) report_error(P.st, FPX_ERR_SLOT_RANGE, i);
          continue;
        }
        const int rel = ring_to_rel(g, local);
        lo = min(lo, rel); hi = max(hi, rel);
        rmin = min(rmin, rec[u].w); rmax = max(rmax, rec[u].w);
        if (vanilla && rec[u].w != 0) { flags |= kTsVanillaRound; continue; }
        int v = voter_index(g, rec[u].x, rec[u].y, rec[u].z);
        if (v < 0) { if (!vanilla) flags |= kTsBadVoter; continue; }   // judged by the exact path (needs Done-ness at i)
        if (!(P.path & 4)) red_min_u32(P.pl.rows + (size_t)local * g.row_words + 2 + v, P.seq_base + (uint32_t)i);
      }
    }
  }
  {
    lo = __reduce_min_sync(full, lo); hi = __reduce_max_sync(full, hi);
    rmin = __reduce_min_sync(full, rmin); rmax = __reduce_max_sync(full, rmax);
    flags = __reduce_or_sync(full, flags);
    if (tid == 0) s_flags = 0;
    if (lane == 0) { s_red[0][warp] = lo; s_red[1][warp] = hi; s_red[2][warp] = rmin; s_red[3][warp] = rmax; }
    __syncthreads();
    if (lane == 0 && flags) atomicOr(&s_flags, flags);
    __syncthreads();
    if (warp == 0) {
      lo = lane < kTW ? s_red[0][lane] : INT_MAX; hi = lane < kTW ? s_red[1][lane] : -1;
      rmin = lane < kTW ? s_red[2][lane] : INT_MAX; rmax = lane < kTW ? s_red[3][lane] : INT_MIN;
      lo = __reduce_min_sync(full, lo); hi = __reduce_max_sync(full, hi);
      rmin = __reduce_min_sync(full, rmin); rmax = __reduce_max_sync(full, rmax);
      if (lane == 0 && hi >= 0) {
        atomicMin(&P.st->ts_min_local, lo); atomicMax(&P.st->ts_max_local, hi);
        atomicMin(&P.st->ts_min_round, rmin); atomicMax(&P.st->ts_max_round, rmax);
        if (s_flags) atomicOr(&P.st->ts_flags, s_flags);
      }
    }
  }
  FPX_MARK(P.st->t_tally, 1);
  grid_sync(P.st);
  FPX_MARK(P.st->t_tally, 2);

  // ---- phase B: which votes complete their key
  const int w_lo = __ldcg(&P.st->ts_min_local), w_hi = __ldcg(&P.st->ts_max_local);   // rel coordinates (live window)
  const int R = __ldcg(&P.st->ts_min_round);
  // (vanilla Mencius: the checked phase A stamped only votes the reference counts, so the rows alone decide)
  const uint32_t flags_a = __ldcg(&P.st->ts_flags);
  bool sweep = !(P.path & 2) && w_hi >= w_lo && (long long)w_hi - w_lo <= 4ll * P.n + 4096 &&
               (vanilla ? !(flags_a & kTsVanillaRound) : (flags_a == 0 && R == __ldcg(&P.st->ts_max_round)));
  // every CTA sweeps a contiguous run of the window's rows (a multiple of the CTA size)
  const int rows_per_cta = sweep ? (int)((((long long)w_hi - w_lo + gridDim.x) / gridDim.x + kTT - 1) / kTT) * kTT : 0;
  const bool keep = rows_per_cta <= P.keep_cap;
  if (sweep) {
    tally_sweep<ROWW, false>(P, w_lo, w_hi, R, rows_per_cta, keep, s_keep, s_ccx, out_base, mx_local);
    FPX_MARK(P.st->t_tally, 3);
    grid_sync(P.st);
    if (P.rlog != nullptr && P.fuse_watermark && blockIdx.x == 0 && tid == 0 && !(__ldcg(&P.st->ts_flags) & kTsAnomaly)) {
      // executeLog's prefix rule (Replica.scala:394-402) from what the sweep saw: every log put of this batch
      // is done (barrier).  Old watermark outside the window: nothing of this batch can move it.  Inside: the
      // first hole the sweep found, else the slot right after the window if that one is empty; anything else
      // is left to the first-hole scan.
      const int lo_w = __ldcg(&P.st->wm_local), W0 = g.base_local + w_lo, W1 = g.base_local + w_hi;
      int f = lo_w;
      bool settled = P.first != 0;       // a call split into several launches: earlier launches moved the log too
      if (settled && lo_w >= W0 && lo_w <= W1) {
        f = __ldcg(&P.st->wm_found);
        if (f == INT_MAX) {
          const int nxt = W1 + 1;
          if (nxt >= g.base_local + g.local_slots) f = g.base_local + g.local_slots;
          else if (__ldcg(&P.rlog[rel_to_ring(g, nxt - g.base_local)]) == kU64Empty) f = nxt;
          else settled = false;
        }
      }
      P.st->wm_found = INT_MAX;
      if (settled) {
        P.st->wm_local = f;
        const int global = f * g.shard_count + g.shard_index;
        P.st->watermark = global;
        if (P.d_watermark) *P.d_watermark = global;
        exchange_publish(P.xch, global);
      } else {
        P.st->wm_need_scan = 1;
      }
    }
    if (__ldcg(&P.st->ts_flags) & kTsAnomaly) {
      // not a steady-state batch after all: forget the sweep's marks, evaluate every vote
      sweep = false;
      for (int wd = blockIdx.x * kTT + tid; wd < nchunks * 32; wd += gridDim.x * kTT)
        __stcg(&P.bw[wd], make_uint2(0u, 0u));
      grid_sync(P.st);
    }
  }
  if (!sweep) {
    if (blockIdx.x == 0 && tid == 0) { P.st->wm_need_scan = 1; P.st->wm_found = INT_MAX; }
    if (vanilla && (flags_a & kTsVanillaRound)) {   // a vote of another round: judge every vote against its row
      tally_stamp_checked(P, wlo, whi, lane);
      grid_sync(P.st);
    }
    tally_exact<ROWW, false>(P, wlo, whi, lane);
    FPX_MARK(P.st->t_tally, 3);
    grid_sync(P.st);
    if (__ldcg(&P.st->ts_flags) & kTsPoison) {
      // some votes belong to slots with several armed rounds (leader change): their table
      // entries are fully stamped now
      tally_exact<ROWW, true>(P, wlo, whi, lane);
      grid_sync(P.st);
    }
  }
  FPX_MARK(P.st->t_tally, 4);

  // ---- phase C: completing votes before every bitmap word of a chunk, and per chunk
  for (int k = gw; k < nchunks; k += total_warps) {
    const uint32_t cnt = __popc(__ldcg(&P.bw[k * 32 + lane].x));
    uint32_t inc = cnt;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      uint32_t o = __shfl_up_sync(full, inc, d);
      if (lane >= d) inc += o;
    }
    __stcg(&P.bw[k * 32 + lane].y, inc - cnt);
    if (lane == 31) __stcg(&P.cc[k], inc);
  }
  FPX_MARK(P.st->t_tally, 5);
  grid_sync(P.st);
  const bool need_scan = __ldcg(&P.st->wm_need_scan) != 0;
  FPX_MARK(P.st->t_tally, 6);

  // ---- phase D: exclusive scan of the chunk counts (every CTA, in shared memory), then the
  //      Chosen stream in the order of the completing votes
  {
    // coalesced copy of the counts, then a blocked scan in place: thread t owns chunks [t*per_t, (t+1)*per_t)
    for (int k = tid; k < nchunks; k += kTT) s_ccx[k] = __ldcg(&P.cc[k]);
    __syncthreads();
    const int per_t = (nchunks + kTT - 1) / kTT;
    const int c0 = min(nchunks, tid * per_t), c1 = min(nchunks, c0 + per_t);
    uint32_t sum = 0;
    for (int k = c0; k < c1; ++k) sum += s_ccx[k];
    uint32_t incl = sum;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      uint32_t o = __shfl_up_sync(full, incl, d);
      if (lane >= d) incl += o;
    }
    if (lane == 31) s_scan[warp] = incl;
    __syncthreads();
    uint32_t run = incl - sum;
#pragma unroll
    for (int wv = 0; wv < kTW; ++wv) if (wv < warp) run += s_scan[wv];
    for (int k = c0; k < c1; ++k) { uint32_t c = s_ccx[k]; s_ccx[k] = run; run += c; }
    __syncthreads();
    uint32_t total = 0;
#pragma unroll
    for (int wv = 0; wv < kTW; ++wv) total += s_scan[wv];

    if (sweep && keep) {
      // the CTA's kept {vote, value} entries: one random 8-byte load (word + prefix), one 8-byte store each
      const long long nrows = (long long)w_hi - w_lo + 1;
      const long long r_begin = (long long)blockIdx.x * rows_per_cta;
      const int mine = (int)max(0ll, min(nrows, r_begin + rows_per_cta) - r_begin);
      for (int e0 = tid; e0 < mine; e0 += kTT * 4) {
        uint2 ent[4];
        uint2 wd[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int e = e0 + u * kTT;
          ent[u] = e < mine ? s_keep[e] : make_uint2(kNoVote, 0u);
          if (ent[u].x != kNoVote) wd[u] = __ldcg(&P.bw[ent[u].x >> 5]);
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          if (ent[u].x == kNoVote) continue;
          const uint32_t i = ent[u].x;
          const uint32_t rank = s_ccx[i >> 10] + wd[u].y + __popc(wd[u].x & ((1u << (i & 31)) - 1u));
          const int e = e0 + u * kTT;
          const long long rel = w_lo + r_begin + e;
          emit_chosen<false>(P, out_base + rank, rel_to_slot(g, rel), rel_to_ring(g, rel), (int)ent[u].y, mx_local);
        }
      }
    } else if (sweep) {
      tally_sweep<ROWW, true>(P, w_lo, w_hi, R, rows_per_cta, false, s_keep, s_ccx, out_base, mx_local);
    } else {
      for (int k = gw; k < nchunks; k += total_warps) {
        const uint2 wd = __ldcg(&P.bw[k * 32 + lane]);
        const uint32_t wpre = out_base + s_ccx[k] + wd.y;        // records before this lane's word
        const int2* src = P.tmp + (size_t)k * kChunkVotes + lane;
        // 8 steps at a time: the parked records are loaded unconditionally (tmp is padded to a whole
        // chunk) so that the 8 loads are in flight together; only completing votes are stored
#pragma unroll
        for (int s0 = 0; s0 < 32; s0 += 8) {
          int2 rec[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) rec[j] = __ldcg(src + (s0 + j) * 32);
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const uint32_t wv = __shfl_sync(full, wd.x, s0 + j);
            const uint32_t pre = __shfl_sync(full, wpre, s0 + j);
            if ((wv >> lane) & 1u)
              emit_chosen<true>(P, pre + __popc(wv & lanemask_lt()), rec[j].x, local_slot(g, rec[j].x), rec[j].y, mx_local);
          }
        }
      }
    }
    if (blockIdx.x == 0 && tid == 0) {
      // every CTA is past its reads of the statistics (barrier after phase C): reset them for the next launch
      P.st->n_chosen = (int)(out_base + total);
      P.st->ts_min_local = INT_MAX; P.st->ts_max_local = -1;
      P.st->ts_min_round = INT_MAX; P.st->ts_max_round = INT_MIN;
      P.st->ts_flags = 0;
      P.st->ts_path = sweep ? 1u : 2u;
    }
  }
  FPX_MARK(P.st->t_tally, 7);
  if (P.rlog == nullptr) return;

  // ---- co-located replica: largest chosen slot, then executeLog's prefix rule (Replica.scala:394-402):
  //      the first hole at or after the old watermark
  mx_local = __reduce_max_sync(full, mx_local);
  if (lane == 0) s_red[0][warp] = mx_local;
  __syncthreads();
  if (warp == 0) {
    int m = __reduce_max_sync(full, lane < kTW ? s_red[0][lane] : INT_MIN);
    if (lane == 0 && m != INT_MIN) atomicMax(&P.st->max_chosen_local, m);
  }
  if (!P.fuse_watermark || !need_scan) return;
  grid_sync(P.st);
  {
    const int lo_w = __ldcg(&P.st->wm_local);
    const int hi_w = min(__ldcg(&P.st->max_chosen_local) + 2, g.base_local + g.local_slots);  // ordinals; one past the last candidate hole
    int found = INT_MAX;
    const long long stride = (long long)gridDim.x * kTT;
    for (long long i = lo_w + (long long)blockIdx.x * kTT + tid; i < hi_w && found == INT_MAX; i += 4 * stride) {
      unsigned long long v[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) v[u] = (i + u * stride < hi_w) ? __ldcg(&P.rlog[rel_to_ring(g, i + u * stride - g.base_local)]) : 0ull;
#pragma unroll
      for (int u = 3; u >= 0; --u)
        if (i + u * stride < hi_w && v[u] == kU64Empty) found = (int)(i + u * stride);   // ascending: the smallest one last
    }
    found = __reduce_min_sync(full, found);
    __syncthreads();
    if (lane == 0) s_red[1][warp] = found;
    __syncthreads();
    if (warp == 0) {
      found = __reduce_min_sync(full, lane < kTW ? s_red[1][lane] : INT_MAX);
      if (lane == 0 && found != INT_MAX) atomicMin(&P.st->wm_found, found);
    }
    grid_sync(P.st);
    if (blockIdx.x == 0 && tid == 0) {
      int f = min(__ldcg(&P.st->wm_found), hi_w);
      f = max(f, lo_w);
      if (f > g.base_local + g.local_slots) f = g.base_local + g.local_slots;
      P.st->wm_local = f;
      P.st->wm_found = INT_MAX;
      const int global = f * g.shard_count + g.shard_index;
      P.st->watermark = global;
      if (P.d_watermark) *P.d_watermark = global;
      exchange_publish(P.xch, global);
    }
  }
  FPX_MARK(P.st->t_tally, 7);
}

}  // namespace fpx
