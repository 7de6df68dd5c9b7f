// fpx_acceptor.cuh -- K2: Acceptor.handlePhase2a for the interleaved delivery
// stream of all acceptors of the config.   S/multipaxos/Acceptor.scala:184-220
//
//   `round` is ONE scalar per acceptor (:95), so for record i addressed to
//   acceptor k the handler's test (:192) is
//        msg.round < max(round_k at batch start, max_{j<i, dst_j==k} msg_j.round)
//   (rejected messages are below the running max, so including them is
//   harmless): an exclusive keyed prefix-max in delivery order.
//
//   Persistent cooperative kernel.  The batch is cut into S contiguous segments
//   (S = 1 unless the batch is too large for L2, see acceptor_segments); inside a
//   segment every warp owns a contiguous range:
//     pass 1  stream the range once, lane k of the warp accumulates the max round
//             addressed to acceptor k (warp redux; one instruction when the whole
//             chunk carries one round -- the steady state);
//     barrier CTA aggregates -> global; every CTA takes the max over the CTAs
//             before it in the segment, over every earlier segment and the
//             acceptors' rounds at batch start = its carry-in;
//     pass 2  stream the range again (now an L2 hit): accept test, vote cell,
//             Phase2b reply, maxVotedSlot.  Replies are written at index i
//             (dense = correct whenever the batch produces no Nack);
//             then pass 1 of the next segment, and its barrier: pass 1 keeps only
//             ONE segment resident in L2 (S + 1 barriers in all);
//     barrier if any Nack was produced (leader change): pass 3 rewrites both
//             reply streams compacted in delivery order from exact prefix counts.
//   Vote cell: states(slot) = State(round, value) (:205-208) is one 64-bit
//   atomicMax of (round+1 : value_id): accepted rounds never decrease in
//   delivery order, so max == last writer, except "same round, different value"
//   which is flagged and resolved to last-in-order by the last block.
#pragma once
#include <algorithm>

#include "fpx_common.cuh"
#include "fpx_scan.cuh"

namespace fpx {

struct VoteConflict { int32_t dst, slot; };

struct AcceptorParams {
  Geometry g;
  const int4* in;
  int32_t n;
  int4* out_p2b;
  int2* out_nack;
  unsigned long long* votes;       // local_slots * voters cells
  int32_t* acc_round;              // num_keys
  int32_t* acc_max_voted;          // num_keys
  uint32_t* accept_bits;           // ceil(n/32)
  int32_t* g_agg;                  // [2][kMaxGrid][kMaxKeys] per-CTA max round per acceptor (segments alternate)
  uint32_t* g_wacc;                // [segments][grid*kAW] accepted records per warp range
  int32_t segments;                // 1 .. kAccMaxSegments
  uint32_t parity;                 // which nack counter this launch uses
  int32_t append;                  // 1: continue the reply streams of the previous launch (chunked host call)
  DevStatus* st;
  VoteConflict* conflicts;
};

constexpr int kAccUnroll = 4;
// one CTA of 32 warps per SM (see fpx_tally.cuh: several CTAs per SM spread up to 2x, and both passes end at a grid barrier)
#ifndef FPX_AT
#define FPX_AT 1024
#endif
constexpr int kAT = FPX_AT;
constexpr int kAW = kAT / 32;
constexpr int kAccMaxSegments = 8;
// Segments of a batch of n records: pass 1 pins at most half of the L2 (16 B per record), the other half
// takes pass 2's replies and vote cells.  More segments cost a grid barrier each and shorten every warp's
// run: cfg2 (3 * 2^20 records) on H100's 50 MB L2 takes 2; 4 measured 11 us slower (DESIGN.md section 4).
inline int acceptor_segments(long long n, long long l2_bytes) {
  const long long seg_bytes = l2_bytes / 2;
  if (seg_bytes <= 0) return 1;
  const long long s = (n * 16 + seg_bytes - 1) / seg_bytes;
  return (int)std::max(1ll, std::min((long long)kAccMaxSegments, s));
}
__device__ __forceinline__ int grp_of(int dst) { return dst >> 16; }

// decode + validate one Phase2a record; key = global acceptor id or -1
__device__ __forceinline__ int decode_p2a(const Geometry& g, const int4& rec, int& key, int& loc, int& vix) {
  key = -1; loc = -1; vix = -1;
  int grp = rec.w >> 16, acc = rec.w & 0xffff;
  if ((uint32_t)grp >= (uint32_t)g.groups || acc >= g.per_group) return FPX_ERR_BAD_ACCEPTOR;
  if ((uint32_t)rec.y > (uint32_t)FPX_MAX_ROUND) return FPX_ERR_ROUND_RANGE;
  int l = local_slot(g, rec.x);
  if (l < 0 && l != kLocalRetired) return FPX_ERR_SLOT_RANGE;   // retired: round compare and reply as usual, the vote cell is gone
  int v = voter_index(g, grp, acc, rec.x);
  if (v < 0 || (g.protocol == FPX_MENCIUS && grp != expected_group(g, rec.x))) return FPX_ERR_BAD_ACCEPTOR;
  key = grp * g.per_group + acc; loc = l; vix = v;
  return 0;
}
// pass 1 only needs the acceptor id and the round; slot-level validity is judged
// (and reported) in pass 2
__device__ __forceinline__ int decode_key(const Geometry& g, const int4& rec) {
  int grp = rec.w >> 16, acc = rec.w & 0xffff;
  if ((uint32_t)grp >= (uint32_t)g.groups || acc >= g.per_group) return -1;
  if ((uint32_t)rec.y > (uint32_t)FPX_MAX_ROUND) return -1;
  return grp * g.per_group + acc;
}
__device__ __noinline__ void acceptor_error(DevStatus* st, int code, int index) { report_error(st, code, index); }

// Pass 2 (kExact = false: effects + dense replies) and pass 3 (kExact = true:
// compacted replies only).  `run` is lane-indexed: lane k holds acceptor k's
// round as of the start of the warp's range.  s_mv is a [num_keys][kAT]
// table of per-thread private maxima of accepted slots (maxVotedSlot, :209).
template <bool kExact>
__device__ __forceinline__ void acceptor_apply(const AcceptorParams& P, int4* out_p2b, int2* out_nack, int wlo, int whi,
                                               int lane, int run, uint32_t pos_base, int* s_mv, uint32_t& wacc,
                                               uint32_t& wnack) {
  const Geometry& g = P.g;
  const unsigned full = 0xffffffffu;
  // the reply stream is write-once: evict_first gets it written back while this kernel
  // still runs instead of during the next kernel's reads.  This is also the last read of
  // the records pass 1 pinned (evict_last): the evict_first load releases them.
  const unsigned long long pol_out = l2_policy_evict_first();
  for (int base = wlo; base < whi; base += 32 * kAccUnroll) {
    int4 rec[kAccUnroll];
    unsigned long long cell[kAccUnroll], old[kAccUnroll];
#pragma unroll
    for (int u = 0; u < kAccUnroll; ++u) {
      int i = base + u * 32 + lane;
      rec[u] = (i < whi) ? ld_hint(P.in + i, pol_out) : make_int4(0, -1, 0, -1);
      cell[u] = 0; old[u] = 0;
    }
#pragma unroll
    for (int u = 0; u < kAccUnroll; ++u) {
      const int i0 = base + u * 32;
      if (i0 >= whi) break;
      const int i = i0 + lane;
      int key, loc, vix;
      bool valid = false;
      if (i < whi) {
        int err = decode_p2a(g, rec[u], key, loc, vix);
        if (err && !kExact) acceptor_error(P.st, err, i);
        valid = err == 0;
      }
      const int r = rec[u].y;
      int mn = __reduce_min_sync(full, valid ? r : INT_MAX);
      int mx = __reduce_max_sync(full, valid ? r : INT_MIN);
      if (mx == INT_MIN) {
        if (!kExact && lane == 0) P.accept_bits[i0 >> 5] = 0;
        continue;
      }
      int my_run = __shfl_sync(full, run, key & 31);
      int cur;
      if (mn == mx) {  // one round in the whole chunk: no in-chunk dependency
        cur = my_run;
        unsigned present = __reduce_or_sync(full, valid ? (1u << key) : 0u);
        if ((present >> lane) & 1u) run = max(run, mx);
      } else {
        int pin = INT_MIN, chunk_agg = INT_MIN;
        unsigned remaining = __ballot_sync(full, valid);
        while (remaining) {
          int leader = __ffs(remaining) - 1;
          int kk = __shfl_sync(full, key, leader);
          bool mine = valid && key == kk;
          int incl = warp_incl_scan<ScanMax>(mine ? r : INT_MIN, lane);
          int ex = __shfl_up_sync(full, incl, 1);
          if (lane == 0) ex = INT_MIN;
          if (mine) pin = ex;
          int tot = __shfl_sync(full, incl, 31);
          if (lane == kk) chunk_agg = tot;
          remaining &= ~__ballot_sync(full, mine);
        }
        cur = max(my_run, pin);
        run = max(run, chunk_agg);
      }
      const bool accept = valid && r >= cur;   // Acceptor.scala:192
      const unsigned b = __ballot_sync(full, accept);
      if (!kExact) {
        if (lane == 0) P.accept_bits[i0 >> 5] = b;
        if (accept) {
          // Phase2b(groupIndex, acceptorIndex, slot, round) (:211-219)
          st_evict_first(out_p2b + i, make_int4(rec[u].w >> 16, rec[u].w & 0xffff, rec[u].x, r), pol_out);
          // states(slot) = State(voteRound = round, voteValue) (:205-208)
          if (loc >= 0) {   // (a retired slot's vote is never read again: Phase1b starts at the chosen watermark, :171-179)
            cell[u] = ((unsigned long long)(uint32_t)(r + 1) << 32) | (uint32_t)rec[u].z;
#ifdef FPX_PROFILE_ACC_RED   // attribution build only (profiles/README.md): wrong state, re-votes go undetected
            red_max_u64(&P.votes[cell_index(g, loc, vix)], cell[u]);
#else
            old[u] = atomicMax(&P.votes[cell_index(g, loc, vix)], cell[u]);
#endif
          }
          // maxVotedSlot = max(maxVotedSlot, slot) (:209): thread-private column
          atomicMax(&s_mv[key * kAT + threadIdx.x], rec[u].x);
        }
        wnack += __popc(__ballot_sync(full, valid && !accept));
      } else {
        uint32_t before = pos_base + wacc + __popc(b & lanemask_lt());
        if (accept) {
          st_stream(out_p2b + before, make_int4(rec[u].w >> 16, rec[u].w & 0xffff, rec[u].x, r));
        } else if (valid) {
          // Nack(round) to leaders(roundSystem.leader(phase2a.round)) (:197-198)
          int ldr = r % g.num_leaders;
          if (g.protocol == FPX_MENCIUS) ldr += (grp_of(rec[u].w) / g.agroups) * g.num_leaders;
          st_stream2(out_nack + ((uint32_t)i - before), make_int2(ldr, cur));
        }
      }
      wacc += __popc(b);
    }
    if (!kExact) {
      // the atomics' return values are only consumed here, after all of the
      // group's loads/atomics are in flight
#pragma unroll
      for (int u = 0; u < kAccUnroll; ++u) {
        if ((old[u] >> 32) == (cell[u] >> 32) && old[u] != cell[u]) {
          uint32_t cidx = atomicAdd(&P.st->n_conflicts, 1u);
          if (cidx < (uint32_t)kMaxConflicts) P.conflicts[cidx] = VoteConflict{rec[u].w, rec[u].x};
        }
      }
    }
  }
}

// Pass 1 over [wlo, whi): lane k returns the max round addressed to acceptor k.  The records are
// tagged evict_last in L2 so that pass 2 (which also writes 24 B/record of replies and vote cells
// through L2) still finds them there; acceptor_segments bounds how much of the batch that pins, and
// pass 2's evict_first load releases them.
__device__ __forceinline__ int acceptor_scan(const AcceptorParams& P, int wlo, int whi, int lane) {
  const Geometry& g = P.g;
  const unsigned full = 0xffffffffu;
  const unsigned long long pol_keep = l2_policy_evict_last();
  int wagg = INT_MIN;
  for (int base = wlo; base < whi; base += 32 * kAccUnroll) {
    int4 rec[kAccUnroll];
#pragma unroll
    for (int u = 0; u < kAccUnroll; ++u) {
      int i = base + u * 32 + lane;
      rec[u] = (i < whi) ? ld_keep(P.in + i, pol_keep) : make_int4(0, -1, 0, -1);
    }
#pragma unroll
    for (int u = 0; u < kAccUnroll; ++u) {
      if (base + u * 32 >= whi) break;
      const int key = decode_key(g, rec[u]);  // -1 for padding lanes too (round -1)
      const bool valid = key >= 0;
      const int r = rec[u].y;
      int mn = __reduce_min_sync(full, valid ? r : INT_MAX);
      int mx = __reduce_max_sync(full, valid ? r : INT_MIN);
      if (mx == INT_MIN) continue;
      if (mn == mx) {
        unsigned present = __reduce_or_sync(full, valid ? (1u << key) : 0u);
        if ((present >> lane) & 1u) wagg = max(wagg, mx);
      } else {
        unsigned remaining = __ballot_sync(full, valid);
        while (remaining) {
          int leader = __ffs(remaining) - 1;
          int kk = __shfl_sync(full, key, leader);
          bool mine = valid && key == kk;
          int m = __reduce_max_sync(full, mine ? r : INT_MIN);
          if (lane == kk) wagg = max(wagg, m);
          remaining &= ~__ballot_sync(full, mine);
        }
      }
    }
  }
  return wagg;
}

// Records of warp gw in segment s: a segment is a contiguous run of seg_len records (a multiple of 32
// when S > 1), inside it warp gw owns [gw*per, (gw+1)*per), so delivery order is (segment, CTA, warp).
__device__ __forceinline__ void acceptor_range(int n, int seg_len, int per, int s, int gw, int& lo, int& hi) {
  const long long s_lo = min((long long)n, (long long)s * seg_len), s_hi = min((long long)n, s_lo + seg_len);
  lo = (int)min(s_hi, s_lo + (long long)gw * per);
  hi = (int)min(s_hi, (long long)lo + per);
}

__global__ void __launch_bounds__(kAT, 1024 / kAT) acceptor_phase2a_kernel(AcceptorParams P) {
  const Geometry& g = P.g;
  extern __shared__ int s_acc_dyn[];  // [num_keys][kAT] private maxVotedSlot columns, [segments][kAT] carry-ins
  int* const s_mv = s_acc_dyn;
  int* const s_run = s_acc_dyn + g.num_keys * kAT;
  __shared__ int s_wagg[kAW][kMaxKeys];
  __shared__ int s_tmp[2][kAW][kMaxKeys];
  __shared__ int s_win;

  const unsigned full = 0xffffffffu;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int total_warps = gridDim.x * kAW;
  const int S = P.segments;
  const int seg_len = S == 1 ? P.n : (((P.n + S - 1) / S) + 31) & ~31;
  const int per = (((seg_len + total_warps - 1) / total_warps) + 31) & ~31;   // contiguous range of every warp
  const int gw = blockIdx.x * kAW + warp;
  uint32_t* nack_ctr = P.parity ? &P.st->nack_total : &P.st->pad[0];
  uint32_t* nack_other = P.parity ? &P.st->pad[0] : &P.st->nack_total;
  if (blockIdx.x == 0 && tid == 0) *nack_other = 0;  // the counter the NEXT launch uses
  // reply-stream bases: 0, or where the previous launch of a chunked call stopped (read by
  // every CTA before the first grid barrier; rewritten only after the last)
  const uint32_t base_p2b = P.append ? (uint32_t)__ldcg(&P.st->n_p2b) : 0u;
  const uint32_t base_nack = P.append ? (uint32_t)__ldcg(&P.st->n_nack) : 0u;
  int4* const out_p2b = P.out_p2b + base_p2b;
  int2* const out_nack = P.out_nack + base_nack;
  for (int k = 0; k < g.num_keys; ++k) s_mv[k * kAT + tid] = INT_MIN;
  FPX_MARK(P.st->t_acceptor, 0);

  // ---- pass 1 of segment 0: per-acceptor max round of the warp's range (lane = acceptor)
  int wlo, whi;
  acceptor_range(P.n, seg_len, per, 0, gw, wlo, whi);
  int wagg = acceptor_scan(P, wlo, whi, lane);
  // lane k: acceptor k's round before the running segment (batch start, then every earlier segment)
  int prev = lane < g.num_keys ? __ldcg(&P.acc_round[lane]) : INT_MIN;
  uint32_t wnack = 0;
  for (int s = 0; s < S; ++s) {
    // ---- the CTA's aggregate of segment s -> global (two buffers: segment s-1's is still being read
    // by CTAs that are not yet past this barrier)
    if (s > 0) __syncthreads();   // every warp has read s_wagg for segment s-1
    s_wagg[warp][lane] = wagg;
    __syncthreads();
    int32_t* const agg = P.g_agg + (s & 1) * kMaxGrid * kMaxKeys;
    if (warp == 0) {
      int cta_agg = INT_MIN;
#pragma unroll
      for (int w = 0; w < kAW; ++w) cta_agg = max(cta_agg, s_wagg[w][lane]);
      __stcg(&agg[blockIdx.x * kMaxKeys + lane], cta_agg);
    }
    if (s == 0) FPX_MARK(P.st->t_acceptor, 1);
    grid_sync(P.st);
    if (s == 0) FPX_MARK(P.st->t_acceptor, 2);

    // ---- carry-in: rounds before segment s + every CTA before this one in segment s; and the max over
    // the whole segment, which is part of the next segment's carry.  Thread t covers CTAs t, t+kAT, ...
    // for every acceptor: all loads independent.
    for (int k = 0; k < g.num_keys; ++k) {
      int vb = INT_MIN, va = INT_MIN;
      for (int c = tid; c < (int)gridDim.x; c += kAT) {
        const int v = __ldcg(&agg[c * kMaxKeys + k]);
        va = max(va, v);
        if (c < (int)blockIdx.x) vb = max(vb, v);
      }
      vb = __reduce_max_sync(full, vb);
      va = __reduce_max_sync(full, va);
      if (lane == 0) { s_tmp[0][warp][k] = vb; s_tmp[1][warp][k] = va; }
    }
    __syncthreads();
    int run = prev;
    if (lane < g.num_keys) {
#pragma unroll
      for (int w = 0; w < kAW; ++w) { run = max(run, s_tmp[0][w][lane]); prev = max(prev, s_tmp[1][w][lane]); }
    }
    for (int w = 0; w < warp; ++w) run = max(run, s_wagg[w][lane]);
    s_run[s * kAT + tid] = run;   // pass 3 starts from the same carry
    if (s == 0) FPX_MARK(P.st->t_acceptor, 3);

    // ---- pass 2 of segment s: decisions + effects, replies at dense positions
    uint32_t wacc = 0;
    acceptor_apply<false>(P, out_p2b, out_nack, wlo, whi, lane, run, 0u, s_mv, wacc, wnack);
    if (lane == 0) __stcg(&P.g_wacc[s * total_warps + gw], wacc);
    // ---- pass 1 of segment s + 1 (published at the top of the next iteration)
    if (s + 1 < S) {
      acceptor_range(P.n, seg_len, per, s + 1, gw, wlo, whi);
      wagg = acceptor_scan(P, wlo, whi, lane);
    }
  }
  if (lane == 0 && wnack) atomicAdd(nack_ctr, wnack);
  __syncthreads();
  for (int k = warp; k < g.num_keys; k += kAW) {
    int m = INT_MIN;
#pragma unroll
    for (int t = lane; t < kAT; t += 32) m = max(m, s_mv[k * kAT + t]);
    m = __reduce_max_sync(full, m);
    if (lane == 0 && m != INT_MIN) atomicMax(&P.acc_max_voted[k], m);
  }
  FPX_MARK(P.st->t_acceptor, 4);
  grid_sync(P.st);
  FPX_MARK(P.st->t_acceptor, 5);

  // round after the batch = max over everything (:204); only now is it safe to
  // overwrite the batch-start value every CTA read above
  if (blockIdx.x == gridDim.x - 1 && warp == 0 && lane < g.num_keys) P.acc_round[lane] = prev;
  const uint32_t total_nacks = __ldcg(nack_ctr);
  if (total_nacks == 0) {
    if (blockIdx.x == 0 && tid == 0) { P.st->n_p2b = (int)base_p2b + P.n; P.st->n_nack = (int)base_nack; }
  } else {
    // ---- pass 3 (leader change only): exact, compacted reply streams.  `before` = records accepted
    // by the warp ranges before this one in delivery order, (segment, warp) major to minor.
    uint32_t before = 0;
    int j0 = 0;
    for (int s = 0; s < S; ++s) {
      const int idx = s * total_warps + gw;
      uint32_t b = 0;
      for (int j = j0 + lane; j < idx; j += 32) b += __ldcg(&P.g_wacc[j]);
      before += __reduce_add_sync(full, b);
      j0 = idx;
      acceptor_range(P.n, seg_len, per, s, gw, wlo, whi);
      uint32_t wacc2 = 0, wnack2 = 0;
      acceptor_apply<true>(P, out_p2b, out_nack, wlo, whi, lane, s_run[s * kAT + tid], before, s_mv, wacc2, wnack2);
      if (s == S - 1 && gw == total_warps - 1 && lane == 0) {
        P.st->n_p2b = (int)(base_p2b + before + wacc2);
        P.st->n_nack = (int)base_nack + P.n - (int)(before + wacc2);
      }
    }
  }

  // ---- CTA 0: same (acceptor, slot, round) voted twice with different values in one batch -> the
  // later delivery must win (map overwrite, :205).  Every conflict was recorded in pass 2, i.e. before
  // the second grid barrier.
  if (blockIdx.x != 0) return;
  uint32_t nc = __ldcg(&P.st->n_conflicts);
  if (nc == 0) return;
  if (nc > (uint32_t)kMaxConflicts) {
    if (tid == 0) { report_error(P.st, FPX_ERR_CONFLICT, 0); P.st->n_conflicts = 0; }
    return;
  }
  for (uint32_t cix = 0; cix < nc; ++cix) {
    int dst = P.conflicts[cix].dst, slot = P.conflicts[cix].slot;
    if (tid == 0) s_win = -1;
    __syncthreads();
    for (int j = tid; j < P.n; j += kAT) {
      int4 rr = P.in[j];
      if (rr.w == dst && rr.x == slot && ((__ldcg(&P.accept_bits[j >> 5]) >> (j & 31)) & 1u)) atomicMax(&s_win, j);
    }
    __syncthreads();
    if (tid == 0 && s_win >= 0) {
      int4 rr = P.in[s_win];
      int l = local_slot(g, slot);
      int v = voter_index(g, dst >> 16, dst & 0xffff, slot);
      P.votes[cell_index(g, l, v)] = ((unsigned long long)(uint32_t)(rr.y + 1) << 32) | (uint32_t)rr.z;
    }
    __syncthreads();
  }
  if (tid == 0) P.st->n_conflicts = 0;
}

}  // namespace fpx
