// fpx_epaxos_graph.cuh -- EPaxos execution on dense prefix dependencies: TarjanDependencyGraph specialised to
// Instance keys and InstancePrefixSet dependencies (S/depgraph/TarjanDependencyGraph.scala:225-451,
// S/epaxos/Replica.scala:864-886).  Vertex (c, j) depends on every (c', j') with j' < w_c'(c, j), except itself
// (subtractOne, Replica.scala:582), executed instances excepted (materializedDiff, :372).
//
//   No edge is materialised and no depth-first search is run.  With a(c, j) = w(c, j) for a live (committed,
//   unexecuted) instance and 0 otherwise, X(v) = the elementwise max of w over v and everything live v reaches
//   is computed as (DESIGN §6b):
//     prefix max     P_c[k] = max_{j<k} a(c, j)                       one segmented scan per column: tile maxima,
//                                                                      tile carries (tile_carry_kernel), tile scans
//     closure        T0_c[k] = max(k e_c, P_c[k]);  T^{m+1}_c[k] = max_c' T^m_c'[T^m_c[k][c']]   pointer jumping
//     per vertex     X(v) = max_c T_c[w_c(v)]
//   v is eligible iff X_c(v) <= A_c (A_c = the column's first absent instance) for every c; with
//   covered(v) = inst_number < X_{inst_replica}(v), the eligible vertices sorted by
//   (sum X, !covered, X, seq, replica, number) are the components in dependency order: a component is a run of
//   covered vertices with one X, an uncovered vertex is a component of its own.
//
//   Work per call scales with each column's live window [lo_c, hi_c): lo_c = the first unexecuted instance,
//   hi_c = 1 + the highest instance ever committed (>= lo_c).  Below lo_c everything is executed (T_c[k] =
//   k e_c), at and above hi_c nothing is live (T_c[k] = max(k e_c, T_c[hi_c])).
#pragma once
#include "fpx_common.cuh"
#include "fpx_scan.cuh"
#include "fpx_sort.cuh"

namespace fpx {

constexpr int kEgMaxN = 7;
constexpr int kEgTile = 1024;          // vertices per tile (scan, closure, compaction)
constexpr int kEgThreads = 256;        // grid-stride kernels
constexpr uint8_t kEgAbsent = 0, kEgCommitted = 1, kEgExecuted = 2;

struct EgState {
  int32_t n, cap;                      // columns (replicas), instances per column
  uint8_t* status;                     // [n * cap] absent / committed / executed, index c * cap + j
  int32_t* seq;                        // [n * cap]
  int32_t* w;                          // [n * cap * n] watermarks, clamped to [0, cap + 1]
  int32_t* claim;                      // [n * cap] commit: lowest batch index that commits the instance
  int32_t* win;                        // [32] lo[8], hi[8], A[8] (first absent), M[8] (max live watermark)
  int32_t* tab[2];                     // [n * (cap + 1) * n] closure tables, T_c[k] at (c * (cap + 1) + k) * n
  int32_t* x;                          // [n * cap * n] X of the window's live vertices
  uint8_t* elig;                       // [n * cap]
  uint8_t* blocker;                    // [n * cap]
  int32_t* ids;                        // [n * cap] eligible vertices, (replica, number) order
  int32_t* tile_agg;                   // [tiles * n]
  int32_t* tile_carry;                 // [tiles * n]
  uint32_t* tile_cnt;                  // [tiles + 1] first the prefix's head flags (1 at a column's first tile), then
                                       // eligible vertices per tile, then their exclusive scan
  uint32_t* changed;                   // [kEgMaxRounds] round m raised changed[m]; [kEgMaxRounds]: eligible count
  DevStatus* st;
};
constexpr int kEgMaxRounds = 40;

// The window of one execute call, read by the host and passed by value: tiles never cross a column.
struct EgWin {
  int32_t lo[kEgMaxN], hi[kEgMaxN];
  int32_t tile_off[kEgMaxN + 1];       // vertex tiles of column c: tile_off[c] .. tile_off[c+1]
  int32_t tab_off[kEgMaxN + 1];        // table entries [lo_c, hi_c] of non-empty columns, prefix
};

__device__ __forceinline__ int eg_tile_col(const EgWin& W, int n, int t) {
  int c = 0;
  while (c + 1 < n && t >= W.tile_off[c + 1]) ++c;
  return c;
}

// T_c[k] of table `tab` for any k in [0, cap + 1]
__device__ __forceinline__ void eg_look(const EgState& S, const EgWin& W, const int32_t* tab, int c, int k, int32_t* y) {
  const int lo = W.lo[c], hi = W.hi[c];
  if (k <= lo || hi == lo) {
#pragma unroll
    for (int q = 0; q < kEgMaxN; ++q) y[q] = 0;
  } else {
    const int32_t* r = tab + ((size_t)c * (S.cap + 1) + min(k, hi)) * S.n;
#pragma unroll
    for (int q = 0; q < kEgMaxN; ++q) y[q] = q < S.n ? __ldcg(r + q) : 0;
  }
#pragma unroll
  for (int q = 0; q < kEgMaxN; ++q)
    if (q == c) y[q] = max(y[q], k);
}

// ---- commit (:225-239): the first record of the batch for an instance wins; an instance outside the handle is
// FPX_ERR_SLOT_RANGE at its record and then no record of the batch is applied.  Rows {rep, num, value, seq, deps[n]}.
__global__ void eg_commit_claim_kernel(EgState S, const int32_t* in, int n_rec) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_rec) return;
  const int32_t* r = in + (size_t)i * (4 + S.n);
  const int rep = r[0], num = r[1];
  if ((unsigned)rep >= (unsigned)S.n || (unsigned)num >= (unsigned)S.cap) { report_error(S.st, FPX_ERR_SLOT_RANGE, i); return; }
  const size_t v = (size_t)rep * S.cap + num;
  if (S.status[v] == kEgAbsent) atomicMin(&S.claim[v], i);
}
__global__ void eg_commit_apply_kernel(EgState S, const int32_t* in, int n_rec) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_rec) return;
  const int32_t* r = in + (size_t)i * (4 + S.n);
  const int rep = r[0], num = r[1];
  if ((unsigned)rep >= (unsigned)S.n || (unsigned)num >= (unsigned)S.cap) return;
  const size_t v = (size_t)rep * S.cap + num;
  if (S.claim[v] != i) return;
  S.claim[v] = INT_MAX;
  if (__ldcg(&S.st->err_word) != ~0ull) return;   // a record of this batch (or an uncollected earlier one) failed
  S.status[v] = kEgCommitted;
  S.seq[v] = r[3];
  for (int q = 0; q < S.n; ++q) S.w[v * S.n + q] = min(max(r[4 + q], 0), S.cap + 1);
  atomicMax(&S.win[8 + rep], num + 1);
}

// ---- updateExecuted (:241-244) for every (c, j < wm[c]) when wm != null, then lo_c = the first unexecuted
// instance (executed instances at or above hi_c do not exist: everything there is absent).  One CTA per column.
__global__ void __launch_bounds__(1024) eg_executed_kernel(EgState S, const int32_t* wm) {
  __shared__ int s_first;
  const int c = blockIdx.x;
  int start = S.win[c];
  const int hi = S.win[8 + c];
  if (wm) {
    const int e = min(max(wm[c], 0), S.cap);
    for (int j = start + threadIdx.x; j < e; j += blockDim.x) S.status[(size_t)c * S.cap + j] = kEgExecuted;
    start = max(start, e);
  }
  if (threadIdx.x == 0) s_first = max(start, hi);
  __syncthreads();
  for (int base = start; base < hi; base += blockDim.x) {
    const int j = base + threadIdx.x;
    if (j < hi && S.status[(size_t)c * S.cap + j] != kEgExecuted) atomicMin(&s_first, j);
    __syncthreads();
    if (s_first < hi) break;
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    S.win[c] = s_first;
    S.win[8 + c] = max(hi, s_first);
  }
}

// ---- execute, step 0: A_c starts at hi_c (everything from hi_c on is absent; hi_c <= cap), M_c at 0, flags clear
__global__ void eg_prepare_kernel(EgState S) {
  const int t = threadIdx.x;
  if (t < kEgMaxN) { S.win[16 + t] = S.win[8 + t]; S.win[24 + t] = 0; }
  for (int m = t; m <= kEgMaxRounds; m += blockDim.x) S.changed[m] = 0;
}

// vector max of the tile, with A_c (first absent) and M_c (largest live watermark, capped at cap) on the side
__global__ void __launch_bounds__(kEgTile) eg_prefix_tile_kernel(EgState S, EgWin W) {
  const int t = blockIdx.x, c = eg_tile_col(W, S.n, t);
  const int j = W.lo[c] + (t - W.tile_off[c]) * kEgTile + threadIdx.x;
  int32_t a[kEgMaxN] = {};
  if (j < W.hi[c]) {
    const size_t v = (size_t)c * S.cap + j;
    const uint8_t s = S.status[v];
    if (s == kEgCommitted) {
#pragma unroll
      for (int q = 0; q < kEgMaxN; ++q)
        if (q < S.n) a[q] = S.w[v * S.n + q];
    } else if (s == kEgAbsent) {
      atomicMin(&S.win[16 + c], j);
    }
  }
#pragma unroll
  for (int q = 0; q < kEgMaxN; ++q) {
    if (q >= S.n) break;
    const int32_t m = cta_reduce<kEgTile>(a[q], ScanMax());
    if (threadIdx.x == 0) {
      S.tile_agg[(size_t)t * S.n + q] = m;
      if (m > 0) atomicMax(&S.win[24 + q], min(m, S.cap));
    }
  }
  if (threadIdx.x == 0) S.tile_cnt[t] = t == W.tile_off[c];   // a column's segment starts with this tile
}

// T0_c[j + 1] = max((j + 1) e_c, P_c[j + 1]) for every window vertex j; T0_c[lo_c] = lo_c e_c
__global__ void __launch_bounds__(kEgTile) eg_prefix_apply_kernel(EgState S, EgWin W) {
  const int t = blockIdx.x, c = eg_tile_col(W, S.n, t);
  const int j = W.lo[c] + (t - W.tile_off[c]) * kEgTile + threadIdx.x;
  const bool in = j < W.hi[c];
  const bool first = t == W.tile_off[c];   // the column starts here: nothing flows in from earlier tiles
  int32_t a[kEgMaxN] = {};
  if (in) {
    const size_t v = (size_t)c * S.cap + j;
    if (S.status[v] == kEgCommitted) {
#pragma unroll
      for (int q = 0; q < kEgMaxN; ++q)
        if (q < S.n) a[q] = S.w[v * S.n + q];
    }
  }
#pragma unroll
  for (int q = 0; q < kEgMaxN; ++q) {
    if (q >= S.n) break;
    a[q] = cta_scan<kEgTile, false>(a[q], ScanMax());
  }
  if (!in) return;
  int32_t* T = S.tab[0];
  const size_t row = (size_t)c * (S.cap + 1);
#pragma unroll
  for (int q = 0; q < kEgMaxN; ++q) {
    if (q >= S.n) break;
    int32_t m = first ? a[q] : max(a[q], S.tile_carry[(size_t)t * S.n + q]);
    if (q == c) m = max(m, j + 1);
    T[(row + j + 1) * S.n + q] = m;
    if (j == W.lo[c]) T[(row + j) * S.n + q] = q == c ? j : 0;
  }
}

// One pointer-jumping round: dst_c[k] = max_c' src_c'[src_c[k][c']] over every table entry of the window.  Round
// m > 0 returns at once when round m - 1 changed nothing (both tables then hold the closure).
__global__ void __launch_bounds__(kEgThreads) eg_round_kernel(EgState S, EgWin W, int m) {
  if (m > 0 && __ldcg(&S.changed[m - 1]) == 0) return;
  const int32_t* src = S.tab[m & 1];
  int32_t* dst = S.tab[(m + 1) & 1];
  const int total = W.tab_off[S.n];
  bool raised = false;
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < total; e += gridDim.x * blockDim.x) {
    int c = 0;
    while (c + 1 < S.n && e >= W.tab_off[c + 1]) ++c;
    const int k = W.lo[c] + (e - W.tab_off[c]);
    const size_t at = ((size_t)c * (S.cap + 1) + k) * S.n;
    int32_t y[kEgMaxN], r[kEgMaxN], z[kEgMaxN];
#pragma unroll
    for (int q = 0; q < kEgMaxN; ++q) { y[q] = q < S.n ? src[at + q] : 0; r[q] = y[q]; }
#pragma unroll
    for (int c2 = 0; c2 < kEgMaxN; ++c2) {
      if (c2 >= S.n) break;
      eg_look(S, W, src, c2, y[c2], z);
#pragma unroll
      for (int q = 0; q < kEgMaxN; ++q) r[q] = max(r[q], z[q]);
    }
#pragma unroll
    for (int q = 0; q < kEgMaxN; ++q) {
      if (q >= S.n) break;
      raised |= r[q] != y[q];
      dst[at + q] = r[q];
    }
  }
  if (__any_sync(0xffffffffu, raised) && (threadIdx.x & 31) == 0) S.changed[m] = 1;
}

// the closure did not settle within the bound: a defect, reported instead of a wrong answer
__global__ void eg_check_kernel(EgState S, int rounds) {
  if (S.changed[rounds - 1]) report_error(S.st, FPX_ERR_CHECK_FAILED, 0);
}

// X, eligibility and blockers of every window vertex; eligible vertices counted per tile
__global__ void __launch_bounds__(kEgTile) eg_closure_kernel(EgState S, EgWin W, int rounds) {
  const int t = blockIdx.x, c = eg_tile_col(W, S.n, t);
  const int j = W.lo[c] + (t - W.tile_off[c]) * kEgTile + threadIdx.x;
  const int32_t* T = S.tab[rounds & 1];
  const bool settled = __ldcg(&S.changed[rounds - 1]) == 0;
  int ok = 0;
  if (j < W.hi[c]) {
    const size_t v = (size_t)c * S.cap + j;
    const uint8_t s = S.status[v];
    S.blocker[v] = s == kEgAbsent && j < S.win[24 + c];
    if (s == kEgCommitted && settled) {
      int32_t x[kEgMaxN] = {}, z[kEgMaxN];
#pragma unroll
      for (int c2 = 0; c2 < kEgMaxN; ++c2) {
        if (c2 >= S.n) break;
        eg_look(S, W, T, c2, S.w[v * S.n + c2], z);
#pragma unroll
        for (int q = 0; q < kEgMaxN; ++q) x[q] = max(x[q], z[q]);
      }
      ok = 1;
#pragma unroll
      for (int q = 0; q < kEgMaxN; ++q) {
        if (q >= S.n) break;
        ok &= x[q] <= S.win[16 + q];
        S.x[v * S.n + q] = x[q];
      }
    }
    S.elig[v] = (uint8_t)ok;
  }
  const int cnt = __syncthreads_count(ok);
  if (threadIdx.x == 0) S.tile_cnt[t] = (uint32_t)cnt;
}

// eligible vertices to ids[] in (replica, number) order; tile_cnt holds the exclusive scan of the tile counts
__global__ void __launch_bounds__(kEgTile) eg_compact_kernel(EgState S, EgWin W) {
  const int t = blockIdx.x, c = eg_tile_col(W, S.n, t);
  const int j = W.lo[c] + (t - W.tile_off[c]) * kEgTile + threadIdx.x;
  const size_t v = (size_t)c * S.cap + j;
  const bool ok = j < W.hi[c] && S.elig[v];
  const uint32_t r = cta_scan<kEgTile, true>(ok ? 1u : 0u, ScanSum());
  if (ok) S.ids[S.tile_cnt[t] + r] = (int32_t)v;
}

__device__ __forceinline__ bool eg_covered(const EgState& S, int32_t v) {
  return v % S.cap < S.x[(size_t)v * S.n + v / S.cap];
}

// sort key `which` of eligible vertex p: 0 seq, 1 + c X_c, n + 1 2 * sum X + !covered
__global__ void eg_key_kernel(EgState S, uint32_t* key, int m, int which) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= m) return;
  const int32_t v = S.ids[p];
  uint32_t k;
  if (which == 0) {
    k = (uint32_t)S.seq[v] ^ 0x80000000u;
  } else if (which <= S.n) {
    k = (uint32_t)S.x[(size_t)v * S.n + which - 1];
  } else {
    uint32_t sum = 0;
    for (int q = 0; q < S.n; ++q) sum += (uint32_t)S.x[(size_t)v * S.n + q];
    k = 2u * sum + (eg_covered(S, v) ? 0u : 1u);
  }
  key[p] = k;
}

// executables in order: rows {replica, number}, head = a component starts (X or covered changes, or uncovered);
// executed.add (:305-311)
__global__ void eg_emit_kernel(EgState S, const uint32_t* perm, int m, int32_t* out, uint8_t* head) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= m) return;
  const int32_t v = S.ids[perm[p]];
  out[2 * p] = v / S.cap;
  out[2 * p + 1] = v % S.cap;
  bool h = p == 0 || !eg_covered(S, v);
  if (!h) {
    const int32_t u = S.ids[perm[p - 1]];
    h = !eg_covered(S, u);
    for (int q = 0; q < S.n && !h; ++q) h = S.x[(size_t)u * S.n + q] != S.x[(size_t)v * S.n + q];
  }
  head[p] = h;
  S.status[v] = kEgExecuted;
}

}  // namespace fpx
