// fpx_scan.cuh -- the scans and reductions of the kernels outside the hot path (own code, no library).
//
//   Operators: ScanSum, ScanMax and ScanOr over u32, i32 or u64, and Seg<Op> over SegVal {value, head flag}:
//   a segmented scan is the plain scan under (a, f) . (b, g) = (g ? b : a op b, f | g), so its result says
//   whether a head was seen at or before the element.  T() is the identity of every operator (ScanMax only
//   runs over non-negative values where it needs one).
//     warp_incl_scan, warp_excl, warp_reduce   one value per lane
//     cta_scan<NT, kExcl>, cta_reduce<NT>      one value per thread of an NT-thread CTA (NT = 256 or 1024).
//                                              Each owns its shared scratch and ends with the barrier that
//                                              makes it reusable, so a caller may run one per column in a loop.
//     tile_offsets_kernel                      one CTA: exclusive sum of per-tile counts, optionally the total
//     tile_carry_kernel                        one CTA: what flows into every tile of a segmented scan from the
//                                              tiles before it, for K columns at once
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace fpx {

struct ScanSum {
  template <class T> __device__ __forceinline__ T operator()(T a, T b) const { return a + b; }
};
struct ScanMax {   // max(b, a): this operand order keeps the acceptor's hot loop compiled as it was
  template <class T> __device__ __forceinline__ T operator()(T a, T b) const { return max(b, a); }
};
struct ScanOr {
  template <class T> __device__ __forceinline__ T operator()(T a, T b) const { return a | b; }
};

template <class T> struct SegVal {
  T v;
  uint32_t f;   // a segment head at or before this element
};
template <class Op> struct Seg {
  template <class T> __device__ __forceinline__ SegVal<T> operator()(SegVal<T> a, SegVal<T> b) const {
    return {b.f ? b.v : Op()(a.v, b.v), a.f | b.f};
  }
};

template <class T> __device__ __forceinline__ T shfl_up(T x, int d) { return __shfl_up_sync(0xffffffffu, x, d); }
template <class T> __device__ __forceinline__ SegVal<T> shfl_up(SegVal<T> x, int d) { return {shfl_up(x.v, d), shfl_up(x.f, d)}; }
template <class T> __device__ __forceinline__ T shfl_idx(T x, int l) { return __shfl_sync(0xffffffffu, x, l); }
template <class T> __device__ __forceinline__ SegVal<T> shfl_idx(SegVal<T> x, int l) { return {shfl_idx(x.v, l), shfl_idx(x.f, l)}; }

template <class Op, class T> __device__ __forceinline__ T warp_incl_scan(T v, int lane, Op op = Op()) {
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const T o = shfl_up(v, d);
    if (lane >= d) v = op(o, v);
  }
  return v;
}
// the exclusive result of a warp scan from its inclusive one: lane 0 gets `first`
template <class T> __device__ __forceinline__ T warp_excl(T incl, int lane, T first) {
  const T o = shfl_up(incl, 1);
  return lane ? o : first;
}
// every lane gets the warp's total
template <class Op, class T> __device__ __forceinline__ T warp_reduce(T v, Op op = Op()) {
#pragma unroll
  for (int d = 16; d; d >>= 1) v = op(v, __shfl_xor_sync(0xffffffffu, v, d));
  return v;
}

// Inclusive (or exclusive) scan of one value per thread in thread order; *total = the CTA's aggregate.
template <int NT, bool kExcl, class Op, class T>
__device__ __forceinline__ T cta_scan(T v, Op op, T* total = nullptr) {
  static_assert(NT % 32 == 0 && NT <= 1024, "one warp scans the warp totals");
  __shared__ T s_w[NT / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const T incl = warp_incl_scan(v, lane, op);
  if (lane == 31) s_w[warp] = incl;
  __syncthreads();
  const T wi = warp_incl_scan(s_w[min(lane, NT / 32 - 1)], lane, op);   // every warp scans the warp totals itself
  const T pre = shfl_idx(wi, warp > 0 ? warp - 1 : 0);
  if (total) *total = shfl_idx(wi, NT / 32 - 1);
  const T mine = kExcl ? warp_excl(incl, lane, T()) : incl;
  __syncthreads();
  return warp > 0 ? op(pre, mine) : mine;
}

// every thread gets the CTA's aggregate
template <int NT, class Op, class T> __device__ __forceinline__ T cta_reduce(T v, Op op) {
  __shared__ T s_w[NT / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  v = warp_reduce(v, op);
  if (lane == 0) s_w[warp] = v;
  __syncthreads();
  v = warp_reduce(lane < NT / 32 ? s_w[lane] : T(), op);
  __syncthreads();
  return v;
}

// Exclusive sum of the m counters c[0, m) in place, 4 per thread; *total = their sum unless total is null.
__global__ void __launch_bounds__(1024) tile_offsets_kernel(uint32_t* c, int m, uint32_t* total) {
  uint32_t run = 0;
  for (int base = 0; base < m; base += 1024 * 4) {
    uint32_t v[4], sum = 0;
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int i = base + threadIdx.x * 4 + u;
      v[u] = i < m ? c[i] : 0u;
      sum += v[u];
    }
    uint32_t chunk;
    uint32_t off = run + cta_scan<1024, true>(sum, ScanSum(), &chunk);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int i = base + threadIdx.x * 4 + u;
      if (i < m) c[i] = off;
      off += v[u];
    }
    run += chunk;
  }
  if (total && threadIdx.x == 0) *total = run;
}

// Tile carries of a segmented scan split into tiles, K columns: agg[t][k] is tile t's aggregate since its last
// segment head (all of it if it holds none), head[t] != 0 when tile t holds a head.  carry[t][k] = the aggregate
// of tiles s .. t - 1, s the last tile before t that holds a head (0 if none): what flows into the elements of
// tile t before its first head.
template <class Op, class T>
__global__ void __launch_bounds__(1024) tile_carry_kernel(const T* agg, const uint32_t* head, T* carry, int tiles, int k) {
  const Seg<Op> op;
  for (int c = 0; c < k; ++c) {
    SegVal<T> run{};
    for (int base = 0; base < tiles; base += 1024) {
      const int t = base + threadIdx.x;
      SegVal<T> x{};
      if (t < tiles) x = {agg[(size_t)t * k + c], head[t]};
      SegVal<T> chunk;
      const SegVal<T> incl = op(run, cta_scan<1024, false>(x, op, &chunk));
      if (t == 0) carry[c] = T();
      if (t + 1 < tiles) carry[(size_t)(t + 1) * k + c] = incl.v;
      run = op(run, chunk);
    }
  }
}

}  // namespace fpx
