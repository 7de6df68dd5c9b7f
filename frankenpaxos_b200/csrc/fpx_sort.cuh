// fpx_sort.cuh -- stable LSD radix sort of a permutation by 32-bit keys (own kernels, no library).
//
//   sort_perm_by_key(perm, keys, n, bits): reorders perm[0..n) so that keys[perm[i]] is
//   non-decreasing, STABLE (ties keep their order in perm).  Sorting by several words is a
//   sequence of calls, least significant word first.  8 bits per pass, three kernels per pass:
//     hist     every CTA counts the digits of its contiguous tile of 2048 entries (shared-memory
//              atomics) -> g_hist[digit][tile]
//     offsets  exclusive scan of g_hist in (digit, tile) order, one CTA (tile_offsets_kernel, fpx_scan.cuh)
//     scatter  every CTA ranks its tile stably: warp w takes the 32-entry chunks w, w+8, ... of the
//              tile; inside a chunk __match_any_sync groups equal digits and the rank is the
//              number of lower lanes in the group; per-(chunk, digit) counts are prefixed over the
//              chunks in shared memory; destination = g_hist[digit][tile] + chunk prefix + rank.
//   Used by the EPaxos conflict index (accesses grouped by table row, delivery order kept inside a
//   row) and by the dependency-graph execution (components in dependency order).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "fpx_scan.cuh"

namespace fpx {

constexpr int kSortTile = 2048;
constexpr int kSortThreads = 256;
constexpr int kSortChunks = kSortTile / 32;   // 64 chunks of 32 entries per tile

__global__ void __launch_bounds__(kSortThreads) sort_hist_kernel(const uint32_t* perm, const uint32_t* keys, int n, int shift,
                                                                 uint32_t* g_hist, int n_tiles) {
  __shared__ uint32_t s_h[256];
  const int tile = blockIdx.x;
  s_h[threadIdx.x] = 0;
  __syncthreads();
  const int base = tile * kSortTile;
  for (int j = threadIdx.x; j < kSortTile; j += kSortThreads) {
    int i = base + j;
    if (i < n) atomicAdd(&s_h[(keys[perm[i]] >> shift) & 255u], 1u);
  }
  __syncthreads();
  g_hist[(size_t)threadIdx.x * n_tiles + tile] = s_h[threadIdx.x];
}

__global__ void __launch_bounds__(kSortThreads) sort_scatter_kernel(const uint32_t* perm_in, uint32_t* perm_out, const uint32_t* keys,
                                                                    int n, int shift, const uint32_t* g_hist, int n_tiles) {
  __shared__ uint16_t s_cnt[kSortChunks][256];   // entries of digit d in chunk c, then exclusive prefix over the chunks
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int tile = blockIdx.x, base = tile * kSortTile;
  for (int j = tid; j < kSortChunks * 256; j += kSortThreads) (&s_cnt[0][0])[j] = 0;
  __syncthreads();
  uint32_t my_perm[kSortChunks / 8], my_rank[kSortChunks / 8];
  uint32_t my_digit[kSortChunks / 8];
#pragma unroll
  for (int r = 0; r < kSortChunks / 8; ++r) {
    const int chunk = r * 8 + warp;
    const int i = base + chunk * 32 + lane;
    const bool live = i < n;
    my_perm[r] = live ? perm_in[i] : 0u;
    const uint32_t d = live ? (keys[my_perm[r]] >> shift) & 255u : 256u + lane;   // dead lanes match nobody
    const unsigned grp = __match_any_sync(0xffffffffu, d);
    my_rank[r] = __popc(grp & ((1u << lane) - 1u));
    my_digit[r] = d;
    if (live && my_rank[r] == 0) s_cnt[chunk][d] = (uint16_t)__popc(grp);
  }
  __syncthreads();
  {   // exclusive prefix over the 64 chunks, one thread per digit
    uint32_t run = 0;
    for (int c = 0; c < kSortChunks; ++c) { uint32_t v = s_cnt[c][tid]; s_cnt[c][tid] = (uint16_t)run; run += v; }
  }
  __syncthreads();
#pragma unroll
  for (int r = 0; r < kSortChunks / 8; ++r) {
    const int chunk = r * 8 + warp;
    const int i = base + chunk * 32 + lane;
    if (i < n) {
      const uint32_t d = my_digit[r];
      perm_out[g_hist[(size_t)d * n_tiles + tile] + s_cnt[chunk][d] + my_rank[r]] = my_perm[r];
    }
  }
}

__global__ void iota_kernel(uint32_t* p, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = (uint32_t)i;
}

// Scratch owned by the caller: perm_tmp[n], g_hist[256 * ceil(n / 2048)].  Result in `perm` (the
// number of passes is made even by sorting a zero digit if needed).  Returns the kernels launched.
static inline int sort_perm_by_key(uint32_t* perm, uint32_t* perm_tmp, const uint32_t* keys, int n, int bits,
                                   uint32_t* g_hist, cudaStream_t stream) {
  if (n <= 1) return 0;
  const int n_tiles = (n + kSortTile - 1) / kSortTile;
  int passes = (bits + 7) / 8;
  if (passes < 1) passes = 1;
  if (passes & 1) passes++;
  uint32_t *src = perm, *dst = perm_tmp;
  for (int p = 0; p < passes; ++p) {
    const int shift = p * 8 < 32 ? p * 8 : 31;   // an extra pass re-sorts by the top bit group: a stable no-op for keys < 2^bits
    const int sh = p * 8 >= 32 ? 31 : shift;
    sort_hist_kernel<<<n_tiles, kSortThreads, 0, stream>>>(src, keys, n, sh, g_hist, n_tiles);
    tile_offsets_kernel<<<1, 1024, 0, stream>>>(g_hist, 256 * n_tiles, nullptr);
    sort_scatter_kernel<<<n_tiles, kSortThreads, 0, stream>>>(src, dst, keys, n, sh, g_hist, n_tiles);
    uint32_t* t = src; src = dst; dst = t;
  }
  return 3 * passes;
}

}  // namespace fpx
