// fpx_reads.cuh -- MultiPaxos linearizable reads (include/fpx.h fpx_reads_*).
//
//   Read tally (Client.handleMaxSlotReply, S/multipaxos/Client.scala:851-931; ReadBatcher.
//   handleBatchMaxSlotReply, S/multipaxos/ReadBatcher.scala:568-623).  Resident state per read
//   key: a ReadRow {id, state, mask of the voters heard from, ...} and one 64-bit cell per voter
//   {stamp:32 | slot:32} holding that voter's LATEST reply.  One batch of replies:
//     keys      sort key = the read key (unknown keys sort last and are skipped)
//     sort      stable radix sort by key (fpx_sort.cuh): per-key segments in delivery order
//     scan<0>   tiles of 1024 sorted replies: segmented OR of the replies' voter bits -> tile aggregates
//     carry     one CTA (tile_carry_kernel): exclusive segmented scan of the tile aggregates (a
//               segment may span any number of tiles)
//     scan<1>   the same OR with the carry: the reply at which the quorum predicate first holds
//               completes the read (cpos); later replies of the read are ignored
//     cells     every counted reply (<= cpos) stores {delivery index + 1, slot} with a 64-bit max:
//               the latest reply of each voter wins, whatever order the sort visits them in
//     settle    one thread per segment: slot = max over the voters in the mask of their latest
//               slot (+ numAcceptorGroups - 1), the record parked at the completing reply's index;
//               stamps are cleared to 0 so replies of later batches are newer
//     compact   completions in the order of the completing reply's delivery index
//
//   Deferred reads (Replica.handleDeferrableRead(s), S/multipaxos/Replica.scala:463-529, and
//   executeLog's processDeferredReads, :394-413).  A slot-sorted pending pool in a ring of
//   pow2 >= pending_capacity {slot, handle} entries, live positions [head, tail), equal slots in
//   arrival order.  A batch: classify against W (tile counts), plan (one CTA: overflow check,
//   counts), one stable sort whose key puts the immediate reads first in delivery order and the
//   deferred ones after them by slot, then the deferred run D is merged with the pool's tail T
//   (entries whose slot > D's smallest slot; usually few, since read slots follow the log) by
//   a rank computed with two binary searches per entry.  Advance: binary search of the first
//   entry with slot >= W', release the prefix.  All counts live on the device (the _dev forms).
#pragma once
#include "fpx_common.cuh"
#include "fpx_scan.cuh"
#include "fpx_sort.cuh"

namespace fpx {

constexpr int kRdTile = 1024;                     // sorted replies per scan CTA, reads per classify CTA
constexpr int kRdOpen = 1, kRdDone = 2;           // ReadRow::state (0: never opened)
constexpr long long kRdNoIndex = (1ll << 55) - 1; // err_word index of an error that belongs to no record

struct ReadRow {
  int32_t id, state;
  uint32_t mask;      // voters whose latest reply is in cells[]
  uint32_t newmask;   // scratch of the running batch: mask at completion / at the segment's end
  int32_t cpos;       // scratch: sorted position of the completing reply, -1 none
  int32_t pad[3];
};

struct ReadsDev {
  unsigned long long err_word;   // min over errors of (index << 8 | -code); ~0 = none
  int32_t n_slots, n_replies, n_released;   // output counts of the last tally / replica / advance
  int32_t watermark;             // the replica's executedWatermark W
  uint32_t head, tail;           // pending pool, logical positions
  uint32_t tail_old;             // replica call: tail before the batch
  uint32_t merge_at;             // replica call: first pool position whose slot > the smallest deferred slot
  int32_t n_imm, n_def;          // replica call: immediate / deferred reads
  int32_t abort;                 // the running call failed its check: later kernels do nothing
  uint32_t rel_from;             // advance: first released position
};

__device__ __forceinline__ void reads_error(ReadsDev* st, int code, long long index) {
  atomicMin(&st->err_word, ((unsigned long long)index << 8) | (unsigned long long)(unsigned)(-code));
}

struct ReadTallyParams {
  const int4* in;                // fpx_max_slot_reply {key, id, voter, slot}
  int n, cap, kind, voters, quorum, flexible, groups, per_group;
  int32_t slot_add;              // numAcceptorGroups - 1, or 0 (flexible Client)
  ReadRow* rows;
  unsigned long long* cells;     // cap x voters
  uint32_t *skey, *perm;
  uint32_t* tile_agg;            // OR since the tile's last head
  uint32_t* tile_head;           // the tile has a segment head
  uint32_t* carry;               // OR flowing into the tile from earlier tiles
  uint32_t* flag;                // [n] reply i completed its read
  int4* parked;                  // [n] the completion record of reply i
  uint32_t* tile_cnt;            // compaction
  int4* out;
  ReadsDev* st;
};

// voter index of a reply in its read's row, -1 if it names no acceptor of the config.  Client: (group,
// acceptor) (Client.scala:877-879); ReadBatcher: acceptorIndex only (ReadBatcher.scala:584), the group
// is not part of the key.
__device__ __forceinline__ int reads_voter(const ReadTallyParams& P, int word) {
  const uint32_t group = (uint32_t)word >> 16, acc = (uint32_t)word & 0xffffu;
  if (acc >= (uint32_t)P.per_group) return -1;
  if (P.kind == FPX_READS_READ_BATCHER) return (int)acc;
  return group < (uint32_t)P.groups ? (int)(group * P.per_group + acc) : -1;
}
// Client flexible: Grid.isReadQuorum (Client.scala:883-887, S/quorums/Grid.scala:35-41); every other
// case `size >= f+1` (Client.scala:880, ReadBatcher.scala:585, flexible or not)
__device__ __forceinline__ bool reads_quorum(const ReadTallyParams& P, uint32_t mask) {
  if (P.kind == FPX_READS_CLIENT && P.flexible) {
    const uint32_t rowmask = (1u << P.per_group) - 1u;
    for (int r = 0; r < P.groups; ++r)
      if (((mask >> (r * P.per_group)) & rowmask) == rowmask) return true;
    return false;
  }
  return __popc(mask) >= P.quorum;
}

__global__ void reads_keys_kernel(ReadTallyParams P) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P.n) return;
  const int key = P.in[i].x;
  P.skey[i] = (uint32_t)key < (uint32_t)P.cap ? (uint32_t)key : (uint32_t)P.cap;
  P.flag[i] = 0;
}

template <int kPass>
__global__ void __launch_bounds__(kRdTile) reads_scan_kernel(ReadTallyParams P) {
  __shared__ uint32_t s_incl[kRdTile];
  const int j = blockIdx.x * kRdTile + threadIdx.x;
  const bool live = j < P.n;
  const int i = live ? (int)P.perm[j] : 0;
  const uint32_t k = live ? P.skey[i] : (uint32_t)P.cap;
  const bool keyed = k < (uint32_t)P.cap;
  const bool head = live && (j == 0 || P.skey[P.perm[j - 1]] != k);
  bool valid = false;
  int v = -1;
  uint32_t val = 0, rmask = 0;
  if (keyed) {
    const int4 rec = P.in[i];
    const ReadRow row = P.rows[k];
    rmask = row.mask;
    // a reply for a read that is not open, already complete, or of another id is ignored
    // (Client.scala:858-874, ReadBatcher.scala:572-580)
    valid = row.state == kRdOpen && rec.y == row.id;
    v = reads_voter(P, rec.z);
    if (valid && v >= 0) val = 1u << v;
    if (head) val |= rmask;
  }
  const SegVal<uint32_t> x = cta_scan<kRdTile, false>(SegVal<uint32_t>{val, head}, Seg<ScanOr>());
  uint32_t incl = x.v;
  if (kPass == 0) {
    if (threadIdx.x == kRdTile - 1) { P.tile_agg[blockIdx.x] = incl; P.tile_head[blockIdx.x] = x.f; }
    return;
  }
  if (!x.f) incl |= P.carry[blockIdx.x];
  s_incl[threadIdx.x] = incl;
  __syncthreads();
  if (!keyed) return;
  const uint32_t excl = head ? rmask : (threadIdx.x == 0 ? P.carry[blockIdx.x] : s_incl[threadIdx.x - 1]);
  const bool before = reads_quorum(P, excl);
  if (valid && !before) {
    if (v < 0) {
      reads_error(P.st, FPX_ERR_BAD_ACCEPTOR, i);   // Grid.isReadQuorum's `require`
    } else if (reads_quorum(P, incl)) {
      P.rows[k].cpos = j;
      P.rows[k].newmask = incl;
    }
  }
  const bool last = j == P.n - 1 || P.skey[P.perm[j + 1]] != k;
  if (last && !reads_quorum(P, incl)) P.rows[k].newmask = incl;
}

__global__ void reads_cells_kernel(ReadTallyParams P) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= P.n) return;
  const int i = (int)P.perm[j];
  const uint32_t k = P.skey[i];
  if (k >= (uint32_t)P.cap) return;
  const int4 rec = P.in[i];
  const ReadRow row = P.rows[k];
  if (row.state != kRdOpen || rec.y != row.id || (row.cpos >= 0 && j > row.cpos)) return;
  const int v = reads_voter(P, rec.z);
  if (v < 0) return;
  // overwrites: the latest reply of each voter (Client.scala:877-879, ReadBatcher.scala:584)
  atomicMax(&P.cells[(size_t)k * P.voters + v], ((unsigned long long)(uint32_t)(i + 1) << 32) | (uint32_t)rec.w);
}

__global__ void reads_settle_kernel(ReadTallyParams P) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= P.n) return;
  const int i = (int)P.perm[j];
  const uint32_t k = P.skey[i];
  if (k >= (uint32_t)P.cap || (j > 0 && P.skey[P.perm[j - 1]] == k)) return;
  ReadRow& row = P.rows[k];
  if (row.state != kRdOpen) return;
  const uint32_t mask = row.newmask;
  unsigned long long* c = P.cells + (size_t)k * P.voters;
  int mx = INT32_MIN;
  for (uint32_t m = mask; m; m &= m - 1) {
    const int v = __ffs(m) - 1;
    const unsigned long long x = c[v];
    mx = max(mx, (int)(uint32_t)x);
    c[v] = x & 0xffffffffull;
  }
  row.mask = mask;
  if (row.cpos >= 0) {
    // Client.scala:892-898, ReadBatcher.scala:592-598; JVM Int arithmetic
    const int slot = (int)((uint32_t)mx + (uint32_t)P.slot_add);
    const int ic = (int)P.perm[row.cpos];
    P.parked[ic] = make_int4((int)k, row.id, slot, 0);
    P.flag[ic] = 1;
    row.state = kRdDone;   // Client: PendingRead; ReadBatcher: batchMaxSlotReplies.remove (:601)
  }
  row.cpos = -1;
}

__global__ void __launch_bounds__(1024) reads_count_kernel(const uint32_t* flag, int n, uint32_t* tile_cnt) {
  const int i = blockIdx.x * 1024 + threadIdx.x;
  const int cnt = __syncthreads_count(i < n && flag[i]);   // flags are 0 or 1
  if (threadIdx.x == 0) tile_cnt[blockIdx.x] = (uint32_t)cnt;
}

// out[tile_off + rank] = parked[i] for every flagged i
__global__ void __launch_bounds__(1024) reads_compact_kernel(const uint32_t* flag, const int4* parked, int n,
                                                             const uint32_t* tile_off, int4* out) {
  const int i = blockIdx.x * 1024 + threadIdx.x;
  const uint32_t f = i < n ? flag[i] : 0u;
  const uint32_t r = cta_scan<1024, true>(f, ScanSum()) + tile_off[blockIdx.x];
  if (f) out[r] = parked[i];
}

// ---------------------------------------------------------------------------------- deferred reads

struct DeferredParams {
  const int2* in;        // fpx_read_request {slot, handle}
  int n;
  int32_t pending_cap;
  uint32_t ring_mask;
  int2* pool;            // ring of {slot, handle}
  int2* tmp;             // [pending_cap] the pool's tail T during a merge
  int2* def;             // [n] the batch's deferred reads by slot
  uint32_t *skey, *perm, *tile_cnt;
  int4* out;             // fpx_read_reply {handle, reply_slot, after_slot, 0}
  ReadsDev* st;
};

// A read with slot < W is answered now; any other one waits for slot (Replica.scala:463, 491)
__global__ void __launch_bounds__(1024) rep_classify_kernel(DeferredParams P) {
  const int i = blockIdx.x * 1024 + threadIdx.x;
  const int W = P.st->watermark;
  bool def = false;
  if (i < P.n) {
    const int slot = P.in[i].x;
    def = slot >= W;
    // immediates first in delivery order, then the deferred reads by slot (slot >= W >= 0: slot + 1 fits)
    P.skey[i] = def ? (uint32_t)slot + 1u : 0u;
  }
  const int cnt = __syncthreads_count(def);
  if (threadIdx.x == 0) P.tile_cnt[blockIdx.x] = (uint32_t)cnt;
}

// One CTA: total deferred reads, the pool's capacity check (FPX_ERR_OVERFLOW_FULL at the first deferred read
// that does not fit, nothing of the batch applied), the call's counts.
__global__ void __launch_bounds__(1024) rep_plan_kernel(DeferredParams P, int tiles) {
  __shared__ uint32_t s_hit_tile, s_hit_base;
  ReadsDev* st = P.st;
  const uint32_t live = st->tail - st->head;
  const uint32_t free_ = (uint32_t)P.pending_cap - live;
  uint32_t m = 0;   // deferred reads of the tiles scanned so far
  for (int base = 0; base < tiles; base += 1024) {
    const int t = base + threadIdx.x;
    const uint32_t c = t < tiles ? P.tile_cnt[t] : 0u;
    uint32_t total;
    const uint32_t off = cta_scan<1024, true>(c, ScanSum(), &total) + m;
    if (c > 0 && off <= free_ && free_ < off + c) { s_hit_tile = t; s_hit_base = off; }
    m += total;
  }
  __syncthreads();
  if (m <= free_) {
    if (threadIdx.x == 0) {
      st->abort = 0;
      st->n_def = (int)m;
      st->n_imm = P.n - (int)m;
      st->n_replies = P.n - (int)m;
      st->tail_old = st->tail;
      st->tail += m;
    }
    return;
  }
  // the deferred read of rank free_ (delivery order) lies in tile s_hit_tile
  const int i = (int)s_hit_tile * 1024 + threadIdx.x;
  const bool def = i < P.n && P.skey[i] != 0u;
  const uint32_t r = cta_scan<1024, true>(def ? 1u : 0u, ScanSum()) + s_hit_base;
  if (def && r == free_) reads_error(st, FPX_ERR_OVERFLOW_FULL, i);
  if (threadIdx.x == 0) { st->abort = 1; st->n_replies = 0; }
}

// first logical pool position in [lo, hi) whose slot > s (upper) or >= s
__device__ __forceinline__ uint32_t pool_bound(const int2* pool, uint32_t mask, uint32_t lo, uint32_t hi, int s, bool upper) {
  while (lo != hi) {
    const uint32_t mid = lo + (hi - lo) / 2;
    const int x = pool[mid & mask].x;
    if (upper ? x <= s : x < s) lo = mid + 1; else hi = mid;
  }
  return lo;
}
__device__ __forceinline__ int array_bound(const int2* a, int n, int s, bool upper) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (upper ? a[mid].x <= s : a[mid].x < s) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// Immediate replies {handle, W - 1, W - 1, 0} (Replica.scala:521-527), the deferred run D by slot, and
// the pool's tail T (entries with slot > D's smallest slot: entries with an equal slot arrived earlier
// and stay in front) copied aside for the merge.  Grid-stride: the counts are on the device.
__global__ void rep_emit_kernel(DeferredParams P) {
  __shared__ uint32_t s_p;
  const ReadsDev* st = P.st;
  if (st->abort) return;
  const int n_imm = st->n_imm, n_def = st->n_def, W = st->watermark;
  const uint32_t tail = st->tail_old;
  if (threadIdx.x == 0) {
    s_p = n_def > 0 ? pool_bound(P.pool, P.ring_mask, st->head, tail, P.in[P.perm[n_imm]].x, true) : tail;
    if (blockIdx.x == 0) P.st->merge_at = s_p;
  }
  __syncthreads();
  const uint32_t p = s_p;
  const int t = (int)(tail - p);
  const int stride = gridDim.x * blockDim.x;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < P.n; j += stride) {
    const int2 r = P.in[P.perm[j]];
    if (j < n_imm) P.out[j] = make_int4(r.y, W - 1, W - 1, 0);
    else P.def[j - n_imm] = r;
  }
  for (int q = blockIdx.x * blockDim.x + threadIdx.x; q < t; q += stride) P.tmp[q] = P.pool[(p + (uint32_t)q) & P.ring_mask];
}

// merge T and D into the pool from merge_at on: a T entry goes after the D entries with a smaller slot,
// a D entry after the T entries with a slot <= its own (T arrived first)
__global__ void rep_merge_kernel(DeferredParams P) {
  const ReadsDev* st = P.st;
  if (st->abort) return;
  const uint32_t p = st->merge_at;
  const int t = (int)(st->tail_old - p), m = st->n_def;
  const int stride = gridDim.x * blockDim.x;
  for (int x = blockIdx.x * blockDim.x + threadIdx.x; x < t + m; x += stride) {
    int2 e;
    int pos;
    if (x < t) { e = P.tmp[x]; pos = x + array_bound(P.def, m, e.x, false); }
    else { e = P.def[x - t]; pos = (x - t) + array_bound(P.tmp, t, e.x, true); }
    P.pool[(p + (uint32_t)pos) & P.ring_mask] = e;
  }
}

// executeLog up to W' (Replica.scala:394-413): the pool's entries with slot < W' leave in (slot, arrival)
// order; W' < W is FPX_ERR_INVALID_ARG.  d_w: the watermark on the device (fpx_step_dev's d_watermark),
// else w.
__global__ void rep_advance_plan_kernel(DeferredParams P, const int32_t* d_w, int32_t w) {
  ReadsDev* st = P.st;
  const int W2 = d_w ? *d_w : w;
  if (W2 < st->watermark) {
    reads_error(st, FPX_ERR_INVALID_ARG, kRdNoIndex);
    st->abort = 1;
    st->n_released = 0;
    return;
  }
  const uint32_t end = pool_bound(P.pool, P.ring_mask, st->head, st->tail, W2, false);
  st->abort = 0;
  st->rel_from = st->head;
  st->n_released = (int)(end - st->head);
  st->head = end;
  st->watermark = W2;
}

// a released read runs right after log entry `slot`, before executedWatermark += 1: ReadReply.slot = slot - 1
// (Replica.scala:405-413, 521-527)
__global__ void rep_advance_emit_kernel(DeferredParams P) {
  const ReadsDev* st = P.st;
  if (st->abort) return;
  const int k = st->n_released;
  const uint32_t from = st->rel_from;
  for (int q = blockIdx.x * blockDim.x + threadIdx.x; q < k; q += gridDim.x * blockDim.x) {
    const int2 e = P.pool[(from + (uint32_t)q) & P.ring_mask];
    P.out[q] = make_int4(e.y, e.x - 1, e.x, 0);
  }
}

// fpx_reads_open: the last record of a key in the batch wins
__global__ void reads_open_claim_kernel(const int2* in, int n, int32_t* claim) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) atomicMax(&claim[in[i].x], i);
}
__global__ void reads_open_apply_kernel(const int2* in, int n, int32_t* claim, ReadRow* rows) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int key = in[i].x;
  if (claim[key] != i) return;
  ReadRow& r = rows[key];
  r.id = in[i].y; r.state = kRdOpen; r.mask = 0; r.cpos = -1;   // MaxSlot(id, {}) (Client.scala:652-660)
  claim[key] = -1;
}

}  // namespace fpx
