// fpx_common.cuh -- shared layouts and device helpers of the sm_90a kernels.
//
// Everything here is integer scatter/gather + order-preserving prefix logic
// bounded by HBM/L2 bandwidth; there is no GEMM-shaped work, hence no
// wgmma.  What matters (DESIGN.md "kernels"): one 128-bit load per
// message record, fully coalesced warp chunks, at most one 32-byte sector per
// random state access (a proxy-leader row IS one sector for <= 6 voters),
// warp ballots/shuffles/redux for the in-order logic, and PERSISTENT
// cooperative kernels (one wave, grid = SMs x resident CTAs) in which every
// warp owns a contiguous range of the delivery stream: cross-range
// dependencies are resolved by "reduce, grid barrier, apply" instead of a
// per-tile look-back chain.
//
// Reference semantics each kernel reproduces are cited at the kernel.
// S/ = shared/src/main/scala/frankenpaxos/ in mwhittaker/frankenpaxos.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/fpx.h"

namespace fpx {

// ---------------------------------------------------------------------------
// constants / layouts
// ---------------------------------------------------------------------------
constexpr uint32_t kUnarmed = 0xffffffffu;      // row.round_word of a never-armed key
constexpr uint32_t kDoneBit = 0x80000000u;      // row.round_word bit: phase2s entry retired (vanilla Mencius)
constexpr uint32_t kPoison = 0xfffffffeu;       // row.round_word: >1 round of this slot armed -> all its keys live in the table
constexpr uint32_t kBusy = 0xfffffffdu;         // row.round_word: being moved to the table (arm kernel only)
constexpr uint32_t kStampEmpty = 0xffffffffu;   // no Phase2b from this voter yet
constexpr uint64_t kU64Empty = ~0ull;
constexpr uint64_t kCellChosen = 0x8000000000000000ull;  // vanilla Mencius: the server's entry is a ChosenEntry
constexpr int kThreads = 256;                     // threads per CTA of the range kernels
constexpr int kWarps = kThreads / 32;
constexpr int kMaxKeys = FPX_MAX_ACCEPTORS;       // acceptors tracked by the round scan (lane = key)
constexpr int kMaxConflicts = 1024;
constexpr int kSms = 132;                         // H100 SXM; sizes grid-stride launches that need no exact count
constexpr int kMaxGrid = kSms * 8;                // upper bound on CTAs of a cooperative launch
constexpr uint32_t kTsBadVoter = 1u, kTsAnomaly = 2u, kTsPoison = 4u, kTsVanillaRound = 8u;  // DevStatus::ts_flags

// Device-resident status block (one per engine).
struct DevStatus {
  unsigned long long err_word;  // min over errors of (index << 8 | -code); ~0 = none
  int32_t n_p2b, n_nack, n_chosen, watermark;
  uint32_t n_conflicts;         // entries in the conflict list of the running call
  uint32_t ticket;              // last-block-done ticket
  int32_t wm_local;             // replica: first local index not yet chosen
  int32_t max_chosen_local;     // replica: largest local index ever chosen
  int32_t wm_found;             // scratch of the watermark scan
  uint32_t bar_count;           // grid barrier: CTAs arrived at the running barrier (self-resetting)
  uint32_t nack_total;          // acceptor kernel: Nacks of the running call
  uint32_t pad[2];              // [0] second Nack counter (parity), [1] tally: a vote hit a poisoned row
  int32_t max_armed_local;      // largest local slot ever armed
  uint32_t bar_gen;             // grid barrier: generation, bumped by the last CTA to arrive
  // tally: statistics of the running batch (phase A), reset by CTA 0 before the kernel ends
  int32_t ts_min_local, ts_max_local;   // window of local slots the batch's votes touch
  int32_t ts_min_round, ts_max_round;   // rounds carried by the batch's votes
  uint32_t ts_flags;                    // kTsBadVoter | kTsAnomaly
  uint32_t ts_path;                     // path the LAST tally launch took: 1 sweep, 2 exact (diagnostic)
  uint32_t n_arm_conflicts;             // entries in the arm kernel's conflict list
  uint32_t wm_need_scan;                // fused tally: the sweep could not settle the watermark, run the first-hole scan
  unsigned long long t_acceptor[8];  // %globaltimer at the phase boundaries of CTA 0 (profiling aid)
  unsigned long long t_tally[8];
};

__device__ __forceinline__ unsigned long long global_timer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
#define FPX_MARK(arr, k) do { if (blockIdx.x == 0 && threadIdx.x == 0) (arr)[k] = global_timer_ns(); } while (0)

// Multi-GPU exchange (fpx_exchange_*): every engine of a sharded log owns a frontier table
// {epoch:32 | first unchosen global slot:32}[shards]; the kernel that publishes an engine's watermark also
// stores its entry into every peer's table through peer-mapped pointers (NVLink), no collective launch.
constexpr int kMaxShards = 64;
struct DevExchange {
  int32_t enabled, n, mine, pad;
  uint32_t epoch;                       // publications so far
  uint32_t pad2;
  unsigned long long* tabs[kMaxShards]; // tabs[p] = shard p's table as mapped into THIS device (nullptr: not attached)
};
__device__ __forceinline__ void exchange_publish(DevExchange* x, int global_frontier) {
  if (x == nullptr || !x->enabled) return;
  const uint32_t ep = ++x->epoch;
  const unsigned long long v = ((unsigned long long)ep << 32) | (uint32_t)global_frontier;
  for (int p = 0; p < x->n; ++p)
    if (x->tabs[p] != nullptr)
      // the entry IS the message (epoch and frontier in one 64-bit word): no ordering with other data needed
      asm volatile("st.global.relaxed.sys.u64 [%0], %1;" ::"l"(x->tabs[p] + x->mine), "l"(v) : "memory");
}

struct Geometry {
  int32_t protocol, f, groups, per_group, flexible, num_leaders;
  int32_t voters;          // acceptors that can vote on one slot (row width)
  int32_t num_keys;        // total acceptors = groups * per_group
  int32_t quorum;          // f + 1 (count predicate)
  int32_t row_words;       // 8 / 16 / 32 uint32 per proxy-leader row
  int32_t slot_capacity;   // global: one past the last slot of the live window (grows with fpx_retire_below)
  int32_t local_slots;     // rows held by this shard = size of the ring
  int32_t base_local;      // ordinal (slot / shard_count) of the first LIVE local slot; lower ones are retired
  int32_t base_ring;       // base_local % local_slots: where the live window starts in the ring
  int32_t shard_index, shard_count;
  uint32_t ovf_mask;       // overflow_capacity - 1, or 0 with ovf_cap == 0
  int32_t ovf_cap;
  // Lemire fastmod/fastdiv constants (M = ceil(2^64 / d)) for the two runtime
  // divisors on the hot path: numAcceptorGroups and shard_count
  unsigned long long m_groups, m_shards;
  int32_t cell_shift;         // vote cells are 8 << cell_shift bytes apart (vanilla Mencius: cell + batch claim share 16 B)
  int32_t lgroups, agroups;   // FPX_MENCIUS: leader groups, acceptor groups per leader group
  unsigned long long m_lgroups, m_agroups;
};

// a % d and a / d for 0 <= a < 2^31, 1 <= d < 2^31, M = 2^64 / d + 1
// (Lemire, Kaser, Kurz: "Faster remainder by direct computation", 2019)
__device__ __forceinline__ uint32_t fastmod_u32(uint32_t a, unsigned long long M, uint32_t d) {
  unsigned long long low = M * a;
  return (uint32_t)__umul64hi(low, d);
}
__device__ __forceinline__ uint32_t fastdiv_u32(uint32_t a, unsigned long long M) {
  return (uint32_t)__umul64hi(M, a);
}

// ---------------------------------------------------------------------------
// small helpers
// ---------------------------------------------------------------------------
__device__ __forceinline__ int4 ld_stream(const int4* p) {
  // streaming 128-bit load: message records are read exactly once
  int4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.s32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
// L2 eviction-priority policies (createpolicy + .L2::cache_hint)
__device__ __forceinline__ unsigned long long l2_policy_evict_last() {
  unsigned long long pol;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ unsigned long long l2_policy_evict_normal() {
  unsigned long long pol;
  asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ unsigned long long l2_policy_evict_first() {
  unsigned long long pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
// streaming 128-bit store whose line is the first candidate for eviction (written back early)
__device__ __forceinline__ void st_evict_first(int4* p, int4 v, unsigned long long pol) {
  asm volatile("st.global.L1::no_allocate.L2::cache_hint.v4.s32 [%0], {%1,%2,%3,%4}, %5;" ::"l"(p), "r"(v.x), "r"(v.y),
               "r"(v.z), "r"(v.w), "l"(pol));
}
__device__ __forceinline__ int4 ld_keep(const int4* p, unsigned long long pol) {
  int4 r;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.s32 {%0,%1,%2,%3}, [%4], %5;"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p), "l"(pol));
  return r;
}
__device__ __forceinline__ int4 ld_hint(const int4* p, unsigned long long pol) {
  int4 r;
  asm volatile("ld.global.L1::no_allocate.L2::cache_hint.v4.s32 {%0,%1,%2,%3}, [%4], %5;"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p), "l"(pol));
  return r;
}
// 64-bit L2 load tagged evict_last, the policy created in place (it folds into the access's memory
// descriptor): no 64-bit policy register stays live across a loop that runs at the 64-register cap
__device__ __forceinline__ unsigned long long ld_u64_evict_last(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("{ .reg .b64 pol; createpolicy.fractional.L2::evict_last.b64 pol, 1.0; "
               "ld.global.cg.L2::cache_hint.u64 %0, [%1], pol; }"
               : "=l"(v) : "l"(p));
  return v;
}

// Reductions WITHOUT a return value.  atomicMin/atomicMax/atomicOr whose result is unused compile to
// ATOMG with the destination discarded (RZ), which still holds a scoreboard slot and a return packet;
// `red` is the fire-and-forget form (REDG).
__device__ __forceinline__ void red_min_u32(uint32_t* p, uint32_t v) {
  asm volatile("red.global.min.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void red_or_u32(uint32_t* p, uint32_t v) {
  asm volatile("red.global.or.b32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void red_min_u64(unsigned long long* p, unsigned long long v) {
  asm volatile("red.global.min.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ void red_max_u64(unsigned long long* p, unsigned long long v) {
  asm volatile("red.global.max.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ void st_stream(int4* p, int4 v) {
  asm volatile("st.global.L1::no_allocate.v4.s32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y),
               "r"(v.z), "r"(v.w));
}
__device__ __forceinline__ void st_stream2(int2* p, int2 v) {
  asm volatile("st.global.L1::no_allocate.v2.s32 [%0], {%1,%2};" ::"l"(p), "r"(v.x), "r"(v.y));
}
__device__ __forceinline__ unsigned lanemask_lt() {
  unsigned m;
  asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
  return m;
}

__device__ __forceinline__ void report_error(DevStatus* st, int code, long long index) {
  unsigned long long w = ((unsigned long long)index << 8) | (unsigned long long)(unsigned)(-code);
  atomicMin(&st->err_word, w);
}

// State is a RING of local_slots rows over the shard's residue class: ordinal u = slot / shard_count lives at
// ring index u % local_slots while base_local <= u < base_local + local_slots.  fpx_retire_below advances
// base_local behind the chosen watermark and recycles the rows, so a long-lived engine never runs out of slots.
// Three coordinates: ring (addresses), rel = u - base_local (the live window, contiguous), slot (global).
constexpr int kLocalRetired = -2;   // below the live window: chosen and executed long ago
// global slot -> ring index of this shard; -1 out of range / other shard, kLocalRetired
__device__ __forceinline__ int local_slot(const Geometry& g, int slot) {
  if ((uint32_t)slot >= (uint32_t)g.slot_capacity) return -1;
  int u = slot;
  if (g.shard_count != 1) {
    uint32_t q = fastdiv_u32((uint32_t)slot, g.m_shards);
    if ((int)((uint32_t)slot - q * (uint32_t)g.shard_count) != g.shard_index) return -1;
    u = (int)q;
  }
  const int rel = u - g.base_local;
  if (rel < 0) return kLocalRetired;
  if (rel >= g.local_slots) return -1;
  const int ring = rel + g.base_ring;
  return ring >= g.local_slots ? ring - g.local_slots : ring;
}
__device__ __forceinline__ int ring_to_rel(const Geometry& g, int ring) {
  const int rel = ring - g.base_ring;
  return rel < 0 ? rel + g.local_slots : rel;
}
__device__ __forceinline__ int rel_to_ring(const Geometry& g, long long rel) {
  const long long r = rel + g.base_ring;
  return (int)(r >= g.local_slots ? r - g.local_slots : r);
}
__device__ __forceinline__ int rel_to_slot(const Geometry& g, long long rel) {
  return (int)((g.base_local + rel) * g.shard_count + g.shard_index);
}

// index of the vote cell of voter v of local slot `local` in the flat slot x voter array
__device__ __forceinline__ size_t cell_index(const Geometry& g, int local, int v) {
  return ((size_t)local * g.voters + v) << g.cell_shift;
}

// (group, acceptor) -> voter index within the slot's row, or -1.
// non-flexible: the slot's group is slot % numAcceptorGroups
// (S/multipaxos/ProxyLeader.scala:190); flexible: every (row, col) of the grid
// (S/multipaxos/ProxyLeader.scala:118-124).
// The acceptor group a slot's Phase2a goes to, or -1 when any group may see it
// (flexible grid).  multipaxos: slot % numAcceptorGroups (ProxyLeader.scala:190);
// mencius: leader group slot % LG, acceptor group (slot / LG) % AG
// (S/mencius/ProxyLeader.scala:169-176,231-234).
__device__ __forceinline__ int expected_group(const Geometry& g, int slot) {
  if (g.flexible) return -1;
  if (g.protocol == FPX_MENCIUS) {
    uint32_t q = g.lgroups > 1 ? fastdiv_u32((uint32_t)slot, g.m_lgroups) : (uint32_t)slot;
    uint32_t lg = (uint32_t)slot - q * (uint32_t)g.lgroups;
    uint32_t ag = g.agroups > 1 ? fastmod_u32(q, g.m_agroups, (uint32_t)g.agroups) : 0u;
    return (int)(lg * (uint32_t)g.agroups + ag);
  }
  return g.groups > 1 ? (int)fastmod_u32((uint32_t)slot, g.m_groups, (uint32_t)g.groups) : 0;
}
__device__ __forceinline__ int voter_index(const Geometry& g, int group, int acceptor, int slot) {
  if ((uint32_t)acceptor >= (uint32_t)g.per_group) return -1;
  if (g.flexible) return (uint32_t)group < (uint32_t)g.groups ? group * g.per_group + acceptor : -1;
  // mencius' Phase2b carries no group (S/mencius/Mencius.proto): only the index counts
  if (g.protocol == FPX_MENCIUS || g.protocol == FPX_VANILLA_MENCIUS) return acceptor;
  if ((uint32_t)group >= (uint32_t)g.groups || group != expected_group(g, slot)) return -1;
  return acceptor;
}

// Quorum predicate over a voter bitmask: non-flexible `size >= f+1`
// (S/multipaxos/ProxyLeader.scala:238-240); flexible Grid.isWriteQuorum, one
// member of every row (S/quorums/Grid.scala:49).
__device__ __forceinline__ bool write_quorum(const Geometry& g, uint32_t mask) {
  if (!g.flexible) return __popc(mask) >= g.quorum;
  uint32_t rowmask = (1u << g.per_group) - 1u;
  for (int r = 0; r < g.groups; ++r) {
    if (((mask >> (r * g.per_group)) & rowmask) == 0) return false;
  }
  return true;
}
__device__ __forceinline__ bool read_quorum(const Geometry& g, uint32_t mask) {
  // Grid.isReadQuorum: some row entirely inside (S/quorums/Grid.scala:40)
  uint32_t rowmask = (1u << g.per_group) - 1u;
  for (int r = 0; r < g.groups; ++r) {
    if (((mask >> (r * g.per_group)) & rowmask) == rowmask) return true;
  }
  return false;
}

__device__ __forceinline__ uint64_t mix64(uint64_t x) {
  x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; x ^= x >> 33;
  return x;
}

// Proxy-leader row: {u32 round_word; i32 value_id; u32 stamp[voters]; pad}.
// round_word = kUnarmed | round | kDoneBit.  stamp[v] = global sequence number
// of the FIRST Phase2b delivery from voter v for this (slot, round).
struct RowRef {
  uint32_t* p;
  __device__ __forceinline__ uint32_t round_word() const { return p[0]; }
  __device__ __forceinline__ int value_id() const { return (int)p[1]; }
  __device__ __forceinline__ uint32_t* stamps() const { return p + 2; }
  __device__ __forceinline__ unsigned long long* hdr64() const { return (unsigned long long*)p; }
};

struct PLState {
  uint32_t* rows;               // local_slots * row_words
  unsigned long long* ovf_keys; // ovf_cap
  uint32_t* ovf_rows;           // ovf_cap * row_words
};

// Find the row of key (slot, round): the primary row while the slot has a single
// armed round, else (poisoned primary) the open-addressing table.  Returns p ==
// nullptr when the key was never armed (ProxyLeader.scala:220-225 `case None`).
__device__ __forceinline__ uint32_t* table_lookup(const Geometry& g, const PLState& s, int slot, int round) {
  if (g.ovf_cap == 0) return nullptr;
  unsigned long long key = ((unsigned long long)(uint32_t)slot << 32) | (uint32_t)round;
  uint32_t h = (uint32_t)mix64(key) & g.ovf_mask;
  for (int probe = 0; probe < g.ovf_cap; ++probe) {
    unsigned long long k = __ldcg(&s.ovf_keys[h]);
    if (k == key) return s.ovf_rows + (size_t)h * g.row_words;
    if (k == kU64Empty) break;
    h = (h + 1) & g.ovf_mask;
  }
  return nullptr;
}
__device__ __forceinline__ RowRef find_row(const Geometry& g, const PLState& s, int local, int slot, int round) {
  RowRef r{s.rows + (size_t)local * g.row_words};
  uint32_t rw = __ldcg(r.p);
  if (rw == kPoison) return RowRef{table_lookup(g, s, slot, round)};
  if (rw != kUnarmed && rw != kBusy && (int)(rw & ~kDoneBit) == round) return r;
  return RowRef{nullptr};
}

// ---------------------------------------------------------------------------
// Grid barrier for cooperative (co-resident) launches: arrival counter + generation.
// The last CTA to arrive resets the counter and bumps the generation, so the barrier
// needs no per-launch bookkeeping on the host (any number of barriers per launch,
// data-dependent paths included, as long as every CTA takes the same path).
// ---------------------------------------------------------------------------
__device__ __forceinline__ void grid_sync(DevStatus* st) {
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t gen, v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(gen) : "l"(&st->bar_gen) : "memory");
    __threadfence();
    if (atomicAdd(&st->bar_count, 1u) == gridDim.x - 1) {
      st->bar_count = 0;
      __threadfence();
      asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(&st->bar_gen) : "memory");
    } else {
      do {
        asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(&st->bar_gen) : "memory");
      } while (v == gen);
    }
    __threadfence();
  }
  __syncthreads();
}

// Contiguous range of the delivery stream owned by the calling warp: warp gw of
// the grid owns [gw*per, (gw+1)*per), per a multiple of 32, so a CTA owns a
// contiguous range too and ranges are ordered by (blockIdx, warp).
__device__ __forceinline__ int warp_range_len(int n) {
  int total_warps = gridDim.x * kWarps;
  return (((n + total_warps - 1) / total_warps) + 31) & ~31;
}
__device__ __forceinline__ int4 ld_cg(const int4* p) { return __ldcg(p); }

__device__ __forceinline__ int warp_incl_scan_max(int v, int lane) {
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    int o = __shfl_up_sync(0xffffffffu, v, d);
    if (lane >= d) v = max(v, o);
  }
  return v;
}

}  // namespace fpx
