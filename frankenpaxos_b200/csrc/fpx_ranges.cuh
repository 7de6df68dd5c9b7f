// fpx_ranges.cuh -- range-fill variants of the vote path (SURVEY 8(f) rank 3):
//
//   S/mencius   Phase2aNoopRange / Phase2bNoopRange / ChosenNoopRange
//     ProxyLeader.handlePhase2aNoopRange   S/mencius/ProxyLeader.scala:255-303   range_arm_kernel
//     Acceptor.handlePhase2aNoopRange      S/mencius/Acceptor.scala:237-291      range_acceptor_kernel + range_fill_kernel
//     ProxyLeader.handlePhase2bNoopRange   S/mencius/ProxyLeader.scala:355-412   range_tally_kernel
//     Replica.handleChosenNoopRange        S/mencius/Replica.scala:464-486       replica_range_{first,fill}_kernel
//   S/vanillamencius   Skip
//     Server.advanceWithSkips (log fill) / handleSkip   S/vanillamencius/Server.scala:577-620, 1144-1168   vm_skip_kernel
//
// A leader group that lags the others closes its gap with ONE message that stands
// for a strided run of Noop slots.  The messages are few (one per lag event), the
// slots they cover are many: the per-message logic (round compare, key table,
// quorum-in-every-group tally) runs in one CTA in delivery order, the per-slot
// effects are coalesced strided fills over the same vote cells / replica log the
// single-slot kernels use, one (record, chunk) tile per CTA.
#pragma once
#include "fpx_common.cuh"
#include "fpx_scan.cuh"

namespace fpx {

// ---------------------------------------------------------------------------
// (slotStart, slotEnd, round) key table of the proxy leader
// (S/mencius/ProxyLeader.scala:86-90 SlotRound; :101-106 PendingPhase2aNoopRange).
// Entry = {state, start, end, round, stamp[32]}: stamp[ag * per_group + a] is the
// delivery sequence number of the first Phase2bNoopRange of acceptor a of acceptor
// group ag, exactly like a proxy-leader row's stamps.
// ---------------------------------------------------------------------------
constexpr int kRangeWords = 36;
constexpr uint32_t kRangeEmpty = 0xffffffffu, kRangeBusy = 0xfffffffdu, kRangePending = 0u, kRangeDone = 1u;
constexpr int32_t kNoHit = 0x7f7f7f7f;    // cudaMemset(0x7f) pattern: "no slot of the range is in the log"

struct RangeTable {
  uint32_t* ent;     // cap * kRangeWords
  uint32_t mask;     // cap - 1
  int32_t cap;
};

__device__ __forceinline__ uint32_t range_hash(int start, int end, int round) {
  return (uint32_t)mix64(((unsigned long long)(uint32_t)start << 32 | (uint32_t)end) * 0x9e3779b97f4a7c15ull +
                         (uint32_t)round);
}
// the entry of a key, or nullptr
__device__ __forceinline__ uint32_t* range_find(const RangeTable& t, int start, int end, int round) {
  uint32_t h = range_hash(start, end, round) & t.mask;
  for (int probe = 0; probe < t.cap; ++probe) {
    uint32_t* e = t.ent + (size_t)h * kRangeWords;
    uint32_t s = *(volatile uint32_t*)e;
    while (s == kRangeBusy) s = *(volatile uint32_t*)e;
    if (s == kRangeEmpty) return nullptr;
    __threadfence();
    if ((int)__ldcg(e + 1) == start && (int)__ldcg(e + 2) == end && (int)__ldcg(e + 3) == round) return e;
    h = (h + 1) & t.mask;
  }
  return nullptr;
}
// insert-if-absent; returns nullptr when the table is full.  *used counts the occupied entries.
__device__ __forceinline__ uint32_t* range_insert(const RangeTable& t, int start, int end, int round, uint32_t* used) {
  uint32_t h = range_hash(start, end, round) & t.mask;
  for (int probe = 0; probe < t.cap; ++probe) {
    uint32_t* e = t.ent + (size_t)h * kRangeWords;
    uint32_t s = atomicCAS(e, kRangeEmpty, kRangeBusy);
    if (s == kRangeEmpty) {
      e[1] = (uint32_t)start; e[2] = (uint32_t)end; e[3] = (uint32_t)round;
      __threadfence();
      atomicExch(e, kRangePending);
      red_add_u32(used, 1u);
      return e;
    }
    while (s == kRangeBusy) s = *(volatile uint32_t*)e;
    __threadfence();
    if ((int)__ldcg(e + 1) == start && (int)__ldcg(e + 2) == end && (int)__ldcg(e + 3) == round) return e;
    h = (h + 1) & t.mask;
  }
  return nullptr;
}

// A non-empty range that lies below base_local * shard_count: every slot of it that this shard holds was
// retired by fpx_retire_below (with one shard: every slot of it).  Its key is Done for good -- it leaves the
// table at the next retire and a late arm does not bring it back.
__device__ __forceinline__ bool range_retired(const Geometry& g, int start, int end) {
  return start < end && (long long)end <= (long long)g.base_local * g.shard_count;
}

// fpx_retire_below: the range table rebuilt into its spare copy (preset to ~0), like ovf_rebuild_kernel: the
// entries of ranges that are not retired under the new geometry g move, whole, to the first free entry of
// their probe sequence; `used` counts them.  One thread per entry.
__global__ void __launch_bounds__(256) range_rebuild_kernel(Geometry g, RangeTable from, uint32_t* to, uint32_t* used) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= from.cap) return;
  const uint32_t* e = from.ent + (size_t)i * kRangeWords;
  const uint32_t state = e[0];
  if (state == kRangeEmpty || range_retired(g, (int)e[1], (int)e[2])) return;
  uint32_t h = range_hash((int)e[1], (int)e[2], (int)e[3]) & from.mask;
  while (atomicCAS(to + (size_t)h * kRangeWords, kRangeEmpty, state) != kRangeEmpty) h = (h + 1) & from.mask;
  for (int w = 1; w < kRangeWords; ++w) to[(size_t)h * kRangeWords + w] = e[w];
  atomicAdd(used, 1u);
}

__device__ __forceinline__ int range_precheck(const Geometry& g, int start, int end, int round) {
  if (start < 0 || end < start || end > g.slot_capacity) return FPX_ERR_SLOT_RANGE;
  if ((uint32_t)round > (uint32_t)FPX_MAX_ROUND) return FPX_ERR_ROUND_RANGE;
  return FPX_OK;
}
// dst = group << 16 | acceptor with group = leader_group * agroups + acceptor_group: the acceptor
// must belong to the leader group that owns the range's slots (slotSystem.leader(slotStartInclusive))
__device__ __forceinline__ bool range_dst_ok(const Geometry& g, int dst, int start) {
  int grp = dst >> 16, a = dst & 0xffff;
  if ((uint32_t)grp >= (uint32_t)g.groups || a >= g.per_group) return false;
  return grp / g.agroups == start % g.lgroups;
}

// ---------------------------------------------------------------------------
// ProxyLeader.handlePhase2aNoopRange (:255-303): states.get(SlotRound(start, end, round)):
// Some(_) -> ignore, None -> PendingPhase2aNoopRange with one empty map per acceptor group.
// A range of one slot shares its key with that slot's Phase2a (:217-219), so it is
// also ignored when the (slot, round) key is armed.  in {start, end, round, _}.
// ---------------------------------------------------------------------------
struct RangeArmParams {
  Geometry g;
  PLState pl;
  RangeTable tab;
  const int4* in;
  int32_t n;
  DevStatus* st;
};

__global__ void __launch_bounds__(256) range_arm_kernel(RangeArmParams P) {
  const Geometry& g = P.g;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < P.n; i += gridDim.x * blockDim.x) {
    int4 rec = P.in[i];
    int c = range_precheck(g, rec.x, rec.y, rec.z);
    if (c != FPX_OK) { report_error(P.st, c, i); continue; }
    if (range_retired(g, rec.x, rec.y)) continue;   // the key is Done (or was never needed): `case Some(_)`
    if (rec.y == rec.x + 1) {
      int l = local_slot(g, rec.x);
      if (l >= 0 && find_row(g, P.pl, l, rec.x, rec.z).p != nullptr) continue;   // `case Some(_)`
    }
    if (range_insert(P.tab, rec.x, rec.y, rec.z, &P.st->rng_used) == nullptr) report_error(P.st, FPX_ERR_OVERFLOW_FULL, i);
  }
}

// ---------------------------------------------------------------------------
// Acceptor.handlePhase2aNoopRange (:237-291), the per-message part.  The acceptor's
// `round` is shared with handlePhase2a, so a batch of ranges runs the same keyed
// running maximum: record i is accepted iff round_i >= max(round of the acceptor
// before the batch, rounds of the earlier records of the same acceptor).  ONE CTA of
// 32 warps: warp k scans the whole batch for acceptor k (lane = record, inclusive
// max-scan by shuffles), then the CTA compacts the replies in delivery order.
//   in  {start, end, round, dst}      out {dst, start, end, round}   nack {leader, round}
//   dec[i] = -1 accepted | nack round (>= 1) | -2 invalid record
// ---------------------------------------------------------------------------
constexpr int kRangeCtaThreads = 1024;
constexpr int32_t kDecInvalid = -2, kDecAccept = -1;

struct RangeAcceptorParams {
  Geometry g;
  const int4* in;
  int32_t n;
  int4* out;
  int2* out_nack;
  int32_t* dec;
  int32_t* acc_round;
  DevStatus* st;
};

// ordered two-stream compaction shared by the one-CTA kernels: returns this thread's
// output position in stream a (flag a) or b (flag b); totals accumulate in s_tot[2]
struct CtaCompactor {
  int* s_cnt;   // [2][32]
  int* s_tot;   // [2]
  __device__ __forceinline__ void pos(bool a, bool b, int lane, int warp, int& pa, int& pb) {
    unsigned ba = __ballot_sync(0xffffffffu, a), bb = __ballot_sync(0xffffffffu, b);
    if (lane == 0) { s_cnt[warp] = __popc(ba); s_cnt[32 + warp] = __popc(bb); }
    __syncthreads();
    int oa = s_tot[0], ob = s_tot[1];
    for (int w = 0; w < warp; ++w) { oa += s_cnt[w]; ob += s_cnt[32 + w]; }
    pa = oa + __popc(ba & lanemask_lt());
    pb = ob + __popc(bb & lanemask_lt());
    __syncthreads();
    if (threadIdx.x == 0) {
      int ta = 0, tb = 0;
      for (int w = 0; w < 32; ++w) { ta += s_cnt[w]; tb += s_cnt[32 + w]; }
      s_tot[0] += ta; s_tot[1] += tb;
    }
    __syncthreads();
  }
};

__global__ void __launch_bounds__(kRangeCtaThreads) range_acceptor_kernel(RangeAcceptorParams P) {
  const Geometry& g = P.g;
  __shared__ int s_cnt[64];
  __shared__ int s_tot[2];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid < 2) s_tot[tid] = 0;
  // phase 0: preconditions
  for (int i = tid; i < P.n; i += kRangeCtaThreads) {
    int4 rec = P.in[i];
    int c = range_precheck(g, rec.x, rec.y, rec.z);
    if (c == FPX_OK && !range_dst_ok(g, rec.w, rec.x)) c = FPX_ERR_BAD_ACCEPTOR;
    if (c != FPX_OK) report_error(P.st, c, i);
    P.dec[i] = c == FPX_OK ? 0 : kDecInvalid;
  }
  __syncthreads();
  // phase 1: warp k = acceptor k
  if (warp < g.num_keys) {
    int cur = P.acc_round[warp];
    for (int base = 0; base < P.n; base += 32) {
      const int i = base + lane;
      bool match = false;
      int r = -1;
      if (i < P.n) {
        int4 rec = P.in[i];
        match = range_precheck(g, rec.x, rec.y, rec.z) == FPX_OK && range_dst_ok(g, rec.w, rec.x) &&
                (rec.w >> 16) * g.per_group + (rec.w & 0xffff) == warp;
        if (match) r = rec.z;
      }
      const int incl = warp_incl_scan<ScanMax>(r, lane);
      const int before = max(cur, warp_excl(incl, lane, -1));  // the acceptor's round when record i is delivered
      if (match) P.dec[i] = r >= before ? kDecAccept : before; // `phase2a.round < round` -> Nack(round) (:245-254)
      cur = max(cur, __shfl_sync(0xffffffffu, incl, 31));      // round = phase2a.round (:259)
    }
    if (lane == 0) P.acc_round[warp] = cur;
  }
  __syncthreads();
  // phase 2: replies in delivery order
  CtaCompactor cc{s_cnt, s_tot};
  for (int base = 0; base < P.n; base += kRangeCtaThreads) {
    const int i = base + tid;
    int d = kDecInvalid;
    int4 rec = make_int4(0, 0, 0, 0);
    if (i < P.n) { d = P.dec[i]; rec = P.in[i]; }
    int pa, pb;
    cc.pos(d == kDecAccept, d >= 0, lane, warp, pa, pb);
    if (d == kDecAccept) P.out[pa] = make_int4(rec.w, rec.x, rec.y, rec.z);   // Phase2bNoopRange (:279-290)
    // leaders(slotSystem.leader(slotStartInclusive))(roundSystem.leader(round)) (:250-252)
    if (d >= 0) P.out_nack[pb] = make_int2(rec.z % g.num_leaders + (rec.x % g.lgroups) * g.num_leaders, d);
  }
  if (tid == 0) { P.st->n_p2b = s_tot[0]; P.st->n_nack = s_tot[1]; }
}

// The per-slot part (:263-277): the slots of [start, end) that belong to the range's leader
// group (slot = start mod LG) AND to this acceptor's group ((slot / LG) % AG == ag) get
// State(round, Noop): first such slot start + m0 * LG, stride LG * AG.  grid = (chunks, records).
struct RangeFillParams {
  Geometry g;
  const int4* in;
  const int32_t* dec;
  unsigned long long* votes;
};

__global__ void __launch_bounds__(256) range_fill_kernel(RangeFillParams P) {
  const Geometry& g = P.g;
  const int j = blockIdx.y;
  if (P.dec[j] != kDecAccept) return;
  const int4 rec = P.in[j];
  const int a = rec.w & 0xffff, ag = (rec.w >> 16) % g.agroups;
  const long long LG = g.lgroups, AG = g.agroups;
  const long long m0 = ((ag - (rec.x / LG) % AG) % AG + AG) % AG;
  const long long first = rec.x + m0 * LG, stride = LG * AG;
  const long long count = first < rec.y ? (rec.y - first + stride - 1) / stride : 0;
  const unsigned long long cell = ((unsigned long long)(uint32_t)(rec.z + 1) << 32) | (uint32_t)FPX_VALUE_NOOP;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < count; t += (long long)gridDim.x * blockDim.x) {
    int l = local_slot(g, (int)(first + t * stride));
    if (l >= 0) red_max_u64(&P.votes[cell_index(g, l, a)], cell);   // states(slot) = State(round, Noop)
  }
}

// ---------------------------------------------------------------------------
// ProxyLeader.handlePhase2bNoopRange (:355-412): phase2bs(acceptorGroupIndex)(acceptorIndex) = msg;
// wait while ANY acceptor group of the leader group has fewer than f+1 votes; the first
// delivery after which none has sends ChosenNoopRange and turns the key Done.  Same
// first-delivery-stamp scheme as the Phase2b tally: ONE CTA, phase A stamps, phase B
// evaluates record i against the stamps below its own and compacts in delivery order.
//   in {dst, start, end, round}   out {start, end}
// ---------------------------------------------------------------------------
struct RangeTallyParams {
  Geometry g;
  PLState pl;
  RangeTable tab;
  const int4* in;
  int32_t n;
  uint32_t seq_base;
  int2* out;
  int32_t* dec;      // entry index + 1, or 0 = ignored
  DevStatus* st;
};

__global__ void __launch_bounds__(kRangeCtaThreads) range_tally_kernel(RangeTallyParams P) {
  const Geometry& g = P.g;
  __shared__ int s_cnt[64];
  __shared__ int s_tot[2];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid < 2) s_tot[tid] = 0;
  for (int i = tid; i < P.n; i += kRangeCtaThreads) {
    const int4 rec = P.in[i];
    int d = 0;
    uint32_t* e = nullptr;
    if (range_retired(g, rec.y, rec.z)) {
      // a retired range was chosen long ago: the vote finds `Done` and is ignored (:372-388)
    } else if ((e = range_find(P.tab, rec.y, rec.z, rec.w)) == nullptr) {
      bool single = false;
      if (rec.z == rec.y + 1) {
        int l = local_slot(g, rec.y);
        single = l >= 0 && find_row(g, P.pl, l, rec.y, rec.w).p != nullptr;   // Some(Done | PendingPhase2a): ignored (:372-388)
      }
      if (!single) report_error(P.st, FPX_ERR_UNKNOWN_SLOT_ROUND, i);         // :364-370 logger.fatal
    } else if (*(volatile uint32_t*)e != kRangeDone) {
      if (!range_dst_ok(g, rec.x, rec.y)) {
        report_error(P.st, FPX_ERR_BAD_ACCEPTOR, i);                          // phase2bs(acceptorGroupIndex): out of bounds
      } else {
        int v = ((rec.x >> 16) % g.agroups) * g.per_group + (rec.x & 0xffff);
        atomicMin(&e[4 + v], P.seq_base + (uint32_t)i);                       // :392-393
        d = (int)((e - P.tab.ent) / kRangeWords) + 1;
      }
    }
    P.dec[i] = d;
  }
  __syncthreads();
  CtaCompactor cc{s_cnt, s_tot};
  for (int base = 0; base < P.n; base += kRangeCtaThreads) {
    const int i = base + tid;
    bool complete = false;
    int4 rec = make_int4(0, 0, 0, 0);
    uint32_t* e = nullptr;
    if (i < P.n && P.dec[i] > 0) {
      rec = P.in[i];
      e = P.tab.ent + (size_t)(P.dec[i] - 1) * kRangeWords;
      const uint32_t seq = P.seq_base + (uint32_t)i;
      const int myag = (rec.x >> 16) % g.agroups;
      if (__ldcg(&e[4 + myag * g.per_group + (rec.x & 0xffff)]) == seq) {     // first delivery of this acceptor
        bool all_before = true, all_with = true;
        for (int ag = 0; ag < g.agroups; ++ag) {
          int cb = 0;
          for (int a = 0; a < g.per_group; ++a) cb += __ldcg(&e[4 + ag * g.per_group + a]) < seq;
          all_before &= cb >= g.quorum;
          all_with &= cb + (ag == myag) >= g.quorum;                          // exists(_.size < quorumSize) (:394)
        }
        complete = all_with && !all_before;
      }
    }
    int pa, pb;
    cc.pos(complete, false, lane, warp, pa, pb);
    if (complete) {
      P.out[pa] = make_int2(rec.y, rec.z);       // ChosenNoopRange(start, end) (:399-409)
      *(volatile uint32_t*)e = kRangeDone;       // states(slotround) = Done (:412); phase B reads stamps only
    }
  }
  if (tid == 0) P.st->n_chosen = s_tot[0];
}

__global__ void renormalize_range_stamps_kernel(RangeTable t) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= t.cap) return;
  uint32_t* e = t.ent + (size_t)i * kRangeWords;
  if (e[0] == kRangeEmpty) return;
  for (int v = 0; v < 32; ++v)
    if (e[4 + v] != kStampEmpty) e[4 + v] = 0;
}

// ---------------------------------------------------------------------------
// Replica.handleChosenNoopRange (:464-486): for slot <- start until end by numLeaderGroups:
// already in the log -> RETURN (the whole handler: nothing after that slot is filled), else
// log.put(slot, Noop).  Two grid passes over (record, chunk) tiles: the first slot of each
// record that is already in the log (min-reduce), then the put-if-absent fill below it.
// Batch contract (FPX_ERR_BATCH_ORDER): two records of one call must not cover a common
// slot -- the second one's stop position would depend on the first one's progress.
//
// kMixed: the same two passes over the multi-slot records of a mixed Chosen / ChosenNoopRange batch
// (fpx_mencius_replica_inbound, below), one CTA row per listed record in turn.  Their one-slot records have been
// put into the log first, each under its own delivery number seq_base + i (first one wins, as in handleChosen), so a
// range of index j stops at its first slot whose entry is older than seq_base + j: put before the call, or by a
// one-slot record delivered before the range.  Its fill then replaces the entries of later one-slot records below
// that stop (atomicMin of the smaller delivery number), which the reference would have found taken.
// ---------------------------------------------------------------------------
struct ReplicaRangeParams {
  Geometry g;
  const int2* in;
  int32_t n;
  uint32_t seq_base;
  unsigned long long* rlog;
  int32_t* first;    // [n], preset to kNoHit (kMixed: [listed records])
  DevStatus* st;
  // kMixed: fpx_mencius_chosen records, the listed multi-slot records' indices and the call's control words
  const int4* in4;
  const int32_t* list;
  const int32_t* ctl;
};

// kMixed: rows of the list that are applied (listed and before the split)
__device__ __forceinline__ int mixed_listed(const ReplicaRangeParams& P) {
  return min(__ldcg(&P.ctl[1]), (int)FPX_MAX_RANGE_BATCH);
}

// one record's first hit: the first slot of rec = [start, end) that is already in the log -> first[y]
template <bool kMixed>
__device__ __forceinline__ void replica_range_first_one(const ReplicaRangeParams& P, int y, int j, int2 rec) {
  const Geometry& g = P.g;
  const long long LG = g.lgroups;
  const long long count = (rec.y - rec.x + LG - 1) / LG;
  int hit = kNoHit;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < count && hit == kNoHit;
       t += (long long)gridDim.x * blockDim.x) {
    int slot = (int)(rec.x + t * LG);
    int l = local_slot(g, slot);
    // ascending per thread: first hit is its minimum.  A retired slot is in the log (executed long ago).
    if (kMixed) {   // an empty entry reads as delivery number 0xffffffff: never older than seq_base + j
      if (l == kLocalRetired || (l >= 0 && (uint32_t)(__ldcg(&P.rlog[l]) >> 32) < P.seq_base + (uint32_t)j)) hit = slot;
    } else {
      if (l == kLocalRetired || (l >= 0 && __ldcg(&P.rlog[l]) != kU64Empty)) hit = slot;
    }
  }
  hit = __reduce_min_sync(0xffffffffu, hit);
  if ((threadIdx.x & 31) == 0 && hit != kNoHit) atomicMin(&P.first[y], hit);
}

// one record's fill below min(end, first[y]); returns the largest ordinal this thread put
template <bool kMixed>
__device__ __forceinline__ int replica_range_fill_one(const ReplicaRangeParams& P, int y, int j, int2 rec) {
  const Geometry& g = P.g;
  const long long LG = g.lgroups;
  const int stop = min(rec.y, __ldcg(&P.first[y]));
  const long long count = stop > rec.x ? (stop - rec.x + LG - 1) / LG : 0;
  int mx = INT_MIN;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < count; t += (long long)gridDim.x * blockDim.x) {
    int l = local_slot(g, (int)(rec.x + t * LG));
    if (l < 0) continue;
    unsigned long long old = atomicMin(&P.rlog[l], ((unsigned long long)(P.seq_base + (uint32_t)j) << 32) |
                                                       (uint32_t)FPX_VALUE_NOOP);
    // another record of this call covers the slot too: the later of the two is at fault.  (kMixed: only a later
    // one-slot record can be there, and the range is right to take the slot from it.)
    if (!kMixed && old != kU64Empty)
      report_error(P.st, FPX_ERR_BATCH_ORDER, max((long long)j, (long long)(uint32_t)(old >> 32) - (long long)P.seq_base));
    mx = max(mx, g.base_local + ring_to_rel(g, l));   // an ordinal, like every other writer of max_chosen_local
  }
  return mx;
}

// kMixed: the listed record of row y (y < rows), or false at the first one at or past the split
__device__ __forceinline__ bool mixed_listed_rec(const ReplicaRangeParams& P, int y, int* j, int2* rec) {
  *j = __ldg(&P.list[y]);
  if (*j >= __ldcg(&P.ctl[0])) return false;      // the list is in delivery order
  const int4 r = __ldg(&P.in4[*j]);
  *rec = make_int2(r.x, r.y);
  return true;
}

template <bool kMixed>
__global__ void __launch_bounds__(256) replica_range_first_kernel(ReplicaRangeParams P) {
  if (!kMixed) {
    const int j = blockIdx.y;
    const int2 rec = P.in[j];
    if (range_precheck(P.g, rec.x, rec.y, 0) != FPX_OK) {
      if (blockIdx.x == 0 && threadIdx.x == 0) report_error(P.st, FPX_ERR_SLOT_RANGE, j);
      return;
    }
    replica_range_first_one<false>(P, j, j, rec);
    return;
  }
  const int rows = mixed_listed(P);
  for (int y = blockIdx.y; y < rows; y += gridDim.y) {
    int j;
    int2 rec;
    if (!mixed_listed_rec(P, y, &j, &rec)) break;
    replica_range_first_one<true>(P, y, j, rec);
  }
}

template <bool kMixed>
__global__ void __launch_bounds__(256) replica_range_fill_kernel(ReplicaRangeParams P) {
  int mx = INT_MIN;
  if (!kMixed) {
    const int j = blockIdx.y;
    const int2 rec = P.in[j];
    if (range_precheck(P.g, rec.x, rec.y, 0) != FPX_OK) return;
    mx = replica_range_fill_one<false>(P, j, j, rec);
  } else {
    const int rows = mixed_listed(P);
    for (int y = blockIdx.y; y < rows; y += gridDim.y) {
      int j;
      int2 rec;
      if (!mixed_listed_rec(P, y, &j, &rec)) break;
      mx = max(mx, replica_range_fill_one<true>(P, y, j, rec));
    }
  }
  mx = __reduce_max_sync(0xffffffffu, mx);
  if ((threadIdx.x & 31) == 0 && mx != INT_MIN) atomicMax(&P.st->max_chosen_local, mx);
}

// ---------------------------------------------------------------------------
// A mixed batch of the replica's Chosen and ChosenNoopRange messages in delivery order (fpx_mencius_replica_inbound):
// record {s, e, v} stands for the slots s, s + LG, ... < e.  Replica.handleChosen (S/mencius/Replica.scala:402-420)
// and handleChosenNoopRange (:464-486) are both "put v into the slots until the first one already in the log", so a
// record of one slot is a put-if-absent and only the records of two or more slots ("ranges") can stop part way.
// The call applies the records before `split`, the smallest of
//   (a) the first range that shares a slot with an earlier range (full extents): its stop would depend on that
//       range's progress;
//   (b) the first range past FPX_MAX_RANGE_BATCH;
// and n.  Passes: mixed_count -> tile_offsets -> mixed_list (the ranges in delivery order, rule (b)) ->
// mixed_overlap (rule (a)) -> mixed_single (the one-slot records, statuses) -> replica_range_first / _fill<true>.
// ctl = {split, ranges}.
// ---------------------------------------------------------------------------
constexpr int kMixPer = 4, kMixThreads = 256, kMixTile = kMixPer * kMixThreads;

struct MixedParams {
  Geometry g;
  const int4* in;
  int32_t n;
  uint32_t seq_base;
  unsigned long long* rlog;
  uint32_t* tile;     // [tiles] ranges per tile, then their exclusive offsets
  int32_t* list;      // [FPX_MAX_RANGE_BATCH] the ranges' record indices, delivery order
  int32_t* first;     // [FPX_MAX_RANGE_BATCH] their stops, preset to kNoHit
  int32_t* ctl;       // {split, ranges}
  DevStatus* st;
};

// slots the record covers (0 for a record that fails range_precheck)
__device__ __forceinline__ long long mixed_count(const Geometry& g, int4 r) {
  if (range_precheck(g, r.x, r.y, 0) != FPX_OK) return 0;
  return (r.y - (long long)r.x + g.lgroups - 1) / g.lgroups;
}

__global__ void __launch_bounds__(kMixThreads) mixed_count_kernel(MixedParams P) {
  uint32_t c = 0;
  for (int u = 0; u < kMixPer; ++u) {
    const int i = blockIdx.x * kMixTile + (int)threadIdx.x * kMixPer + u;
    if (i < P.n) c += mixed_count(P.g, __ldg(&P.in[i])) >= 2;
  }
  c = cta_reduce<kMixThreads>(c, ScanSum());
  if (threadIdx.x == 0) P.tile[blockIdx.x] = c;
  if (blockIdx.x == 0 && threadIdx.x == 0) P.ctl[0] = P.n;
}

__global__ void __launch_bounds__(kMixThreads) mixed_list_kernel(MixedParams P) {
  bool multi[kMixPer];
  uint32_t c = 0;
  const int i0 = blockIdx.x * kMixTile + (int)threadIdx.x * kMixPer;
#pragma unroll
  for (int u = 0; u < kMixPer; ++u) {
    multi[u] = i0 + u < P.n && mixed_count(P.g, __ldg(&P.in[i0 + u])) >= 2;
    c += multi[u];
  }
  uint32_t rank = __ldcg(&P.tile[blockIdx.x]) + cta_scan<kMixThreads, true>(c, ScanSum());
#pragma unroll
  for (int u = 0; u < kMixPer; ++u) {
    if (!multi[u]) continue;
    if (rank < (uint32_t)FPX_MAX_RANGE_BATCH) {
      P.list[rank] = i0 + u;
      P.first[rank] = kNoHit;
    } else if (rank == (uint32_t)FPX_MAX_RANGE_BATCH) {
      atomicMin(&P.ctl[0], i0 + u);                 // rule (b)
    }
    ++rank;
  }
}

// Rule (a) over the listed ranges: every pair (p < q) of ranks, by 256 x 256 tiles of pairs claimed in turn by a
// fixed grid.  Two ranges share a slot iff they start in the same residue mod LG and max(starts) < min(ends).
__global__ void __launch_bounds__(kMixThreads) mixed_overlap_kernel(MixedParams P) {
  __shared__ int s_s[kMixThreads], s_e[kMixThreads];
  const int K = min(__ldcg(&P.ctl[1]), (int)FPX_MAX_RANGE_BATCH);
  const long long T = (K + kMixThreads - 1) / kMixThreads;
  const int LG = P.g.lgroups;
  for (long long t = blockIdx.x; t < T * (T + 1) / 2; t += gridDim.x) {
    // t -> (q, p), p <= q: t = q (q + 1) / 2 + p
    long long q = (long long)((sqrt(8.0 * (double)t + 1.0) - 1.0) / 2.0);
    while (q * (q + 1) / 2 > t) --q;
    while ((q + 1) * (q + 2) / 2 <= t) ++q;
    const long long p = t - q * (q + 1) / 2;
    const int rp = (int)p * kMixThreads + threadIdx.x, rq = (int)q * kMixThreads + threadIdx.x;
    __syncthreads();
    if (rp < K) {
      const int4 r = __ldg(&P.in[__ldcg(&P.list[rp])]);
      s_s[threadIdx.x] = r.x; s_e[threadIdx.x] = r.y;
    }
    __syncthreads();
    if (rq >= K) continue;
    const int j = __ldcg(&P.list[rq]);
    const int4 r = __ldg(&P.in[j]);
    const int res = r.x % LG;
    const int hi = min(kMixThreads, p == q ? (int)threadIdx.x : K - (int)p * kMixThreads);
    bool hit = false;
    for (int k = 0; k < hi; ++k) {
      const int s = s_s[k];
      hit |= s % LG == res && max(s, r.x) < min(s_e[k], r.y);
    }
    if (hit) atomicMin(&P.ctl[0], j);
  }
}

// The one-slot records before the split: put-if-absent under their delivery number (the smallest wins), like
// replica_chosen_kernel; and the statuses of every record before the split.
__global__ void __launch_bounds__(kMixThreads) mixed_single_kernel(MixedParams P) {
  const Geometry& g = P.g;
  const int split = __ldcg(&P.ctl[0]);
  int mx = INT_MIN;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < split; i += gridDim.x * blockDim.x) {
    const int4 r = __ldg(&P.in[i]);
    if (range_precheck(g, r.x, r.y, 0) != FPX_OK) { report_error(P.st, FPX_ERR_SLOT_RANGE, i); continue; }
    if (mixed_count(g, r) != 1) continue;
    const int l = local_slot(g, r.x);
    if (l < 0) continue;                                   // retired: in the log already (range_precheck bounds it)
    red_min_u64(&P.rlog[l], ((unsigned long long)(P.seq_base + (uint32_t)i) << 32) | (uint32_t)r.z);
    mx = max(mx, g.base_local + ring_to_rel(g, l));
  }
  mx = __reduce_max_sync(0xffffffffu, mx);
  if ((threadIdx.x & 31) == 0 && mx != INT_MIN) atomicMax(&P.st->max_chosen_local, mx);
}

// ---------------------------------------------------------------------------
// Vanilla Mencius skips.  rec {server, start, stop, own}: the slots start, start + n, ...
// < stop (nextClassicRound of the coordinator) of server `server`'s log become
// ChosenEntry(Noop).
//   own = 1  advanceWithSkips' fill at the skipping server (Server.scala:610-620): every
//            slot must be vacant -- logger.check(!log.contains), check(!phase2s.contains)
//            -> FPX_ERR_CHECK_FAILED;
//   own = 0  handleSkip (:1144-1168): choose(slot, Noop) -- log.put unconditionally,
//            phase2s.remove (:622-625).
// ---------------------------------------------------------------------------
struct VmSkipParams {
  Geometry g;
  const int4* in;
  unsigned long long* votes;
  uint32_t* rows;
  DevStatus* st;
};

// advanceWithSkips' fill of one own slot (:613-618) at ring position l: log.put(ChosenEntry(Noop)) into a vacant
// cell.  False where the slot is not vacant -- logger.check(!log.contains), check(!phase2s.contains) (:613-614).
// Shared by the own = 1 skip and the self-revocation of fpx_vm_phase1a_wire.
__device__ __forceinline__ bool vm_fill_own(const Geometry& g, unsigned long long* votes, const uint32_t* rows, int l,
                                            int server) {
  const unsigned long long old = atomicCAS(&votes[cell_index(g, l, server)], 0ull, kCellChosen | (uint32_t)FPX_VALUE_NOOP);
  return old == 0ull && __ldcg(rows + (size_t)l * g.row_words) == kUnarmed;
}

__global__ void __launch_bounds__(256) vm_skip_kernel(VmSkipParams P) {
  const Geometry& g = P.g;
  const int j = blockIdx.y;
  const int4 rec = P.in[j];
  const int server = rec.x, n = g.per_group;
  int c = FPX_OK;
  if ((uint32_t)server >= (uint32_t)n) c = FPX_ERR_BAD_ACCEPTOR;
  else if (rec.y < 0 || rec.z < rec.y || rec.z > g.slot_capacity) c = FPX_ERR_SLOT_RANGE;
  else if (rec.w && rec.y % n != server) c = FPX_ERR_BAD_ACCEPTOR;
  if (c != FPX_OK) {
    if (blockIdx.x == 0 && threadIdx.x == 0) report_error(P.st, c, j);
    return;
  }
  const long long count = (rec.z - rec.y + (long long)n - 1) / n;
  const unsigned long long chosen = kCellChosen | (uint32_t)FPX_VALUE_NOOP;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < count; t += (long long)gridDim.x * blockDim.x) {
    const int slot = (int)(rec.y + t * n);
    const int l = local_slot(g, slot);
    if (l < 0) {
      // retired: a ChosenEntry at every server -- not vacant for the fill (:613-614), already chosen for handleSkip
      if (l == kLocalRetired && rec.w) report_error(P.st, FPX_ERR_CHECK_FAILED, j);
      continue;
    }
    unsigned long long* cell = &P.votes[cell_index(g, l, server)];
    uint32_t* row = P.rows + (size_t)l * g.row_words;
    if (rec.w) {
      if (!vm_fill_own(g, P.votes, P.rows, l, server)) report_error(P.st, FPX_ERR_CHECK_FAILED, j);
    } else {
      red_max_u64(cell, chosen);                                                      // choose: log.put (:624)
      if (slot % n == server && __ldcg(row) != kUnarmed) red_or_u32(row, kDoneBit);   // phase2s.remove(slot) (:625)
    }
  }
}

}  // namespace fpx
