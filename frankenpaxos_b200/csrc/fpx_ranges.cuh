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
// ---------------------------------------------------------------------------
struct ReplicaRangeParams {
  Geometry g;
  const int2* in;
  int32_t n;
  uint32_t seq_base;
  unsigned long long* rlog;
  int32_t* first;    // [n], preset to kNoHit
  DevStatus* st;
};

__global__ void __launch_bounds__(256) replica_range_first_kernel(ReplicaRangeParams P) {
  const Geometry& g = P.g;
  const int j = blockIdx.y;
  const int2 rec = P.in[j];
  if (range_precheck(g, rec.x, rec.y, 0) != FPX_OK) {
    if (blockIdx.x == 0 && threadIdx.x == 0) report_error(P.st, FPX_ERR_SLOT_RANGE, j);
    return;
  }
  const long long LG = g.lgroups;
  const long long count = (rec.y - rec.x + LG - 1) / LG;
  int hit = kNoHit;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < count && hit == kNoHit;
       t += (long long)gridDim.x * blockDim.x) {
    int slot = (int)(rec.x + t * LG);
    int l = local_slot(g, slot);
    // ascending per thread: first hit is its minimum.  A retired slot is in the log (executed long ago).
    if (l == kLocalRetired || (l >= 0 && __ldcg(&P.rlog[l]) != kU64Empty)) hit = slot;
  }
  hit = __reduce_min_sync(0xffffffffu, hit);
  if ((threadIdx.x & 31) == 0 && hit != kNoHit) atomicMin(&P.first[j], hit);
}

__global__ void __launch_bounds__(256) replica_range_fill_kernel(ReplicaRangeParams P) {
  const Geometry& g = P.g;
  const int j = blockIdx.y;
  const int2 rec = P.in[j];
  if (range_precheck(g, rec.x, rec.y, 0) != FPX_OK) return;
  const long long LG = g.lgroups;
  const int stop = min(rec.y, __ldcg(&P.first[j]));
  const long long count = stop > rec.x ? (stop - rec.x + LG - 1) / LG : 0;
  int mx = INT_MIN;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < count; t += (long long)gridDim.x * blockDim.x) {
    int l = local_slot(g, (int)(rec.x + t * LG));
    if (l < 0) continue;
    unsigned long long old = atomicMin(&P.rlog[l], ((unsigned long long)(P.seq_base + (uint32_t)j) << 32) |
                                                       (uint32_t)FPX_VALUE_NOOP);
    if (old != kU64Empty)   // another record of this call covers the slot too: the later of the two is at fault
      report_error(P.st, FPX_ERR_BATCH_ORDER, max((long long)j, (long long)(uint32_t)(old >> 32) - (long long)P.seq_base));
    mx = max(mx, g.base_local + ring_to_rel(g, l));   // an ordinal, like every other writer of max_chosen_local
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
      unsigned long long old = atomicCAS(cell, 0ull, chosen);                      // log.put(nextSlot, ChosenEntry(Noop)) (:615-618)
      if (old != 0ull || __ldcg(row) != kUnarmed) report_error(P.st, FPX_ERR_CHECK_FAILED, j);   // :613-614
    } else {
      red_max_u64(cell, chosen);                                                      // choose: log.put (:624)
      if (slot % n == server && __ldcg(row) != kUnarmed) red_or_u32(row, kDoneBit);   // phase2s.remove(slot) (:625)
    }
  }
}

}  // namespace fpx
