#pragma once
#include "fpx_common.cuh"
#include "fpx_ranges.cuh"

namespace fpx {

// ===========================================================================
// K1  ProxyLeader.handlePhase2a  -- "arm"   S/multipaxos/ProxyLeader.scala:175-215
//   states.get((slot, round)): Some -> ignore (:177-183); None -> Pending(phase2a,
//   {}) (:213).  Warp-strided 32-record chunks; the key's header {round_word,
//   value_id} is claimed with ONE 64-bit CAS, four of them in flight per lane.  A
//   second round for a slot moves the slot's keys to the (slot, round) table and
//   poisons the primary row (arm_finish).  Two arms of one key with DIFFERENT
//   values inside one batch (never produced by a correct leader) are resolved to
//   "first in delivery order wins" by the last block of the launch.
// ===========================================================================
struct ArmConflict { int32_t slot, round; };

struct ArmParams {
  Geometry g;
  PLState pl;
  const int4* in;
  int32_t n;
  DevStatus* st;
  ArmConflict* conflicts;
  uint32_t* win_bits;  // ceil(n/32): record i created its key's entry
  unsigned long long* votes;  // vanilla Mencius (vanilla != 0): the coordinator votes for itself
  int32_t vanilla;
  RangeTable rng;      // mencius: one-slot Phase2aNoopRange keys share the key space (check_rng != 0)
  int32_t check_rng;
};

__device__ __forceinline__ void note_arm_conflict(const ArmParams& P, int slot, int round) {
  uint32_t c = atomicAdd(&P.st->n_arm_conflicts, 1u);
  if (c < (uint32_t)kMaxConflicts) P.conflicts[c] = ArmConflict{slot, round};
}

// returns true if this record installed the header
__device__ __forceinline__ bool claim_header(const ArmParams& P, RowRef r, int slot, int round, int value,
                                             bool* other_round) {
  unsigned long long want = ((unsigned long long)(uint32_t)value << 32) | (uint32_t)round;
  unsigned long long old = atomicCAS(r.hdr64(), kU64Empty, want);
  *other_round = false;
  if (old == kU64Empty) return true;
  uint32_t orw = (uint32_t)old;
  if ((int)(orw & ~kDoneBit) != round) { *other_round = true; return false; }
  if ((uint32_t)(old >> 32) != (uint32_t)value) note_arm_conflict(P, slot, round);
  return false;
}

// table slot of key (slot, round), inserting the key if absent; nullptr = table full
__device__ __forceinline__ uint32_t* table_insert(const ArmParams& P, int slot, int round) {
  const Geometry& g = P.g;
  if (g.ovf_cap == 0) return nullptr;
  unsigned long long key = ((unsigned long long)(uint32_t)slot << 32) | (uint32_t)round;
  uint32_t h = (uint32_t)mix64(key) & g.ovf_mask;
  for (int probe = 0; probe < g.ovf_cap; ++probe) {
    unsigned long long k = atomicCAS(&P.pl.ovf_keys[h], kU64Empty, key);
    if (k == kU64Empty || k == key) return P.pl.ovf_rows + (size_t)h * g.row_words;
    h = (h + 1) & g.ovf_mask;
  }
  return nullptr;
}

// second stage of one arm: `old` is what the 64-bit CAS on the primary row's header
// returned.  Returns true if this record created the key's entry.
//
// A slot's primary row holds its ONLY armed round.  When a second round of the slot is
// armed (leader change: Leader.handlePhase1b re-proposes chosenWatermark..maxSlot in the
// new round, S/multipaxos/Leader.scala:551-562; both (slot, round) keys then tally
// independently, ProxyLeader.scala:135) the first round's entry -- header and stamps, which
// are quiescent during an arm call -- is moved to the (slot, round) table and the primary
// header is poisoned for good; from then on every key of that slot lives in the table.
// That is what lets the tally kernel stamp votes without loading the header first.
__device__ __forceinline__ bool arm_finish(const ArmParams& P, const int4& rec, unsigned long long old, int i) {
  const Geometry& g = P.g;
  const int slot = rec.x, round = rec.y, value = rec.z;
  if (old == kU64Empty) return true;                       // Pending(phase2a, {}) created (:213)
  uint32_t* prim = P.pl.rows + (size_t)local_slot(g, slot) * g.row_words;
  unsigned long long* hdr = (unsigned long long*)prim;
  while (true) {
    uint32_t orw = (uint32_t)old;
    if (orw == kBusy) {                                    // another record is moving the row: wait
      __nanosleep(64);
      old = *(volatile unsigned long long*)hdr;
      continue;
    }
    if (orw == kPoison) {
      uint32_t* t = table_insert(P, slot, round);
      if (t == nullptr) { report_error(P.st, FPX_ERR_OVERFLOW_FULL, i); return false; }
      bool dummy;
      return claim_header(P, RowRef{t}, slot, round, value, &dummy);
    }
    if ((int)(orw & ~kDoneBit) == round) {                 // `case Some(_)`: ignore (:177-183)
      if ((uint32_t)(old >> 32) != (uint32_t)value) note_arm_conflict(P, slot, round);
      return false;
    }
    // a second round for this slot: move the first one to the table, poison the primary
    unsigned long long busy = (old & 0xffffffff00000000ull) | kBusy;
    unsigned long long prev = atomicCAS(hdr, old, busy);
    if (prev != old) { old = prev; continue; }
    uint32_t* t = table_insert(P, slot, (int)(orw & ~kDoneBit));
    if (t == nullptr) {
      report_error(P.st, FPX_ERR_OVERFLOW_FULL, i);
      atomicExch(hdr, old);
      return false;
    }
    t[0] = orw;
    t[1] = (uint32_t)(old >> 32);
    for (int v = 0; v < g.voters; ++v) t[2 + v] = prim[2 + v];
    __threadfence();
    old = (old & 0xffffffff00000000ull) | kPoison;
    atomicExch(hdr, old);
  }
}

constexpr int kArmUnroll = 8;
constexpr int kArmThreads = 1024;   // one CTA of 32 warps per SM, at most one wave (grid-stride loop)

// The arm work of warp `gwarp` of `total_warps` (arm_kernel; also called from the acceptor kernel when
// fpx_step_dev runs both roles in one launch).  Warp-strided 32-record chunks; per lane kArmUnroll
// independent record loads, then kArmUnroll independent header CASes, are in flight before any result is
// used.  Only the row index and the CAS result stay live across the round trip; the rare slow paths
// (key exists, second round of a slot, vanilla self vote) re-read their record.
__device__ __forceinline__ int arm_chunks(const ArmParams& P, int gwarp, int total_warps, int lane) {
  const Geometry& g = P.g;
  const int n_chunks = (P.n + 31) >> 5;
  int max_local = -1;
  for (int c0 = gwarp * kArmUnroll; c0 < n_chunks; c0 += total_warps * kArmUnroll) {
    unsigned long long old[kArmUnroll];
    unsigned long long want[kArmUnroll];
    int local[kArmUnroll];          // row of the record, -1: not a valid arm
    {
      int4 rec[kArmUnroll];
#pragma unroll
      for (int u = 0; u < kArmUnroll; ++u) {
        int i = (c0 + u) * 32 + lane;
        rec[u] = (c0 + u < n_chunks && i < P.n) ? ld_stream(P.in + i) : make_int4(-1, 0, 0, 0);  // {slot, round, value_id, dst}
      }
#pragma unroll
      for (int u = 0; u < kArmUnroll; ++u) {
        int i = (c0 + u) * 32 + lane;
        local[u] = -1;
        old[u] = 0;
        if (c0 + u < n_chunks && i < P.n) {
          int l = local_slot(g, rec[u].x);
          if (l < 0) {
            if (l != kLocalRetired) report_error(P.st, FPX_ERR_SLOT_RANGE, i);   // retired: the key is Done, `case Some(_)` (:177-183)
          } else if ((uint32_t)rec[u].y > (uint32_t)FPX_MAX_ROUND) {
            report_error(P.st, FPX_ERR_ROUND_RANGE, i);
          } else if (P.vanilla && rec[u].y != 0) {
            report_error(P.st, FPX_ERR_ROUND_RANGE, i);    // Server.handleClientRequest proposes in round 0 (:779, :806-815)
          } else if (P.vanilla && ((rec[u].w >> 16) != 0 || (rec[u].w & 0xffff) >= g.per_group ||
                                   rec[u].x % g.per_group != (rec[u].w & 0xffff))) {
            report_error(P.st, FPX_ERR_BAD_ACCEPTOR, i);   // only the slot's owner coordinates it (:773, slotSystem)
          } else if (P.check_rng && range_find(P.rng, rec[u].x, rec[u].x + 1, rec[u].y) != nullptr) {
            // S/mencius: SlotRound(slot, slot+1, round) is held by a one-slot Phase2aNoopRange:
            // `case Some(_)` -> ignored (mencius/ProxyLeader.scala:220-226)
          } else {
            // the header is READ first: a plain load misses to DRAM far more cheaply than an atomic does,
            // and a key that already exists needs no CAS at all (`case Some(_)`, :177-183).  The row is
            // tagged evict_last: the tally's stamps and sweep come back to it within the same step (not
            // for vanilla Mencius, whose step measured 0.4 % slower with the hint).
            local[u] = l;
            want[u] = ((unsigned long long)(uint32_t)rec[u].z << 32) | (uint32_t)rec[u].y;
            const unsigned long long* hdr = (const unsigned long long*)(P.pl.rows + (size_t)l * g.row_words);
            old[u] = P.vanilla ? __ldcg(hdr) : ld_u64_evict_last(hdr);
          }
        }
      }
    }
#pragma unroll
    for (int u = 0; u < kArmUnroll; ++u)
      if (local[u] >= 0 && old[u] == kU64Empty)
        old[u] = atomicCAS((unsigned long long*)(P.pl.rows + (size_t)local[u] * g.row_words), kU64Empty, want[u]);
#pragma unroll
    for (int u = 0; u < kArmUnroll; ++u) {
      if (c0 + u >= n_chunks) break;
      int i = (c0 + u) * 32 + lane;
      bool won = local[u] >= 0 && old[u] == kU64Empty;       // Pending(phase2a, {}) created (:213)
      int self = -1;
      if (local[u] >= 0 && old[u] != kU64Empty) {            // rare: the key exists, or a second round of the slot
        const int4 rec = __ldcg(P.in + i);
        won = arm_finish(P, rec, old[u], i);
        self = rec.w & 0xffff;
      } else if (won && P.vanilla) {
        self = rel_to_slot(g, ring_to_rel(g, local[u])) % g.per_group;   // the owner coordinates its slot (checked above)
      }
      if (won && P.vanilla) {
        // Server.handleClientRequest: log.put(slot, PendingEntry(0, 0, value)) (:779) and
        // phase2s(slot).phase2bs = {index -> Phase2b} (:818-825): own vote, stamped "before everything".
        // A NEW Phase 2 entry: stamps of stray votes that arrived before it existed (ignored by the
        // reference, stamped blindly by the tally) go -- the rest of the row is rewritten with wide stores.
        uint32_t* row = P.pl.rows + (size_t)local[u] * g.row_words;
        auto stamp = [&](int w) { return w - 2 == self ? 0u : kStampEmpty; };
        *(uint2*)(row + 2) = make_uint2(stamp(2), stamp(3));
        for (int w = 4; w < g.row_words; w += 4) *(uint4*)(row + w) = make_uint4(stamp(w), stamp(w + 1), stamp(w + 2), stamp(w + 3));
        // vote cell {round + 1 : value}; want = {value : round}
        red_max_u64(&P.votes[cell_index(g, local[u], self)], (((want[u] & 0xffffffffull) + 1ull) << 32) | (want[u] >> 32));
      }
      unsigned wb = __ballot_sync(0xffffffffu, won);
      if (lane == 0) P.win_bits[c0 + u] = wb;
      int ml = __reduce_max_sync(0xffffffffu, won ? local[u] : -1);
      if (lane == 0 && ml > max_local) max_local = ml;
    }
  }
  return max_local;
}

// Two arms of one key with different values: if the key was created by a record of THIS batch, the
// lowest-index arm is the one the reference would have kept (later ones hit `case Some(_)`, :177-183);
// if it existed before the batch, the stored value stands.  One CTA, after every arm of the batch.
__device__ __forceinline__ void arm_resolve_conflicts(const ArmParams& P) {
  const Geometry& g = P.g;
  __shared__ int s_min, s_any;
  uint32_t nc = __ldcg(&P.st->n_arm_conflicts);
  if (nc == 0) return;
  if (nc > (uint32_t)kMaxConflicts) {
    if (threadIdx.x == 0) { report_error(P.st, FPX_ERR_CONFLICT, 0); P.st->n_arm_conflicts = 0; }
    return;
  }
  for (uint32_t c = 0; c < nc; ++c) {
    int slot = P.conflicts[c].slot, round = P.conflicts[c].round;
    if (threadIdx.x == 0) { s_min = INT_MAX; s_any = 0; }
    __syncthreads();
    for (int j = threadIdx.x; j < P.n; j += blockDim.x) {
      int4 rec = P.in[j];
      if (rec.x == slot && rec.y == round) {
        atomicMin(&s_min, j);
        if ((__ldcg(&P.win_bits[j >> 5]) >> (j & 31)) & 1u) s_any = 1;
      }
    }
    __syncthreads();
    if (threadIdx.x == 0 && s_any && s_min != INT_MAX) {
      RowRef r = find_row(g, P.pl, local_slot(g, slot), slot, round);
      if (r.p != nullptr) r.p[1] = (uint32_t)P.in[s_min].z;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) P.st->n_arm_conflicts = 0;
}

__global__ void __launch_bounds__(kArmThreads, 1) arm_kernel(ArmParams P) {
  const int lane = threadIdx.x & 31;
  const int max_local = arm_chunks(P, blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), gridDim.x * (blockDim.x >> 5), lane);
  if (lane == 0 && max_local >= 0) atomicMax(&P.st->max_armed_local, max_local);

  // ---- last block: conflicting arms of one key
  __shared__ bool s_last;
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();   // cumulative: orders the whole CTA's writes (barrier above) before the ticket
    s_last = (atomicAdd(&P.st->ticket, 1u) == gridDim.x - 1);
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  if (threadIdx.x == 0) P.st->ticket = 0;
  arm_resolve_conflicts(P);
}

}  // namespace fpx
