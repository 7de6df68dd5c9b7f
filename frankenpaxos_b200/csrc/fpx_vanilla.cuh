// fpx_vanilla.cuh -- vanilla Mencius (S/vanillamencius/Server.scala), SURVEY 8(a) row a9.
// The per-slot round compare of Server.handlePhase2a (:1001-1082) is per log
// entry, so records of different (slot, server) cells are independent: one
// thread per record, one 64-bit atomicMax per vote cell.  Cell = {hi: round+1 |
// chosen bit 31, lo: value}; a ChosenEntry compares above every vote, so it is
// absorbing under atomicMax exactly like `case Some(chosen: ChosenEntry)` (:1017).
#pragma once
#include "fpx_common.cuh"

namespace fpx {

struct VmParams {
  Geometry g;
  const int4* in;
  int4* out;
  int32_t n;
  unsigned long long* votes;   // [local_slots][n][2]: {vote cell, (~batch tag : min index) claim} -- 16 bytes, one sector
  uint32_t* rows;              // proxy-leader rows (phase2s)
  uint32_t tag;
  DevStatus* st;
};

#ifndef FPX_VM_UNROLL
#define FPX_VM_UNROLL 4
#endif
#ifndef FPX_VM_CTAS_PER_SM
#define FPX_VM_CTAS_PER_SM 8      // CTAs of the grid-stride launch per SM
#endif
constexpr int kVmUnroll = FPX_VM_UNROLL;

// 128-bit compare-and-swap (ATOMG.E.CAS.128, sm_90+): {e0, e1} is the expected value on entry and the
// value found on return
__device__ __forceinline__ bool cas128(unsigned long long* p, unsigned long long& e0, unsigned long long& e1,
                                       unsigned long long n0, unsigned long long n1) {
  unsigned long long o0, o1;
  asm volatile("{\n .reg .b128 d, b, c;\n mov.b128 b, {%2, %3};\n mov.b128 c, {%4, %5};\n"
               " atom.global.cas.b128 d, [%6], b, c;\n mov.b128 {%0, %1}, d;\n}"
               : "=l"(o0), "=l"(o1) : "l"(e0), "l"(e1), "l"(n0), "l"(n1), "l"(p) : "memory");
  const bool ok = o0 == e0 && o1 == e1;
  e0 = o0; e1 = o1;
  return ok;
}

// handlePhase2a.  in {slot, round, value, dst = server}; out {kind, server, slot, round|value}
// The vote cell and the claim word of the batch contract ("one Phase2a per (slot, server) per call") share
// 16 bytes: a message is ONE 128-bit load (which brings the sector into L2 -- atomics that miss L2 are several
// times slower than loads that do) and ONE 128-bit compare-and-swap that installs the new cell and the claim
// together.  The swap can only fail when another message of this call took the cell in between, which is the
// contract violation itself.  kVmUnroll messages per thread are in flight through every stage.
#ifndef FPX_VM_PREFETCH
#define FPX_VM_PREFETCH 1   // the records of round k+1 are in flight while round k's cell loads and swaps run
#endif
__global__ void __launch_bounds__(256, 3) vm_phase2a_kernel(VmParams P) {
  const Geometry& g = P.g;
  const int stride = gridDim.x * blockDim.x;
  const int t0 = blockIdx.x * blockDim.x + threadIdx.x;
#if FPX_VM_PREFETCH
  int4 nxt[kVmUnroll];
#pragma unroll
  for (int u = 0; u < kVmUnroll; ++u) {
    const int i = t0 + u * stride;
    nxt[u] = i < P.n ? ld_stream(P.in + i) : make_int4(0, 0, 0, 0);
  }
#endif
  for (int i0 = t0; i0 < P.n; i0 += stride * kVmUnroll) {
    int4 rec[kVmUnroll];
    int rk[kVmUnroll], rw[kVmUnroll];     // reply kind (-1: none) and its last word
    unsigned long long* cellp[kVmUnroll];
    unsigned long long pre0[kVmUnroll], pre1[kVmUnroll];
    bool okc[kVmUnroll];
#if FPX_VM_PREFETCH
#pragma unroll
    for (int u = 0; u < kVmUnroll; ++u) rec[u] = nxt[u];
#pragma unroll
    for (int u = 0; u < kVmUnroll; ++u) {
      const long long i = (long long)i0 + (long long)stride * kVmUnroll + (long long)u * stride;
      nxt[u] = i < P.n ? ld_stream(P.in + i) : make_int4(0, 0, 0, 0);
    }
#else
#pragma unroll
    for (int u = 0; u < kVmUnroll; ++u) {
      const int i = i0 + u * stride;
      rec[u] = i < P.n ? ld_stream(P.in + i) : make_int4(0, 0, 0, 0);
    }
#endif
#pragma unroll
    for (int u = 0; u < kVmUnroll; ++u) {
      const int i = i0 + u * stride;
      cellp[u] = nullptr;
      rk[u] = -1; rw[u] = 0;
      if (i >= P.n) continue;
      const int server = rec[u].w & 0xffff;
      const int local = local_slot(g, rec[u].x);
      int c = local == -1 ? FPX_ERR_SLOT_RANGE
              : ((rec[u].w >> 16) != 0 || server >= g.per_group) ? FPX_ERR_BAD_ACCEPTOR
              : (uint32_t)rec[u].y > (uint32_t)FPX_MAX_ROUND ? FPX_ERR_ROUND_RANGE : FPX_OK;
      if (c != FPX_OK) { report_error(P.st, c, i); continue; }
      // kLocalRetired (fpx_retire_below): the entry is a ChosenEntry whose value is the shared log's executed
      // entry -- the reference's Chosen(slot, value), :1016-1025, without the value
      if (local < 0) { rk[u] = FPX_VM_REPLY_CHOSEN_RETIRED; continue; }
      cellp[u] = P.votes + cell_index(g, local, server);
      asm volatile("ld.global.cg.v2.u64 {%0,%1}, [%2];" : "=l"(pre0[u]), "=l"(pre1[u]) : "l"(cellp[u]));
    }
#pragma unroll
    for (int u = 0; u < kVmUnroll; ++u) {
      okc[u] = false;
      if (cellp[u] == nullptr) continue;
      const int i = i0 + u * stride;
      const unsigned long long old = pre0[u];
      const unsigned long long mine = ((unsigned long long)(uint32_t)(rec[u].y + 1) << 32) | (uint32_t)rec[u].z;
      unsigned long long nw = old;
      if (old & kCellChosen) {
        // Chosen(slot, chosen.value, chosen.isRevocation) (:1018-1027)
        rk[u] = (old & kCellRevocation) ? FPX_VM_REPLY_CHOSEN_REVOCATION : FPX_VM_REPLY_CHOSEN; rw[u] = (int)(uint32_t)old;
      } else if ((uint32_t)(old >> 32) > (uint32_t)(mine >> 32)) {
        rk[u] = 1; rw[u] = (int)(uint32_t)(old >> 32) - 1;               // Phase2Nack(slot, round) (:1044-1051)
      } else {
        nw = mine;                                                       // log.put(slot, PendingEntry(round, round, value)) (:1054-1058)
        rk[u] = 0; rw[u] = rec[u].y;                                     // Phase2b(serverIndex, slot, round) (:1077-1081)
      }
      if ((uint32_t)(pre1[u] >> 32) != ~P.tag)                           // nobody of this call has the cell yet
        okc[u] = cas128(cellp[u], pre0[u], pre1[u], nw, ((unsigned long long)(~P.tag) << 32) | (uint32_t)i);
    }
#pragma unroll
    for (int u = 0; u < kVmUnroll; ++u) {
      const int i = i0 + u * stride;
      if (i >= P.n) continue;
      if (cellp[u] != nullptr && !okc[u]) {
        // a second Phase2a for this cell in one call (pre1 = the claim that beat this one): the engine cannot
        // order the two
        report_error(P.st, FPX_ERR_BATCH_ORDER, max((long long)i, (long long)(uint32_t)pre1[u]));
        rk[u] = -1; rw[u] = 0;
      }
      st_stream(P.out + i, make_int4(rk[u], rec[u].w & 0xffff, rec[u].x, rw[u]));
    }
  }
}

// handleChosen -> choose (:1170-1197, :622-640).  in {is_revocation, server, slot, value}; REV = false
// (fpx_vm_learn_chosen) does not read is_revocation.  A cell learned with and without isRevocation keeps it: the
// cell is a max.
template <bool REV>
__global__ void __launch_bounds__(256) vm_learn_chosen_kernel(VmParams P) {
  const Geometry& g = P.g;
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P.n) return;
  int4 rec = P.in[i];
  int server = rec.y, slot = rec.z;
  int local = local_slot(g, slot);
  if (local < 0 && local != kLocalRetired) { report_error(P.st, FPX_ERR_SLOT_RANGE, i); return; }
  if ((uint32_t)server >= (uint32_t)g.per_group) { report_error(P.st, FPX_ERR_BAD_ACCEPTOR, i); return; }
  if (local == kLocalRetired) return;   // retired: every server's entry is a ChosenEntry already, nothing to learn
  const unsigned long long rev = REV && rec.x != 0 ? kCellRevocation : 0ull;
  red_max_u64(&P.votes[cell_index(g, local, server)], kCellChosen | rev | (uint32_t)rec.w);   // ChosenEntry (:624)
  if (slot % g.per_group == server) {                                                       // phase2s.remove(slot) (:625)
    uint32_t* row = P.rows + (size_t)local * g.row_words;
    if (row[0] != kUnarmed) red_or_u32(row, kDoneBit);
  }
}

__global__ void vm_claim_init_kernel(unsigned long long* votes, size_t n_cells) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_cells) votes[2 * i + 1] = ~0ull;
}

}  // namespace fpx
