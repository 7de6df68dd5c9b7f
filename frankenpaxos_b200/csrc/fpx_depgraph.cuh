// fpx_depgraph.cuh -- EPaxos execution: the dependency graph on the GPU (SURVEY 8(f) rank 4).
//
//   Reference: depgraph.TarjanDependencyGraph, S/depgraph/TarjanDependencyGraph.scala:225-451 --
//   commit (:225-239, repeated keys ignored), updateExecuted (:241-244), executeByComponent (:296-318)
//   = Tarjan's strongly connected components interlaced with an eligibility check: a vertex is
//   executable iff everything it transitively depends on (executed keys excepted,
//   `dependencies.materializedDiff(executed)`, :372-448) is committed; components are returned in
//   reverse topological order, each sorted by (sequenceNumber, key) (:441-444).  Consumer:
//   epaxos.Replica.execute, S/epaxos/Replica.scala:569-600 hands the committed instance to the graph.
//
//   A depth-first search does not parallelise; the same RESULT is computed data-parallel, one
//   cooperative kernel, every phase a fixed point of an edge relaxation (one thread per vertex, grid
//   barrier per round):
//     eligibility   inel(v) = some dependency is neither committed nor executed, or inel(dependency)
//     components    trim (a vertex whose dependencies are all assigned is its own component), then
//                   colouring: every unassigned eligible vertex pushes the largest key that reaches it
//                   along its edges; a vertex whose colour is its own key is the root of a component,
//                   and the component is the set of vertices of that colour that reach the root
//     order         level(component) = 1 + max level of the components it depends on
//   and the executables are the eligible vertices sorted by (level, component, sequenceNumber, key)
//   (fpx_sort.cuh).  The reference's order among INDEPENDENT components is the iteration order of a
//   mutable.Map (:343) -- unpinned by its tests, which accept any; here it is (level, root key).
//   `numBlockers` (an early exit of that hash-order loop, :358-363) is not offered: every blocker is found.
#pragma once
#include "fpx_common.cuh"
#include "fpx_sort.cuh"

namespace fpx {

constexpr int kDgThreads = 1024;
constexpr int32_t kDgAbsent = 0, kDgCommitted = 1, kDgExecuted = 2;
constexpr uint32_t kDgNoLevel = 0x7fffffffu;

struct DgState {
  int32_t cap;                 // keys are 0 .. cap-1
  int32_t* status;             // [cap] absent / committed / executed
  int32_t* seq;                // [cap] sequence number
  int32_t* dep_off;            // [cap] first dependency in the pool
  int32_t* dep_cnt;            // [cap]
  int32_t* pool;               // dependency keys
  int32_t* claim;              // [cap] commit: lowest batch index that commits the key
  // execute scratch
  uint8_t* inel;               // [cap] committed but not executable
  uint8_t* blocker;            // [cap] uncommitted key something committed waits for
  uint8_t* mark;               // [cap]
  int32_t* color;              // [cap]
  int32_t* comp;               // [cap] component = its root key, -1 unassigned
  uint32_t* level;             // [cap] sort key: level of the component, kDgNoLevel = not executable now
  uint32_t* seq_key;           // [cap] sort key: sequence number, order-preserving unsigned
  uint32_t* comp_key;          // [cap] sort key: component
  uint32_t* flags;             // [0..2] changed flags in rotation, [3] number of executables
  DevStatus* st;
};

// commit, pass 1: the first record of the batch (delivery order) for a key wins (:230-234)
__global__ void dg_commit_claim_kernel(DgState S, const int32_t* keys, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int k = keys[i];
  if ((uint32_t)k >= (uint32_t)S.cap) { report_error(S.st, FPX_ERR_SLOT_RANGE, i); return; }
  if (S.status[k] == kDgAbsent) atomicMin(&S.claim[k], i);
}
// commit, pass 2: vertices(key) = Vertex(key, sequenceNumber, dependencies) (:238)
__global__ void dg_commit_apply_kernel(DgState S, const int32_t* keys, const int32_t* seqs, const int32_t* dep_off,
                                       const int32_t* deps, int n, int pool_base) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int k = keys[i];
  if ((uint32_t)k >= (uint32_t)S.cap || S.claim[k] != i) return;
  S.claim[k] = INT_MAX;
  S.status[k] = kDgCommitted;
  S.seq[k] = seqs[i];
  S.dep_off[k] = pool_base + dep_off[i];
  S.dep_cnt[k] = dep_off[i + 1] - dep_off[i];
  for (int d = dep_off[i]; d < dep_off[i + 1]; ++d) S.pool[pool_base + d] = deps[d];
}
// updateExecuted (:241-244)
__global__ void dg_update_executed_kernel(DgState S, const int32_t* keys, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int k = keys[i];
  if ((uint32_t)k >= (uint32_t)S.cap) { report_error(S.st, FPX_ERR_SLOT_RANGE, i); return; }
  S.status[k] = kDgExecuted;
}

// One fixed-point round is over when no thread raised flags[round % 3].  Three flags in rotation: while
// round r runs, CTA 0 clears the flag of round r+1; the flag of round r-1 may still be being read by CTAs
// that have not left that round's barrier yet, so it is left alone until round r+1.
// kDgMaxRounds bounds every loop (a defect must not hang a cooperative kernel).
constexpr int kDgRoundSlack = 64;
__device__ __forceinline__ bool dg_round_end(DgState& S, int& round) {
  grid_sync(S.st);
  const bool changed = __ldcg(&S.flags[round % 3]) != 0;
  round++;
  if (round > 8 * S.cap + kDgRoundSlack) {
    if (blockIdx.x == 0 && threadIdx.x == 0) report_error(S.st, FPX_ERR_CHECK_FAILED, 0);
    return false;
  }
  return changed;
}
__device__ __forceinline__ void dg_round_begin(DgState& S, int round) {
  if (blockIdx.x == 0 && threadIdx.x == 0) S.flags[(round + 1) % 3] = 0;
}
#define DG_RAISE(S, round) (S).flags[(round) % 3] = 1

__global__ void __launch_bounds__(kDgThreads, 1) dg_execute_kernel(DgState S) {
  const int stride = gridDim.x * kDgThreads;
  const int t0 = blockIdx.x * kDgThreads + threadIdx.x;
  int round = 0;
  if (t0 == 0) { S.flags[0] = 0; S.flags[1] = 0; S.flags[2] = 0; S.flags[3] = 0; }
  // ---- eligibility, seed: a dependency that is neither committed nor executed blocks (:386-392).
  // `blocker` is cleared by the host before the launch: vertex w's flag is set by whichever thread owns a
  // vertex depending on w, possibly in an earlier stride iteration than the one that reaches w.
  for (int v = t0; v < S.cap; v += stride) {
    S.comp[v] = -1;
    S.mark[v] = 0;
    S.level[v] = kDgNoLevel;
    uint8_t bad = 0;
    if (S.status[v] == kDgCommitted) {
      for (int d = 0; d < S.dep_cnt[v]; ++d) {
        int w = S.pool[S.dep_off[v] + d];
        if ((uint32_t)w >= (uint32_t)S.cap) { bad = 1; continue; }        // a key outside the graph can never be committed
        if (__ldcg(&S.status[w]) == kDgAbsent) { bad = 1; S.blocker[w] = 1; }
      }
    }
    S.inel[v] = bad;
  }
  grid_sync(S.st);
  // ---- eligibility, closure: ineligible dependencies make their dependents ineligible (:393-404)
  do {
    dg_round_begin(S, round);
    for (int v = t0; v < S.cap; v += stride) {
      if (S.status[v] != kDgCommitted || S.inel[v]) continue;
      for (int d = 0; d < S.dep_cnt[v]; ++d) {
        int w = S.pool[S.dep_off[v] + d];
        if ((uint32_t)w < (uint32_t)S.cap && S.status[w] == kDgCommitted && __ldcg(&S.inel[w])) {
          S.inel[v] = 1;
          DG_RAISE(S, round);
          break;
        }
      }
    }
  } while (dg_round_end(S, round));
  // from here on "live" = committed and eligible; executed dependencies are not edges (materializedDiff)
#define DG_LIVE(v) (S.status[v] == kDgCommitted && !S.inel[v])
  // ---- components: colouring until every live vertex is assigned
  while (true) {
    // trim: a vertex whose live dependencies are all assigned already is a component of its own (the
    // acyclic part of the graph -- chains -- never reaches the colouring)
    do {
      dg_round_begin(S, round);
      for (int v = t0; v < S.cap; v += stride) {
        if (!DG_LIVE(v) || S.comp[v] >= 0) continue;
        bool open = false;
        for (int d = 0; d < S.dep_cnt[v] && !open; ++d) {
          int w = S.pool[S.dep_off[v] + d];
          open = (uint32_t)w < (uint32_t)S.cap && w != v && DG_LIVE(w) && __ldcg(&S.comp[w]) < 0;
        }
        if (!open) { S.comp[v] = v; S.level[v] = 0; DG_RAISE(S, round); }
      }
    } while (dg_round_end(S, round));
    // any unassigned live vertex left?  colour = own key
    dg_round_begin(S, round);
    for (int v = t0; v < S.cap; v += stride) {
      if (DG_LIVE(v) && S.comp[v] < 0) { S.color[v] = v; S.mark[v] = 0; DG_RAISE(S, round); }
    }
    if (!dg_round_end(S, round)) break;
    // push the largest key that reaches a vertex along the edges (forward reachability)
    do {
      dg_round_begin(S, round);
      for (int v = t0; v < S.cap; v += stride) {
        if (!DG_LIVE(v) || S.comp[v] >= 0) continue;
        const int cv = __ldcg(&S.color[v]);
        for (int d = 0; d < S.dep_cnt[v]; ++d) {
          int w = S.pool[S.dep_off[v] + d];
          if ((uint32_t)w >= (uint32_t)S.cap || !DG_LIVE(w) || S.comp[w] >= 0) continue;
          if (atomicMax(&S.color[w], cv) < cv) DG_RAISE(S, round);
        }
      }
    } while (dg_round_end(S, round));
    // roots, then backward closure inside a colour class: v reaches the root iff some dependency of the
    // same colour does
    for (int v = t0; v < S.cap; v += stride)
      if (DG_LIVE(v) && S.comp[v] < 0 && S.color[v] == v) S.mark[v] = 1;
    grid_sync(S.st);
    do {
      dg_round_begin(S, round);
      for (int v = t0; v < S.cap; v += stride) {
        if (!DG_LIVE(v) || S.comp[v] >= 0 || S.mark[v]) continue;
        for (int d = 0; d < S.dep_cnt[v]; ++d) {
          int w = S.pool[S.dep_off[v] + d];
          if ((uint32_t)w >= (uint32_t)S.cap || !DG_LIVE(w) || S.comp[w] >= 0) continue;
          if (S.color[w] == S.color[v] && __ldcg(&S.mark[w])) { S.mark[v] = 1; DG_RAISE(S, round); break; }
        }
      }
    } while (dg_round_end(S, round));
    for (int v = t0; v < S.cap; v += stride)
      if (DG_LIVE(v) && S.comp[v] < 0 && S.mark[v]) { S.comp[v] = S.color[v]; S.level[v] = 0; }
    grid_sync(S.st);
  }
  // ---- order: level(v) = max over dependencies (level + 1 across components, level inside one)
  do {
    dg_round_begin(S, round);
    for (int v = t0; v < S.cap; v += stride) {
      if (!DG_LIVE(v)) continue;
      uint32_t lv = __ldcg(&S.level[v]);
      for (int d = 0; d < S.dep_cnt[v]; ++d) {
        int w = S.pool[S.dep_off[v] + d];
        if ((uint32_t)w >= (uint32_t)S.cap || !DG_LIVE(w)) continue;
        uint32_t lw = __ldcg(&S.level[w]) + (S.comp[w] != S.comp[v] ? 1u : 0u);
        if (lw > lv) lv = lw;
      }
      // members of one component share a level: also pull the component's root up to date
      if (lv > __ldcg(&S.level[v])) { S.level[v] = lv; DG_RAISE(S, round); }
      if (atomicMax(&S.level[S.comp[v]], lv) < lv) DG_RAISE(S, round);
      uint32_t lr = __ldcg(&S.level[S.comp[v]]);
      if (lr > lv) { S.level[v] = lr; DG_RAISE(S, round); }
    }
  } while (dg_round_end(S, round));
#undef DG_LIVE
  // ---- sort keys and the count of executables
  uint32_t cnt = 0;
  for (int v = t0; v < S.cap; v += stride) {
    const bool live = S.status[v] == kDgCommitted && !S.inel[v];
    S.seq_key[v] = (uint32_t)S.seq[v] ^ 0x80000000u;
    S.comp_key[v] = live ? (uint32_t)S.comp[v] : 0u;
    if (!live) S.level[v] = kDgNoLevel;
    cnt += live;
  }
  cnt = __reduce_add_sync(0xffffffffu, cnt);
  if ((threadIdx.x & 31) == 0 && cnt) atomicAdd(&S.flags[3], cnt);
}

// after the sorts: executables[p] = perm[p], head[p] = first member of its component; executed.add (:305-311)
__global__ void dg_emit_kernel(DgState S, const uint32_t* perm, int n_exec, int32_t* out_keys, uint8_t* out_head) {
  int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_exec) return;
  const int v = (int)perm[p];
  out_keys[p] = v;
  out_head[p] = p == 0 || S.comp[perm[p - 1]] != S.comp[v];
  S.status[v] = kDgExecuted;
}

}  // namespace fpx
