// fpx_conflict.cuh -- EPaxos's top-1 conflict index on the GPU (SURVEY 8(f) rank 4).
//
//   Reference: KeyValueStore.typedTopKConflictIndex(k = 1), S/statemachine/KeyValueStore.scala:219-302
//   (put :229-251, putSnapshot :253-254, getTopOneConflicts :256-300), TopOne S/util/TopOne.scala:6-24;
//   consumer epaxos.Replica.computeSequenceNumberAndDependencies, S/epaxos/Replica.scala:569-600, which for
//   every PreAccept first asks for the conflicts (:1252) and then indexes the command (:1274).
//
//   Per key the index keeps one TopOne of the gets and one of the sets: per leader column the largest
//   instance id + 1 (0 = none).  A get conflicts with the sets of its keys, a set with their gets and
//   sets; a command without keys conflicts with the snapshots only; snapshots conflict with everything.
//   For a batch in delivery order command i must see exactly the commands j < i: per (key, kind, column)
//   an EXCLUSIVE RUNNING MAX in delivery order -- the primitive of the acceptors' ballot compare-and-set
//   (fpx_acceptor.cuh), here over an open key space:
//     rows     every (command, key) access finds / claims its key's row of a resident open-addressing
//              table {sets[n], gets[n]}
//     sort     the accesses are grouped by row, delivery order kept inside a row (fpx_sort.cuh, stable)
//     scan     segmented exclusive prefix-max over the sorted accesses, vector state of 2n columns:
//              block-level segmented scans per 1024-access tile, tile carries chained by one CTA
//              (tile_carry_kernel, fpx_scan.cuh)
//     emit     query = resident row (as of before the batch) merged with the exclusive prefix, merged over
//              the command's keys with atomicMax into deps[i][:]; the last access of a row folds the
//              row's batch total into the table.
#pragma once
#include "fpx_common.cuh"
#include "fpx_scan.cuh"
#include "fpx_sort.cuh"

namespace fpx {

constexpr int kCiMaxLeaders = 8;
constexpr int kCiTile = 1024;
constexpr uint32_t kCiNoRow = 0xffffffffu;

struct CiParams {
  int32_t n_leaders, n_cmd, n_acc, mode;   // mode 0: query then put, 1: put only, 2: query only
  uint32_t row_mask;                       // table capacity - 1
  const int32_t *leader, *id, *key_off, *keys;
  const uint8_t* is_set;
  int32_t* tab_keys;                       // [cap] key of the row, INT32_MIN = empty
  int32_t* tab;                            // [cap][2][n_leaders]  sets, gets
  int32_t* tab_new;                        // [cap][2][n_leaders]  new value of the rows a batch touched
  int32_t* snapshots;                      // [n_leaders]
  uint32_t* acc_row;                       // [n_acc] row of access a (kCiNoRow: duplicate key of its command)
  int32_t* acc_cmd;                        // [n_acc]
  uint32_t* perm;                          // [n_acc] accesses sorted by (row, a)
  int32_t* tile_agg;                       // [tiles][2*n_leaders] aggregate of the tile's LAST segment
  uint32_t* tile_head;                     // [tiles] a row starts in the tile
  int32_t* tile_carry;                     // [tiles][2*n_leaders] prefix entering the tile's FIRST segment
  int32_t* deps_out;                       // [n_cmd][n_leaders]
  DevStatus* st;
};

constexpr int32_t kCiEmptyKey = INT32_MIN;

// (1) deps_out = snapshots; rows of every access (one thread per command: commands carry few keys).  acc_row
//     arrives all kCiNoRow (memset by the host), so a rejected command's accesses have no row.
__global__ void ci_rows_kernel(CiParams P) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P.n_cmd) return;
  if (P.mode != 1)
    for (int c = 0; c < P.n_leaders; ++c) P.deps_out[(size_t)i * P.n_leaders + c] = P.snapshots[c];   // :271 / :293, :261-262
  const int lo = P.key_off[i], hi = P.key_off[i + 1];
  if ((uint32_t)P.leader[i] >= (uint32_t)P.n_leaders || P.id[i] < 0 || hi < lo || lo < 0 || hi > P.n_acc) {
    report_error(P.st, FPX_ERR_INVALID_ARG, i);
    return;
  }
  for (int a = lo; a < hi; ++a) {
    const int key = P.keys[a];
    P.acc_cmd[a] = i;
    bool dup = false;
    for (int b = lo; b < a && !dup; ++b) dup = P.keys[b] == key;      // a key listed twice counts once
    uint32_t row = kCiNoRow;
    if (key == kCiEmptyKey) {
      report_error(P.st, FPX_ERR_INVALID_ARG, i);
    } else if (!dup) {
      uint32_t h = (uint32_t)mix64((uint64_t)(uint32_t)key) & P.row_mask;
      for (uint32_t probe = 0; probe <= P.row_mask; ++probe) {
        int32_t k = __ldcg(&P.tab_keys[h]);
        if (k == kCiEmptyKey && P.mode != 2) k = atomicCAS(&P.tab_keys[h], kCiEmptyKey, key);   // a query creates nothing
        if (k == key || (k == kCiEmptyKey && P.mode != 2)) { row = h; break; }
        if (k == kCiEmptyKey) break;                                                              // query of an unknown key
        h = (h + 1) & P.row_mask;
      }
      if (row == kCiNoRow && P.mode != 2) report_error(P.st, FPX_ERR_OVERFLOW_FULL, i);
    }
    P.acc_row[a] = row;
  }
}

// column of an access in the row's 2n-vector: sets first, then gets
__device__ __forceinline__ int ci_col(const CiParams& P, int cmd) {
  return (P.is_set[cmd] ? 0 : P.n_leaders) + P.leader[cmd];
}

// (2) kPass = 0: aggregate of every tile's last segment per column, and whether a row starts in the tile.
//     kPass = 1: exclusive prefixes (with the carry into the tile's first segment), query merge into
//                deps_out, and the new value of every row (written by the row's last access into tab_new).
template <int kPass>
__global__ void __launch_bounds__(kCiTile) ci_scan_kernel(CiParams P) {
  __shared__ int s_prev[kCiTile];
  const int tid = threadIdx.x;
  const int tile = blockIdx.x;
  const int j = tile * kCiTile + tid;                   // position in sorted order
  const bool live = j < P.n_acc;
  const uint32_t a = live ? P.perm[j] : 0u;
  const uint32_t row = live ? P.acc_row[a] : kCiNoRow;
  const int cmd = live ? P.acc_cmd[a] : 0;
  const bool head = live && (j == 0 || P.acc_row[P.perm[j - 1]] != row);   // first access of its row
  const bool real = live && row != kCiNoRow;
  const int my_col = real ? ci_col(P, cmd) : -1;
  const int my_val = real ? P.id[cmd] + 1 : 0;         // TopOne.put: max(id + 1) (:12-15)
  const int nc = 2 * P.n_leaders;
  int excl[2 * kCiMaxLeaders];
#pragma unroll
  for (int c = 0; c < 2 * kCiMaxLeaders; ++c) {
    if (c >= nc) break;
    const int contrib = (my_col == c && P.mode != 2) ? my_val : 0;   // a pure query indexes nothing
    SegVal<int> x = cta_scan<kCiTile, false>(SegVal<int>{contrib, head}, Seg<ScanMax>());
    if (kPass == 0) {
      if (tid == kCiTile - 1) {
        P.tile_agg[(size_t)tile * nc + c] = x.v;
        P.tile_head[tile] = x.f;
      }
      continue;
    }
    const int carry = P.tile_carry[(size_t)tile * nc + c];
    if (!x.f) x.v = max(x.v, carry);
    s_prev[tid] = x.v;
    __syncthreads();
    excl[c] = head ? 0 : (tid == 0 ? carry : s_prev[tid - 1]);   // inclusive value of the previous access of the row
    __syncthreads();
  }
  if (kPass == 0 || !real) return;
  const bool is_set = P.is_set[cmd] != 0;
  const int32_t* trow = P.tab + (size_t)row * nc;       // as of before the batch: pass 1 never writes `tab`
  const bool last_of_row = (j + 1 >= P.n_acc) || P.acc_row[P.perm[j + 1]] != row;
#pragma unroll
  for (int c = 0; c < 2 * kCiMaxLeaders; ++c) {
    if (c >= nc) break;
    const int e = max(excl[c], __ldcg(&trow[c]));
    // getTopOneConflicts (:256-300): the sets of the key always, its gets only for a set
    if (P.mode != 1 && (c < P.n_leaders || is_set) && e > 0)
      atomicMax(&P.deps_out[(size_t)cmd * P.n_leaders + (c < P.n_leaders ? c : c - P.n_leaders)], e);
    if (last_of_row && P.mode != 2) P.tab_new[(size_t)row * nc + c] = max(e, my_col == c ? my_val : 0);
  }
}

// (3) the rows' new values become resident (after every access of the batch has read the old ones)
__global__ void ci_fold_kernel(CiParams P) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= P.n_acc) return;
  const uint32_t row = P.acc_row[P.perm[j]];
  if (row == kCiNoRow) return;
  if (j + 1 < P.n_acc && P.acc_row[P.perm[j + 1]] == row) return;
  const int nc = 2 * P.n_leaders;
  for (int c = 0; c < nc; ++c) P.tab[(size_t)row * nc + c] = P.tab_new[(size_t)row * nc + c];
}

// putSnapshot (:253-254)
__global__ void ci_snapshot_kernel(int32_t* snapshots, int leader, int id) { snapshots[leader] = max(snapshots[leader], id + 1); }

}  // namespace fpx
