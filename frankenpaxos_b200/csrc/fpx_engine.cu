// fpx_engine.cu -- host side of libfpx.so: the C ABI of include/fpx.h.
//
// One fpx_engine owns, on one GPU: the vote cells of every acceptor of the
// config (flat slot x voter array of 64-bit {round, value} cells), the proxy
// leader's per-(slot, round) rows, the overflow table for secondary rounds, the
// replica log, one CUDA stream, and pinned/device staging for the host-pointer
// entry points.  No CPU fallback exists: without a CUDA device fpx_create fails
// with FPX_ERR_NO_DEVICE.
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <memory>
#include <new>
#include <string>
#include <vector>

#include "fpx_acceptor.cuh"
#include "fpx_arm.cuh"
#include "fpx_common.cuh"
#include "fpx_conflict.cuh"
#include "fpx_debug.h"
#include "fpx_depgraph.cuh"
#include "fpx_epaxos.cuh"
#include "fpx_epaxos_graph.cuh"
#include "fpx_host.h"
#include "fpx_ranges.cuh"
#include "fpx_reads.cuh"
#include "fpx_replica_misc.cuh"
#include "fpx_tally.cuh"
#include "fpx_vanilla.cuh"
#include "fpx_wire.cuh"
#include "fpx_wire_phase1.cuh"
#include "fpx_wire_reads.cuh"
#include "fpx_vm_revoke.cuh"

using namespace fpx;

constexpr int kMaxEvents = 16;
constexpr int kTallySmem = 200 * 1024 / (1024 / kTT);  // dynamic shared memory of a tally CTA (one CTA of 1024 threads per SM)
constexpr int kStepRing = 1024;
// votes one tally launch takes: its scan of the per-chunk counts (4 B per 1024 votes) uses at most 40 KB of the
// dynamic shared memory; a larger call is cut into several launches (tally_launch)
constexpr int32_t kTallyMaxSub = (40 * 1024 / 4) * kChunkVotes;

// The wire codec's device buffers of a handle (fpx_engine, fpx_epaxos), grown on demand: the host forms' copies of
// their inputs and outputs, and the encoders' tile sums
struct WireBuf { void* p = nullptr; size_t cap = 0; };
struct WireStage {
  WireBuf bytes, offs;                 // a message batch: bytes and offsets
  WireBuf kind, rec, sender, out, arena, voffs, tiles;
  WireBuf aux;                         // EPaxos: the encoder's output rows, the pack's local deps
  WireBuf rw_scratch, rw_out;          // the replica decode's per-message and per-tile scratch, its host-form output
  WireBuf p1_scratch, p1_out, spans;   // the leader's Phase 1: messages, entries, window; its host-form output; Phase2a spans
};

struct fpx_engine {
  CudaResources res;                   // every buffer, stream and event below
  fpx_config cfg;
  Geometry g;
  cudaStream_t stream = nullptr;
  cudaStream_t h2d_stream = nullptr, d2h_stream = nullptr;  // copy engines of the chunk-pipelined host calls
  cudaEvent_t ev[16] = {};
  // device state
  uint32_t* rows = nullptr;
  unsigned long long* ovf_keys = nullptr;
  uint32_t* ovf_rows = nullptr;
  unsigned long long* ovf_keys_spare = nullptr;   // fpx_retire_below rebuilds the overflow table into these and swaps
  uint32_t* ovf_rows_spare = nullptr;
  unsigned long long* votes = nullptr;
  int32_t* acc_round = nullptr;
  int32_t* acc_max_voted = nullptr;
  unsigned long long* rlog = nullptr;
  uint32_t vm_tag = 1;
  unsigned long long* vm_raise = nullptr;  // vanilla Mencius: raised entries' {voteRound, value}, on first Phase1a
  uint32_t* rng_tab = nullptr;             // mencius: (start, end, round) key table of the NoopRange path
  uint32_t* rng_tab_spare = nullptr;       // its rebuild target (fpx_retire_below)
  int32_t rng_cap = 0;
  int32_t* rng_dec = nullptr;              // per-record scratch of the range kernels (FPX_MAX_RANGE_BATCH)
  uint32_t rng_seq_base = 1;               // Phase2bNoopRange delivery sequence numbers
  int unit_ranges = 0;                     // a one-slot range was ever armed: arms must look at the range keys
  int32_t* mix = nullptr;                  // mencius: scratch of the mixed replica call (fpx_mencius_replica_inbound)
  // fpx_step_dev: CUDA events around the acceptor and tally kernels of the last kStepRing steps
  std::vector<cudaEvent_t> step_ev;        // [kStepRing][4], created on first use
  WireStage wire;
  DevStatus* st = nullptr;
  // multi-GPU exchange
  DevExchange* xch = nullptr;          // device copy of the exchange descriptor
  DevExchange h_xch;                   // host mirror
  unsigned long long* xch_table = nullptr;   // this engine's frontier table [kMaxShards]
  void* xch_opened[kMaxShards] = {};   // peer tables opened with cudaIpcOpenMemHandle
  uint32_t xch_epoch = 0;              // publications issued so far (host count)
  int32_t* xch_out = nullptr;          // result of fpx_global_watermark: [1 + kMaxShards]
  // scratch
  uint32_t* bits = nullptr;            // accept / win bitmask, max_batch/32 words
  int32_t* g_agg = nullptr;            // [2][kMaxGrid][kMaxKeys] acceptor kernel CTA aggregates
  uint32_t* g_wacc = nullptr;          // [kAccMaxSegments][kMaxGrid*kAW] accepted per warp range
  uint2* t_bw = nullptr;               // tally: completing-vote bitmap of the running batch + per-word prefix
  uint32_t* t_cc = nullptr;            // tally: completing votes per 1024-vote chunk
  void* t_tmp = nullptr;               // tally: Chosen records parked at their vote's index (max_batch * 8)
  int tally_path = 0;                  // 0 auto, 2 force the exact per-vote path
  int acc_segments = 0;                // acceptor kernel: 0 = from the batch size and the L2 size, else forced
  long long l2_bytes = 0;
  void* conflicts = nullptr;           // kMaxConflicts * 8 bytes (acceptor kernel)
  void* arm_conflicts = nullptr;       // kMaxConflicts * 8 bytes (arm kernel)
  uint32_t* arm_bits = nullptr;        // arm kernel: record i created its key, max_batch/32 words
  // staging for host-pointer calls
  void* d_in = nullptr;                // max_batch * 16
  void* d_out_a = nullptr;             // max_batch * 16 (p2b)
  void* d_out_b = nullptr;             // max_batch * 8  (nack / chosen)
  DevStatus* h_st = nullptr;           // pinned mirror
  // fpx_step_submit / fpx_step_wait: two lanes of device staging + pinned status
  struct Lane {
    void *d_p2a = nullptr, *d_p2b = nullptr, *d_arm = nullptr, *d_out_p2b = nullptr, *d_out_nack = nullptr, *d_out_chosen = nullptr;
    cudaEvent_t ev_p2a = nullptr, ev_p2b = nullptr, ev_acc = nullptr, ev_done = nullptr, ev_d2h = nullptr;
    DevStatus* h_st = nullptr;
    fpx_p2b* out_p2b = nullptr; fpx_nack* out_nack = nullptr; fpx_chosen* out_chosen = nullptr;
    int32_t n_p2a = 0;
    bool ready = false;                // every resource above exists
    bool busy = false;
  } lane[2];
  int lane_head = 0, lane_tail = 0, lanes_in_flight = 0;
  // host bookkeeping
  uint32_t parity = 0;                 // nack counter the next acceptor launch uses
  int grid_acceptor = 0;               // co-resident CTAs of the cooperative kernels
  int grid_tally = 0;
  int occ_acceptor = 0, occ_tally = 0; // resident CTAs per SM each kernel could have alone
  int tally_max_sub = 0;               // votes one tally launch takes (shared-memory scan of the chunk counts)
  int num_sms = 0;
  uint32_t seq_base = 1;               // Phase2b delivery sequence numbers
  uint32_t rseq_base = 1;              // Chosen delivery sequence numbers
  int32_t last_p2b_n = 0;
  int64_t launches = 0;
  std::string last_error;
};

// --------------------------------------------------------------------------- status blocks (DevStatus, ReadsDev)

// a fresh status block: no error, every other field 0
template <class S>
static S fresh_status() {
  S st;
  memset(&st, 0, sizeof(S));
  st.err_word = ~0ull;
  return st;
}

// writes `init` to the device's status block through the pinned mirror
template <class H, class S>
static int status_init(H* h, S* hs, S* ds, cudaStream_t s, const S& init = fresh_status<S>()) {
  *hs = init;
  CK(h, cudaMemcpyAsync(ds, hs, sizeof(S), cudaMemcpyHostToDevice, s));
  CK(h, cudaStreamSynchronize(s));
  return FPX_OK;
}

// The error word of a status block already copied to the host: *status is the first error's status (FPX_OK:
// none) and *err_index its record (-1: none, or an error of the reads handle that belongs to no record).  The
// word is cleared on the device (the reference process would be dead: cleared for the caller's reset), and the
// clear waited for if `sync`.  Returns FPX_ERR_CUDA if the clear failed, else FPX_OK.
template <class H, class S>
static int take_error(H* h, const S& hs, S* ds, cudaStream_t s, bool sync, int* status, int64_t* err_index) {
  const unsigned long long w = hs.err_word;
  *status = FPX_OK;
  if (err_index) *err_index = -1;
  if (w == ~0ull) return FPX_OK;
  long long idx = (long long)(w >> 8);
  if constexpr (std::is_same<S, ReadsDev>::value) idx = idx == kRdNoIndex ? -1 : idx;
  if (err_index) *err_index = idx;
  *status = -(int)(w & 0xff);
  const unsigned long long none = ~0ull;
  CK(h, cudaMemcpyAsync(&ds->err_word, &none, 8, cudaMemcpyHostToDevice, s));
  if (sync) CK(h, cudaStreamSynchronize(s));
  return FPX_OK;
}

// copies the status block to its pinned mirror once the stream's work is done, and takes its error (take_error)
template <class H, class S>
static int read_status(H* h, S* hs, S* ds, cudaStream_t s, int* status, int64_t* err_index) {
  CK(h, cudaMemcpyAsync(hs, ds, sizeof(S), cudaMemcpyDeviceToHost, s));
  CK(h, cudaStreamSynchronize(s));
  return take_error(h, *hs, ds, s, true, status, err_index);
}

// read_status for callers that return either: FPX_ERR_CUDA if a CUDA call failed, else the block's status
template <class H, class S>
static int collect_status(H* h, S* hs, S* ds, cudaStream_t s, int64_t* err_index) {
  int status = FPX_OK;
  const int c = read_status(h, hs, ds, s, &status, err_index);
  return c != FPX_OK ? c : status;
}

static int validate(const fpx_config* c) {
  // Config.checkValid, S/multipaxos/Config.scala:32-147 (clauses the path reads)
  if (c->f < 1) return FPX_ERR_CONFIG;
  if (c->num_leaders < c->f + 1) return FPX_ERR_CONFIG;
  if (c->num_replicas < c->f + 1) return FPX_ERR_CONFIG;
  if (c->num_acceptor_groups < 1 || c->acceptors_per_group < 1) return FPX_ERR_CONFIG;
  if (!c->flexible) {
    if (c->acceptors_per_group != 2 * c->f + 1) return FPX_ERR_CONFIG;
  } else {
    if (std::min(c->num_acceptor_groups, c->acceptors_per_group) - 1 < c->f) return FPX_ERR_CONFIG;
  }
  // engine limits
  if (c->protocol != FPX_MULTIPAXOS && c->protocol != FPX_MENCIUS && c->protocol != FPX_VANILLA_MENCIUS)
    return FPX_ERR_UNSUPPORTED;
  // S/vanillamencius/Config.scala:13-17: 2f+1 servers, no grid, one "group"
  if (c->protocol == FPX_VANILLA_MENCIUS && (c->flexible || c->num_acceptor_groups != 1)) return FPX_ERR_CONFIG;
  int lgroups = 1;
  if (c->protocol == FPX_MENCIUS) {
    // S/mencius/Config.scala:40-100: >= 1 leader group of >= f+1 leaders, groups of 2f+1 acceptors
    if (c->flexible || c->num_leader_groups < 1) return FPX_ERR_CONFIG;
    lgroups = c->num_leader_groups;
  } else if (c->num_leader_groups > 1) {
    return FPX_ERR_CONFIG;
  }
  long long total = (long long)lgroups * c->num_acceptor_groups * c->acceptors_per_group;
  if (total > FPX_MAX_ACCEPTORS) return FPX_ERR_UNSUPPORTED;
  int voters = c->flexible ? (int)total : c->acceptors_per_group;
  if (voters > FPX_MAX_VOTERS_PER_SLOT) return FPX_ERR_UNSUPPORTED;
  if (c->slot_capacity < 1 || c->max_batch < 1) return FPX_ERR_INVALID_ARG;
  if (c->shard_count < 1 || c->shard_index < 0 || c->shard_index >= c->shard_count) return FPX_ERR_INVALID_ARG;
  if (c->overflow_capacity < 0 || (c->overflow_capacity & (c->overflow_capacity - 1)) != 0)
    return FPX_ERR_INVALID_ARG;
  return FPX_OK;
}

static const void* tally_kernel_ptr(int row_words) {
  switch (row_words) {
    case 8: return (const void*)tally_kernel<8>;
    case 16: return (const void*)tally_kernel<16>;
    default: return (const void*)tally_kernel<32>;
  }
}

static int reset_state(fpx_engine* e) {
  const Geometry& g = e->g;
  size_t row_bytes = (size_t)g.local_slots * g.row_words * 4;
  CK(e, cudaMemsetAsync(e->rows, 0xff, row_bytes, e->stream));
  if (g.ovf_cap) {
    CK(e, cudaMemsetAsync(e->ovf_keys, 0xff, (size_t)g.ovf_cap * 8, e->stream));
    CK(e, cudaMemsetAsync(e->ovf_rows, 0xff, (size_t)g.ovf_cap * g.row_words * 4, e->stream));
  }
  CK(e, cudaMemsetAsync(e->votes, 0, ((size_t)g.local_slots * g.voters * 8) << g.cell_shift, e->stream));
  if (g.cell_shift) {   // vanilla Mencius: the claim word next to every vote cell starts at ~0
    vm_claim_init_kernel<<<(unsigned)(((size_t)g.local_slots * g.voters + 255) / 256), 256, 0, e->stream>>>(e->votes, (size_t)g.local_slots * g.voters);
    CK(e, cudaGetLastError());
  }
  CK(e, cudaMemsetAsync(e->acc_round, 0xff, kMaxKeys * 4, e->stream));      // round = -1 (Acceptor.scala:95)
  CK(e, cudaMemsetAsync(e->acc_max_voted, 0xff, kMaxKeys * 4, e->stream));  // maxVotedSlot = -1 (:104)
  CK(e, cudaMemsetAsync(e->rlog, 0xff, (size_t)g.local_slots * 8, e->stream));
  if (e->rng_tab) CK(e, cudaMemsetAsync(e->rng_tab, 0xff, (size_t)e->rng_cap * kRangeWords * 4, e->stream));
  e->rng_seq_base = 1;
  e->unit_ranges = 0;
  DevStatus init = fresh_status<DevStatus>();
  init.max_chosen_local = -1;
  init.max_armed_local = -1;
  init.wm_found = INT_MAX;
  init.ts_min_local = INT_MAX; init.ts_max_local = -1;
  init.ts_min_round = INT_MAX; init.ts_max_round = INT_MIN;
  init.watermark = g.shard_index;
  int c = status_init(e, e->h_st, e->st, e->stream, init);
  if (c != FPX_OK) return c;
  CK(e, cudaMemsetAsync(e->xch_table, 0, kMaxShards * 8, e->stream));
  e->h_xch.epoch = 0;
  e->xch_epoch = 0;
  CK(e, cudaMemcpyAsync(e->xch, &e->h_xch, sizeof(DevExchange), cudaMemcpyHostToDevice, e->stream));
  CK(e, cudaStreamSynchronize(e->stream));
  e->g.base_local = 0;
  e->g.base_ring = 0;
  e->g.slot_capacity = e->cfg.slot_capacity;
  e->parity = 0;
  e->seq_base = 1;
  e->rseq_base = 1;
  e->last_p2b_n = 0;
  return FPX_OK;
}

// The host form of a call on the staging buffer: `bytes` of `in` to d_in, `launch(d_in)`, then fpx_sync into *r
// (a local one if null) and *err_index.
template <class F>
static int staged_call(fpx_engine* e, const void* in, size_t bytes, int64_t* err_index, fpx_sync_result* r, F launch) {
  CK(e, cudaSetDevice(e->cfg.device));
  CK(e, cudaMemcpyAsync(e->d_in, in, bytes, cudaMemcpyHostToDevice, e->stream));
  int c = launch(e->d_in);
  if (c != FPX_OK) return c;
  fpx_sync_result local;
  if (!r) r = &local;
  r->err_index = -1;   // fpx_sync leaves *r alone when a CUDA call fails
  c = fpx_sync(e, r);
  if (err_index) *err_index = r->err_index;
  return c;
}

extern "C" {

int fpx_abi_version(void) { return FPX_ABI_VERSION; }

const char* fpx_strerror(int s) {
  switch (s) {
    case FPX_OK: return "ok";
    case FPX_ERR_INVALID_ARG: return "invalid argument";
    case FPX_ERR_CONFIG: return "Config.checkValid failed";
    case FPX_ERR_CUDA: return "CUDA error";
    case FPX_ERR_UNKNOWN_SLOT_ROUND: return "Phase2b for a (slot, round) that was never armed (logger.fatal)";
    case FPX_ERR_BAD_ACCEPTOR: return "acceptor is not a member of the quorum system (require)";
    case FPX_ERR_SLOT_RANGE: return "slot out of range for this engine/shard";
    case FPX_ERR_ROUND_RANGE: return "round out of range";
    case FPX_ERR_OVERFLOW_FULL: return "secondary (slot, round) overflow table full";
    case FPX_ERR_CONFLICT: return "too many same-key/different-value conflicts in one batch";
    case FPX_ERR_NO_DEVICE: return "no CUDA device";
    case FPX_ERR_UNSUPPORTED: return "configuration not supported by this engine build";
    case FPX_ERR_BATCH_ORDER: return "batch contract violated (fpx_epaxos_*: nothing applied, split the batch at err_index; vanilla Mencius Phase2a / Mencius range fill: half applied, fpx_reset)";
    case FPX_ERR_CHECK_FAILED: return "a logger.check of the reference failed";
    case FPX_ERR_WIRE: return "malformed protobuf message (InvalidProtocolBufferException)";
    case FPX_ERR_EXCHANGE_TIMEOUT: return "a shard of the log did not publish its watermark in time";
    case FPX_ERR_EPAXOS_STATE: return "transitionToPreAcceptPhase on a committed instance / regressing ballot";
    default: return "unknown status";
  }
}

const char* fpx_last_error(const fpx_engine* e) { return e ? e->last_error.c_str() : ""; }

int fpx_create(fpx_engine** out, const fpx_config* cfg) {
  if (!out || !cfg || cfg->struct_size != (int32_t)sizeof(fpx_config)) return FPX_ERR_INVALID_ARG;
  *out = nullptr;
  int v = validate(cfg);
  if (v != FPX_OK) return v;
  if (!device_exists(cfg->device)) return FPX_ERR_NO_DEVICE;
  std::unique_ptr<fpx_engine> e(new (std::nothrow) fpx_engine());   // freed with all it holds on a failed return
  if (!e) return FPX_ERR_INVALID_ARG;
  e->cfg = *cfg;
  CudaResources& R = e->res;
  R.device = cfg->device;
  Geometry& g = e->g;
  g.protocol = cfg->protocol;
  g.f = cfg->f;
  g.lgroups = cfg->protocol == FPX_MENCIUS ? cfg->num_leader_groups : 1;
  g.agroups = cfg->num_acceptor_groups;
  g.groups = g.lgroups * g.agroups;
  g.per_group = cfg->acceptors_per_group;
  g.flexible = cfg->flexible ? 1 : 0;
  g.num_leaders = cfg->num_leaders;
  g.num_keys = g.groups * g.per_group;
  g.voters = g.flexible ? g.num_keys : g.per_group;
  g.quorum = g.f + 1;
  g.row_words = g.voters <= 6 ? 8 : (g.voters <= 14 ? 16 : 32);
  g.slot_capacity = cfg->slot_capacity;
  g.shard_index = cfg->shard_index;
  g.shard_count = cfg->shard_count;
  g.local_slots = (cfg->slot_capacity - cfg->shard_index + cfg->shard_count - 1) / cfg->shard_count;
  if (g.local_slots < 1) g.local_slots = 1;
  g.base_local = 0;
  g.base_ring = 0;
  g.cell_shift = cfg->protocol == FPX_VANILLA_MENCIUS ? 1 : 0;
  g.ovf_cap = cfg->overflow_capacity;
  g.ovf_mask = g.ovf_cap ? (uint32_t)g.ovf_cap - 1u : 0u;
  g.m_groups = ~0ull / (unsigned long long)g.groups + 1ull;
  g.m_shards = ~0ull / (unsigned long long)g.shard_count + 1ull;
  g.m_lgroups = ~0ull / (unsigned long long)g.lgroups + 1ull;
  g.m_agroups = ~0ull / (unsigned long long)g.agroups + 1ull;

  CK(e, cudaSetDevice(cfg->device));
  CK(e, R.stream(&e->stream));
  CK(e, R.stream(&e->h2d_stream));
  CK(e, R.stream(&e->d2h_stream));
  for (int i = 0; i < kMaxEvents; ++i) CK(e, R.event(&e->ev[i], cudaEventDisableTiming));
  size_t mb = (size_t)cfg->max_batch;
  CK(e, R.alloc(&e->rows, (size_t)g.local_slots * g.row_words * 4));
  if (g.ovf_cap) {
    CK(e, R.alloc(&e->ovf_keys, (size_t)g.ovf_cap * 8));
    CK(e, R.alloc(&e->ovf_rows, (size_t)g.ovf_cap * g.row_words * 4));
    CK(e, R.alloc(&e->ovf_keys_spare, (size_t)g.ovf_cap * 8));
    CK(e, R.alloc(&e->ovf_rows_spare, (size_t)g.ovf_cap * g.row_words * 4));
  }
  CK(e, R.alloc(&e->votes, ((size_t)g.local_slots * g.voters * 8) << g.cell_shift));
  CK(e, R.alloc(&e->acc_round, kMaxKeys * 4));
  CK(e, R.alloc(&e->acc_max_voted, kMaxKeys * 4));
  CK(e, R.alloc(&e->rlog, (size_t)g.local_slots * 8));
  if (cfg->protocol == FPX_MENCIUS) {
    e->rng_cap = std::max(1024, g.ovf_cap);
    CK(e, R.alloc(&e->rng_tab, (size_t)e->rng_cap * kRangeWords * 4));
    CK(e, R.alloc(&e->rng_tab_spare, (size_t)e->rng_cap * kRangeWords * 4));
    // fpx_mencius_replica_inbound: {split, ranges, -, -}, the ranges' indices, the per-tile counts
    const size_t tiles = ((size_t)cfg->max_batch + kMixTile - 1) / kMixTile;
    CK(e, R.alloc(&e->mix, (4 + (size_t)FPX_MAX_RANGE_BATCH + tiles + 1) * 4));
  }
  if (cfg->protocol != FPX_MULTIPAXOS) CK(e, R.alloc(&e->rng_dec, (size_t)(FPX_MAX_RANGE_BATCH + 1) * 4));
  CK(e, R.alloc(&e->st, sizeof(DevStatus)));
  CK(e, R.alloc(&e->xch, sizeof(DevExchange)));
  CK(e, R.alloc(&e->xch_table, kMaxShards * 8));
  CK(e, R.alloc(&e->xch_out, (1 + kMaxShards) * 4));
  CK(e, R.alloc(&e->bits, (mb / 32 + 2) * 4));
  CK(e, R.alloc(&e->g_agg, (size_t)2 * kMaxGrid * kMaxKeys * 4));
  CK(e, R.alloc(&e->g_wacc, (size_t)kAccMaxSegments * kMaxGrid * kAW * 4));
  CK(e, R.alloc(&e->t_bw, (mb / kChunkVotes + 2) * 32 * 8));
  CK(e, R.alloc(&e->t_cc, (mb / kChunkVotes + 2) * 4));
  CK(e, R.alloc(&e->t_tmp, (mb + kChunkVotes) * 8));   // padded to a whole chunk: phase D loads unconditionally
  {
    // cooperative (co-resident) grids: SMs x resident CTAs per SM
    cudaDeviceProp prop;
    CK(e, cudaGetDeviceProperties(&prop, cfg->device));
    if (!prop.cooperativeLaunch) return FPX_ERR_UNSUPPORTED;
    e->num_sms = prop.multiProcessorCount;
    e->l2_bytes = prop.l2CacheSize;
    int occ = 0;
    CK(e, cudaFuncSetAttribute(acceptor_phase2a_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                               (kMaxKeys + kAccMaxSegments) * kAT * 4));
    CK(e, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, acceptor_phase2a_kernel, kAT,
                                                        (size_t)(g.num_keys + kAccMaxSegments) * kAT * 4));
    e->occ_acceptor = std::max(occ, 1);
    e->grid_acceptor = std::min(std::max(occ, 1) * e->num_sms, kMaxGrid);
    // the tally's dynamic shared memory: scan of the per-chunk counts (4 B per 1024 votes) + the CTA's kept
    // {vote, value} entries of the sweep (8 B per window row); one launch takes at most 40 KB of it for the scan
    const int smem_cap = kTallySmem;
    e->tally_max_sub = kTallyMaxSub;
    const void* tk = tally_kernel_ptr(g.row_words);
    CK(e, cudaFuncSetAttribute(tk, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_cap));
    CK(e, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, tk, kTT, smem_cap));
    e->occ_tally = std::max(occ, 1);
    e->grid_tally = std::min(std::max(occ, 1) * e->num_sms, kMaxGrid);
  }
  CK(e, R.alloc(&e->conflicts, kMaxConflicts * 8));
  CK(e, R.alloc(&e->arm_conflicts, kMaxConflicts * 8));
  CK(e, R.alloc(&e->arm_bits, (mb / 32 + 2) * 4));
  CK(e, R.alloc(&e->d_in, mb * 16));
  CK(e, R.alloc(&e->d_out_a, mb * 16));
  CK(e, R.alloc(&e->d_out_b, mb * 8));
  CK(e, R.alloc_pinned(&e->h_st, sizeof(DevStatus)));
  memset(&e->h_xch, 0, sizeof(e->h_xch));
  e->h_xch.n = g.shard_count <= kMaxShards ? g.shard_count : 0;
  e->h_xch.mine = g.shard_index;
  e->h_xch.tabs[g.shard_index < kMaxShards ? g.shard_index : 0] = g.shard_count <= kMaxShards ? e->xch_table : nullptr;
  e->h_xch.enabled = g.shard_count > 1 && g.shard_count <= kMaxShards;
  int r = reset_state(e.get());
  if (r != FPX_OK) return r;
  // test / A-B knob: FPX_TALLY_PATH=exact makes every tally launch take the per-vote path
  if (const char* tp = getenv("FPX_TALLY_PATH")) e->tally_path = strcmp(tp, "exact") == 0 ? 2 : 0;
  *out = e.release();
  return FPX_OK;
}

void fpx_destroy(fpx_engine* e) {
  if (!e) return;
  e->res.sync();   // no kernel reads a peer's table once its mapping is closed
  for (void* p : e->xch_opened) if (p) cudaIpcCloseMemHandle(p);
  delete e;
}

int fpx_reset(fpx_engine* e) {
  if (!e) return FPX_ERR_INVALID_ARG;
  CK(e, cudaSetDevice(e->cfg.device));
  return reset_state(e);
}

void* fpx_stream(fpx_engine* e) { return e ? (void*)e->stream : nullptr; }

// Slide the live window: every slot below `slot` is chosen and executed (slot <= the watermark this engine last
// published) and will not be needed again -- its row, vote cells and log entry are recycled for the slots
// slot_capacity ahead.  Messages for retired slots afterwards behave as the reference's would on a key that is
// Done / a log entry that exists: arms, votes and Chosen records are ignored, a Phase2a is still answered
// (round compare, Phase2b / Nack) but not recorded.  Vanilla Mencius answers it with reply kind 3.
// The key tables (secondary (slot, round) keys, mencius noop ranges) drop the keys of retired slots: each is
// rebuilt into its spare copy and the two are swapped -- kernels take PLState / RangeTable by value at launch,
// and every earlier launch has finished (fpx_sync).  A table that holds no key (the count the insert paths keep
// in the status block, read by that same sync) is left alone, so the steady state costs one recycle_kernel.
static int rebuild_tables(fpx_engine* e) {
  const Geometry& g = e->g;
  if (g.ovf_cap && e->h_st->ovf_used != 0) {
    CK(e, cudaMemsetAsync(e->ovf_keys_spare, 0xff, (size_t)g.ovf_cap * 8, e->stream));
    CK(e, cudaMemsetAsync(e->ovf_rows_spare, 0xff, (size_t)g.ovf_cap * g.row_words * 4, e->stream));
    CK(e, cudaMemsetAsync(&e->st->ovf_used, 0, 4, e->stream));
    ovf_rebuild_kernel<<<(g.ovf_cap + 255) / 256, 256, 0, e->stream>>>(g, e->ovf_keys, e->ovf_rows, e->ovf_keys_spare,
                                                                      e->ovf_rows_spare, &e->st->ovf_used);
    e->launches++;
    CK(e, cudaGetLastError());
    std::swap(e->ovf_keys, e->ovf_keys_spare);
    std::swap(e->ovf_rows, e->ovf_rows_spare);
  }
  if (e->rng_tab && e->h_st->rng_used != 0) {
    CK(e, cudaMemsetAsync(e->rng_tab_spare, 0xff, (size_t)e->rng_cap * kRangeWords * 4, e->stream));
    CK(e, cudaMemsetAsync(&e->st->rng_used, 0, 4, e->stream));
    range_rebuild_kernel<<<(e->rng_cap + 255) / 256, 256, 0, e->stream>>>(
        g, RangeTable{e->rng_tab, (uint32_t)e->rng_cap - 1u, e->rng_cap}, e->rng_tab_spare, &e->st->rng_used);
    e->launches++;
    CK(e, cudaGetLastError());
    std::swap(e->rng_tab, e->rng_tab_spare);
  }
  return FPX_OK;
}

int fpx_retire_below(fpx_engine* e, int32_t slot) {
  if (!e || slot < 0) return FPX_ERR_INVALID_ARG;
  CK(e, cudaSetDevice(e->cfg.device));
  fpx_sync_result r;
  int c = fpx_sync(e, &r);
  if (c != FPX_OK) return c;
  if (slot > r.watermark) return FPX_ERR_INVALID_ARG;                    // only the executed prefix may go
  Geometry& g = e->g;
  // first ordinal of this shard whose slot is >= `slot`
  long long new_base = ((long long)slot - g.shard_index + g.shard_count - 1) / g.shard_count;
  if (new_base < g.base_local) new_base = g.base_local;
  const int count = (int)std::min<long long>(new_base - g.base_local, g.local_slots);
  if (count == 0) return FPX_OK;
  recycle_kernel<<<std::min(count * 8 + 255, kSms * 2048) / 256 + 1, 256, 0, e->stream>>>(g, e->rows, e->votes, e->rlog, 0, count);
  e->launches++;
  CK(e, cudaGetLastError());
  g.base_local = (int32_t)new_base;
  g.base_ring = (int32_t)(new_base % g.local_slots);
  long long cap = (long long)e->cfg.slot_capacity + (long long)g.base_local * g.shard_count;
  g.slot_capacity = (int32_t)std::min<long long>(cap, 0x7fffffffll);
  return rebuild_tables(e);
}

int fpx_set_coop_ctas_per_sm(fpx_engine* e, int32_t ctas_per_sm) {
  if (!e || ctas_per_sm < 0) return FPX_ERR_INVALID_ARG;
  int a = ctas_per_sm == 0 ? e->occ_acceptor : std::min(e->occ_acceptor, ctas_per_sm);
  int t = ctas_per_sm == 0 ? e->occ_tally : std::min(e->occ_tally, ctas_per_sm);
  e->grid_acceptor = std::min(a * e->num_sms, kMaxGrid);
  e->grid_tally = std::min(t * e->num_sms, kMaxGrid);
  return FPX_OK;
}

// Undocumented profiling aid (not part of include/fpx.h): phase-boundary
// timestamps (ns) CTA 0 of the last acceptor / tally launch recorded.
int fpx_debug_phase_times(fpx_engine* e, unsigned long long* acceptor8, unsigned long long* tally8) {
  if (!e) return FPX_ERR_INVALID_ARG;
  CK(e, cudaStreamSynchronize(e->stream));
  CK(e, cudaMemcpy(acceptor8, e->st->t_acceptor, 64, cudaMemcpyDeviceToHost));
  CK(e, cudaMemcpy(tally8, e->st->t_tally, 64, cudaMemcpyDeviceToHost));
  return FPX_OK;
}
int64_t fpx_launch_count(const fpx_engine* e) { return e ? e->launches : 0; }
// Undocumented test/profiling aids: force the tally's exact per-vote path (path = 2; 0 = automatic), and
// which paths the last tally and arm launches took.
int fpx_debug_set_tally_path(fpx_engine* e, int32_t path) {
  if (!e || (path & ~6)) return FPX_ERR_INVALID_ARG;
  e->tally_path = path;
  return FPX_OK;
}
// Undocumented test/profiling aid: cut every acceptor launch into `segments` pipelined segments
// (1 .. kAccMaxSegments; 0 = automatic, from the batch size and the L2 size).
int fpx_debug_set_acceptor_segments(fpx_engine* e, int32_t segments) {
  if (!e || segments < 0 || segments > kAccMaxSegments) return FPX_ERR_INVALID_ARG;
  e->acc_segments = segments;
  return FPX_OK;
}
// Undocumented test aid: cut every tally call into launches of at most `votes` votes (1 .. kTallyMaxSub;
// 0 = kTallyMaxSub), so that small batches run the state a call carries from one launch to the next.
int fpx_debug_set_tally_max_sub(fpx_engine* e, int32_t votes) {
  if (!e || votes < 0 || votes > kTallyMaxSub) return FPX_ERR_INVALID_ARG;
  e->tally_max_sub = votes == 0 ? kTallyMaxSub : votes;
  return FPX_OK;
}
// out[0]: the last tally launch's path (1 sweep, 2 exact); out[1]: the last arm launch's (1 per-record CAS,
// 2 certified batch of fresh keys, plain row stores); 0 = no such launch since the engine was created or reset.
int fpx_debug_last_paths(fpx_engine* e, int32_t* out) {
  if (!e || !out) return FPX_ERR_INVALID_ARG;
  CK(e, cudaStreamSynchronize(e->stream));
  CK(e, cudaMemcpy(&out[0], &e->st->ts_path, 4, cudaMemcpyDeviceToHost));
  CK(e, cudaMemcpy(&out[1], &e->st->arm_path, 4, cudaMemcpyDeviceToHost));
  return FPX_OK;
}
// Undocumented test aids: the host's 32-bit counters {seq_base (Phase2b stamps), rseq_base (Chosen log numbers),
// rng_seq_base (Phase2bNoopRange stamps), vm_tag (vanilla Mencius batch tag)}, so that a test can start them just
// below their wrap and run the renormalization and tag-reuse paths through real calls.  Host fields only: no
// device memory is written.  Each value must lie in 1 .. 0xfffffffe, the range the counters themselves take.
static bool counter_ok(uint32_t v) { return v != 0u && v != 0xffffffffu; }
int fpx_debug_set_counters(fpx_engine* e, uint32_t seq_base, uint32_t rseq_base, uint32_t rng_seq_base, uint32_t vm_tag) {
  if (!e || !counter_ok(seq_base) || !counter_ok(rseq_base) || !counter_ok(rng_seq_base) || !counter_ok(vm_tag))
    return FPX_ERR_INVALID_ARG;
  e->seq_base = seq_base;
  e->rseq_base = rseq_base;
  e->rng_seq_base = rng_seq_base;
  e->vm_tag = vm_tag;
  return FPX_OK;
}
int fpx_debug_get_counters(fpx_engine* e, uint32_t* out) {
  if (!e || !out) return FPX_ERR_INVALID_ARG;
  out[0] = e->seq_base; out[1] = e->rseq_base; out[2] = e->rng_seq_base; out[3] = e->vm_tag;
  return FPX_OK;
}

// --------------------------------------------------------------------------- device entry points

static int check_n(fpx_engine* e, const void* p, int32_t n) {
  if (!e || n < 0 || n > e->cfg.max_batch || (n > 0 && !p)) return FPX_ERR_INVALID_ARG;
  return FPX_OK;
}

static ArmParams arm_params(fpx_engine* e, const fpx_p2a* d_in, int32_t n, int vanilla) {
  ArmParams P;
  P.g = e->g;
  P.pl = PLState{e->rows, e->ovf_keys, e->ovf_rows};
  P.in = (const int4*)d_in;
  P.n = n;
  P.st = e->st;
  P.conflicts = (ArmConflict*)e->arm_conflicts;
  P.win_bits = e->arm_bits;
  P.votes = e->votes;
  P.vanilla = vanilla;
  P.rng = RangeTable{e->rng_tab, (uint32_t)e->rng_cap - 1u, e->rng_cap};
  P.check_rng = e->unit_ranges;
#if defined(FPX_PROFILE_ARM_NOCAS) || defined(FPX_PROFILE_ARM_STORE)
  P.fast = 0;   // attribution builds time the per-record loop
#else
  P.fast = !vanilla && !P.check_rng;
#endif
  return P;
}

static int arm_launch(fpx_engine* e, const fpx_p2a* d_in, int32_t n, int vanilla) {
  int c = check_n(e, d_in, n);
  if (c != FPX_OK || n == 0) return c;
  ArmParams P = arm_params(e, d_in, n, vanilla);
  int arm_blocks = std::min((n + kArmThreads * kArmUnroll - 1) / (kArmThreads * kArmUnroll), e->num_sms);
  void* args[] = {&P};
  if (P.fast)
    CK(e, cudaLaunchCooperativeKernel((const void*)arm_kernel<true>, dim3(arm_blocks), dim3(kArmThreads), args, 0, e->stream));
  else
    arm_kernel<false><<<arm_blocks, kArmThreads, 0, e->stream>>>(P);
  e->launches++;
  CK(e, cudaGetLastError());
  return FPX_OK;
}

int fpx_proxyleader_arm_dev(fpx_engine* e, const fpx_p2a* d_in, int32_t n) {
  if (e && e->g.protocol == FPX_VANILLA_MENCIUS) return FPX_ERR_UNSUPPORTED;  // use fpx_vm_client_request
  return arm_launch(e, d_in, n, 0);
}

static int acceptor_launch(fpx_engine* e, const fpx_p2a* d_in, int32_t n, fpx_p2b* d_out_p2b, fpx_nack* d_out_nack,
                           int append, cudaStream_t stream);

int fpx_acceptor_phase2a_dev(fpx_engine* e, const fpx_p2a* d_in, int32_t n, fpx_p2b* d_out_p2b,
                             fpx_nack* d_out_nack) {
  return acceptor_launch(e, d_in, n, d_out_p2b, d_out_nack, 0, e ? e->stream : nullptr);
}

static int acceptor_launch(fpx_engine* e, const fpx_p2a* d_in, int32_t n, fpx_p2b* d_out_p2b, fpx_nack* d_out_nack,
                           int append, cudaStream_t stream) {
  int c = check_n(e, d_in, n);
  if (c != FPX_OK) return c;
  if (n > 0 && (!d_out_p2b || !d_out_nack)) return FPX_ERR_INVALID_ARG;
  if (e->g.protocol == FPX_VANILLA_MENCIUS) return FPX_ERR_UNSUPPORTED;  // use fpx_vm_phase2a
  if (n == 0) {
    if (!append) CK(e, cudaMemsetAsync(&e->st->n_p2b, 0, 8, stream));
    return FPX_OK;
  }
  AcceptorParams P;
  P.g = e->g;
  P.in = (const int4*)d_in;
  P.n = n;
  P.out_p2b = (int4*)d_out_p2b;
  P.out_nack = (int2*)d_out_nack;
  P.votes = e->votes;
  P.acc_round = e->acc_round;
  P.acc_max_voted = e->acc_max_voted;
  P.accept_bits = e->bits;
  P.g_agg = e->g_agg;
  P.g_wacc = e->g_wacc;
  P.st = e->st;
  P.conflicts = (VoteConflict*)e->conflicts;
  int grid = std::max(1, std::min(e->grid_acceptor, (n + kAT - 1) / kAT));
  P.segments = e->acc_segments > 0 ? e->acc_segments : acceptor_segments(n, e->l2_bytes);
  P.parity = e->parity;
  P.append = append;
  e->parity ^= 1u;
  void* args[] = {&P};
  CK(e, cudaLaunchCooperativeKernel((const void*)acceptor_phase2a_kernel, dim3(grid), dim3(kAT), args,
                                    (size_t)(e->g.num_keys + P.segments) * kAT * 4, stream));
  e->launches++;
  CK(e, cudaGetLastError());
  return FPX_OK;
}

static int renormalize_rlog_if_needed(fpx_engine* e, int32_t bound);

// fuse: 0 = the proxy leader alone; 1 = + the co-located replica's handleChosen and watermark (fpx_step_dev)
static int tally_launch(fpx_engine* e, const fpx_p2b* d_in, int32_t n, fpx_chosen* d_out, int fuse, int32_t* d_wm) {
  int c = check_n(e, d_in, n);
  if (c != FPX_OK) return c;
  if (n > 0 && !d_out) return FPX_ERR_INVALID_ARG;
  e->last_p2b_n = n;
  if (n == 0) {
    CK(e, cudaMemsetAsync(&e->st->n_chosen, 0, 4, e->stream));
    return fuse ? fpx_chosen_watermark_dev(e, d_wm) : FPX_OK;
  }
  if (fuse) {
    c = renormalize_rlog_if_needed(e, 2 * n > n ? 2 * n : n);
    if (c != FPX_OK) return c;
  }
  if (e->seq_base > 0xffffffffu - (uint32_t)n - 16u) {
    size_t nrows = (size_t)e->g.local_slots;
    renormalize_stamps_kernel<<<(unsigned)((nrows + 255) / 256), 256, 0, e->stream>>>(e->g, e->rows, nrows);
    if (e->g.ovf_cap)
      renormalize_stamps_kernel<<<(e->g.ovf_cap + 255) / 256, 256, 0, e->stream>>>(e->g, e->ovf_rows,
                                                                                   (size_t)e->g.ovf_cap);
    e->launches += 2;
    e->seq_base = 1;
  }
  const void* tk = tally_kernel_ptr(e->g.row_words);
  for (int32_t done = 0; done < n;) {
    int32_t sub = std::min(n - done, e->tally_max_sub);
    int grid = std::max(1, std::min(e->grid_tally, (sub + kTT - 1) / kTT));
    TallyParams P;
    P.g = e->g;
    P.pl = PLState{e->rows, e->ovf_keys, e->ovf_rows};
    P.in = (const int4*)d_in + done;
    P.n = sub;
    P.seq_base = e->seq_base;
    P.out_chosen = (int2*)d_out;
    P.bw = e->t_bw;
    P.cc = e->t_cc;
    P.tmp = (int2*)e->t_tmp;
    P.first = done == 0;
    P.index_base = done;                           // error indices are call indices (first offender in delivery order)
    P.path = e->tally_path;
    P.votes = e->votes;
    P.rlog = fuse ? e->rlog : nullptr;
    P.rseq_base = e->rseq_base + (uint32_t)done;   // later sub-launches number their records after earlier ones
    P.fuse_watermark = fuse && done + sub == n;
    P.d_watermark = d_wm;
    P.xch = e->xch;
    P.st = e->st;
    e->seq_base += (uint32_t)sub;
    void* args[] = {&P};
    const int nchunks = (sub + kChunkVotes - 1) / kChunkVotes;
    const size_t smem = kTallySmem;
    P.keep_cap = (int)((smem - (size_t)((nchunks + 1) & ~1) * 4) / 8);
    CK(e, cudaLaunchCooperativeKernel(tk, dim3(grid), dim3(kTT), args, smem, e->stream));
    e->launches++;
    done += sub;
  }
  if (fuse) e->xch_epoch++;                    // the fused tail published the watermark once
  if (fuse) e->rseq_base += 2u * (uint32_t)n;  // numbers used: below rseq_base + done + sub <= rseq_base + 2n
  CK(e, cudaGetLastError());
  return FPX_OK;
}

int fpx_proxyleader_phase2b_dev(fpx_engine* e, const fpx_p2b* d_in, int32_t n, fpx_chosen* d_out) {
  return tally_launch(e, d_in, n, d_out, 0, nullptr);
}

static int renormalize_rlog_if_needed(fpx_engine* e, int32_t bound) {
  if (e->rseq_base > 0xffffffffu - (uint32_t)bound - 16u) {
    size_t nl = (size_t)e->g.local_slots;
    renormalize_rlog_kernel<<<(unsigned)((nl + 255) / 256), 256, 0, e->stream>>>(e->rlog, nl);
    e->launches++;
    e->rseq_base = 1;
    CK(e, cudaGetLastError());
  }
  return FPX_OK;
}

static int replica_launch(fpx_engine* e, const fpx_chosen* d_in, int32_t n, int32_t bound) {
  if (bound == 0) return FPX_OK;
  int rc = renormalize_rlog_if_needed(e, bound);
  if (rc != FPX_OK) return rc;
  ReplicaParams P;
  P.g = e->g;
  P.in = (const int2*)d_in;
  P.n = n;
  P.seq_base = e->rseq_base;
  P.rlog = e->rlog;
  P.st = e->st;
  e->rseq_base += (uint32_t)bound;
  int blocks = std::max(1, std::min((bound + 256 * kReplicaUnroll - 1) / (256 * kReplicaUnroll), e->num_sms * 8));
  replica_chosen_kernel<<<blocks, 256, 0, e->stream>>>(P);
  e->launches++;
  CK(e, cudaGetLastError());
  return FPX_OK;
}

int fpx_replica_chosen_dev(fpx_engine* e, const fpx_chosen* d_in, int32_t n) {
  int c = check_n(e, d_in, n);
  if (c != FPX_OK) return c;
  return replica_launch(e, d_in, n, n);
}

int fpx_replica_chosen_last_dev(fpx_engine* e, const fpx_chosen* d_in) {
  if (!e || (!d_in && e->last_p2b_n > 0)) return FPX_ERR_INVALID_ARG;
  return replica_launch(e, d_in, -1, e->last_p2b_n);
}

int fpx_chosen_watermark_dev(fpx_engine* e, int32_t* d_out) {
  if (!e) return FPX_ERR_INVALID_ARG;
  watermark_scan_kernel<<<e->num_sms * 4, 256, 0, e->stream>>>(e->g, e->rlog, e->st, d_out, e->xch);
  e->launches += 1;
  e->xch_epoch++;
  CK(e, cudaGetLastError());
  return FPX_OK;
}

int fpx_step_dev(fpx_engine* e, const fpx_p2a* d_arm, int32_t n_arm, const fpx_p2a* d_p2a, int32_t n_p2a,
                 fpx_p2b* d_out_p2b, fpx_nack* d_out_nack, const fpx_p2b* d_p2b, int32_t n_p2b, fpx_chosen* d_out_chosen,
                 int32_t* d_watermark, int32_t ring_slot) {
  if (!e) return FPX_ERR_INVALID_ARG;
  cudaEvent_t* ev = nullptr;
  if (ring_slot >= 0) {
    if (e->step_ev.empty()) {   // all or nothing: a failed attempt's events stay with the owner until destroy
      std::vector<cudaEvent_t> ring(kStepRing * 4);
      for (cudaEvent_t& x : ring) CK(e, e->res.event(&x, cudaEventDefault));
      e->step_ev.swap(ring);
    }
    ev = e->step_ev.data() + (size_t)(ring_slot % kStepRing) * 4;
  }
  // The arm batch and the acceptor batch touch disjoint state (proxy-leader rows / vote cells), so their
  // order is free; the acceptors go first so that the rows armed last are still L2-resident when the
  // votes are tallied.  The co-located replica (handleChosen + watermark) rides in the tally kernel.
  // (Running the arm batch inside the acceptor kernel was tried and lost: the rows were cold again
  // for the tally and the acceptor's second pass slowed down.)
  if (ev) CK(e, cudaEventRecord(ev[0], e->stream));
  int c = fpx_acceptor_phase2a_dev(e, d_p2a, n_p2a, d_out_p2b, d_out_nack);
  if (c != FPX_OK) return c;
  if (ev) CK(e, cudaEventRecord(ev[1], e->stream));
  c = fpx_proxyleader_arm_dev(e, d_arm, n_arm);
  if (c != FPX_OK) return c;
  if (ev) CK(e, cudaEventRecord(ev[2], e->stream));
  c = tally_launch(e, d_p2b, n_p2b, d_out_chosen, 1, d_watermark);
  if (c != FPX_OK) return c;
  if (ev) CK(e, cudaEventRecord(ev[3], e->stream));
  return FPX_OK;
}

int fpx_step_kernel_ms(fpx_engine* e, int32_t ring_slot, float* acceptor_ms, float* tally_ms) {
  if (!e || e->step_ev.empty() || ring_slot < 0 || !acceptor_ms || !tally_ms) return FPX_ERR_INVALID_ARG;
  cudaEvent_t* ev = e->step_ev.data() + (size_t)(ring_slot % kStepRing) * 4;
  CK(e, cudaEventSynchronize(ev[3]));
  CK(e, cudaEventElapsedTime(acceptor_ms, ev[0], ev[1]));
  CK(e, cudaEventElapsedTime(tally_ms, ev[2], ev[3]));
  return FPX_OK;
}

// --------------------------------------------------------------------------- asynchronous host step

// A lane is ready once all of its resources exist; the pieces of a failed attempt stay with the owner until
// destroy, and the next fpx_step_submit tries the whole set again.
static int lane_init(fpx_engine* e, fpx_engine::Lane& ln) {
  if (ln.ready) return FPX_OK;
  size_t mb = (size_t)e->cfg.max_batch;
  CudaResources& R = e->res;
  CK(e, R.alloc(&ln.d_p2a, mb * 16)); CK(e, R.alloc(&ln.d_p2b, mb * 16)); CK(e, R.alloc(&ln.d_arm, mb * 16));
  CK(e, R.alloc(&ln.d_out_p2b, mb * 16)); CK(e, R.alloc(&ln.d_out_nack, mb * 8)); CK(e, R.alloc(&ln.d_out_chosen, mb * 8));
  for (cudaEvent_t* ev : {&ln.ev_p2a, &ln.ev_p2b, &ln.ev_acc, &ln.ev_done, &ln.ev_d2h})
    CK(e, R.event(ev, cudaEventDisableTiming));
  CK(e, R.alloc_pinned(&ln.h_st, sizeof(DevStatus)));
  ln.ready = true;
  return FPX_OK;
}

int fpx_step_submit(fpx_engine* e, const fpx_p2a* arm, int32_t n_arm, const fpx_p2a* p2a, int32_t n_p2a,
                    const fpx_p2b* p2b, int32_t n_p2b, fpx_p2b* out_p2b, fpx_nack* out_nack, fpx_chosen* out_chosen) {
  int c = check_n(e, p2a, n_p2a);
  if (c == FPX_OK) c = check_n(e, p2b, n_p2b);
  if (c == FPX_OK && arm != nullptr) c = check_n(e, arm, n_arm);
  if (c != FPX_OK) return c;
  if ((n_p2a > 0 && (!out_p2b || !out_nack)) || (n_p2b > 0 && !out_chosen)) return FPX_ERR_INVALID_ARG;
  if (e->g.protocol == FPX_VANILLA_MENCIUS) return FPX_ERR_UNSUPPORTED;
  if (e->lanes_in_flight >= 2) return FPX_ERR_INVALID_ARG;   // fpx_step_wait first
  CK(e, cudaSetDevice(e->cfg.device));
  fpx_engine::Lane& ln = e->lane[e->lane_head];
  c = lane_init(e, ln);
  if (c != FPX_OK) return c;
  // inputs: copy stream (the lane's previous kernels have finished: its step was waited for)
  if (n_p2a) CK(e, cudaMemcpyAsync(ln.d_p2a, p2a, (size_t)n_p2a * 16, cudaMemcpyHostToDevice, e->h2d_stream));
  if (arm && n_arm) CK(e, cudaMemcpyAsync(ln.d_arm, arm, (size_t)n_arm * 16, cudaMemcpyHostToDevice, e->h2d_stream));
  CK(e, cudaEventRecord(ln.ev_p2a, e->h2d_stream));
  if (n_p2b) CK(e, cudaMemcpyAsync(ln.d_p2b, p2b, (size_t)n_p2b * 16, cudaMemcpyHostToDevice, e->h2d_stream));
  CK(e, cudaEventRecord(ln.ev_p2b, e->h2d_stream));
  // kernels: the engine's stream
  CK(e, cudaStreamWaitEvent(e->stream, ln.ev_p2a, 0));
  c = fpx_acceptor_phase2a_dev(e, (const fpx_p2a*)ln.d_p2a, n_p2a, (fpx_p2b*)ln.d_out_p2b, (fpx_nack*)ln.d_out_nack);
  if (c != FPX_OK) return c;
  CK(e, cudaEventRecord(ln.ev_acc, e->stream));
  c = arm ? fpx_proxyleader_arm_dev(e, (const fpx_p2a*)ln.d_arm, n_arm)
          : fpx_proxyleader_arm_dev(e, (const fpx_p2a*)ln.d_p2a, n_p2a);
  if (c != FPX_OK) return c;
  CK(e, cudaStreamWaitEvent(e->stream, ln.ev_p2b, 0));
  c = tally_launch(e, (const fpx_p2b*)ln.d_p2b, n_p2b, (fpx_chosen*)ln.d_out_chosen, 1, nullptr);
  if (c != FPX_OK) return c;
  CK(e, cudaMemcpyAsync(ln.h_st, e->st, sizeof(DevStatus), cudaMemcpyDeviceToHost, e->stream));
  CK(e, cudaEventRecord(ln.ev_done, e->stream));
  // replies: second copy stream, while the tally runs (dense positions = the stream unless a Nack was produced)
  CK(e, cudaStreamWaitEvent(e->d2h_stream, ln.ev_acc, 0));
  if (n_p2a) CK(e, cudaMemcpyAsync(out_p2b, ln.d_out_p2b, (size_t)n_p2a * 16, cudaMemcpyDeviceToHost, e->d2h_stream));
  CK(e, cudaEventRecord(ln.ev_d2h, e->d2h_stream));
  ln.out_p2b = out_p2b; ln.out_nack = out_nack; ln.out_chosen = out_chosen; ln.n_p2a = n_p2a;
  ln.busy = true;
  e->lane_head ^= 1;
  e->lanes_in_flight++;
  return FPX_OK;
}

int fpx_step_wait(fpx_engine* e, int32_t* n_out_p2b, int32_t* n_out_nack, int32_t* n_out_chosen, int32_t* watermark,
                  int64_t* err_index) {
  if (err_index) *err_index = -1;
  if (!e || e->lanes_in_flight == 0) return FPX_ERR_INVALID_ARG;
  CK(e, cudaSetDevice(e->cfg.device));
  fpx_engine::Lane& ln = e->lane[e->lane_tail];
  CK(e, cudaEventSynchronize(ln.ev_done));
  const DevStatus& st = *ln.h_st;   // copied behind the step's kernels by fpx_step_submit
  int status = FPX_OK;
  const int c = take_error(e, st, e->st, e->stream, false, &status, err_index);
  if (c != FPX_OK) return c;
  if (status == FPX_OK && st.n_chosen > 0)
    CK(e, cudaMemcpyAsync(ln.out_chosen, ln.d_out_chosen, (size_t)st.n_chosen * 8, cudaMemcpyDeviceToHost, e->d2h_stream));
  if (status == FPX_OK && st.n_nack > 0) {   // leader change in this batch: the dense copy is not the stream
    if (st.n_p2b) CK(e, cudaMemcpyAsync(ln.out_p2b, ln.d_out_p2b, (size_t)st.n_p2b * 16, cudaMemcpyDeviceToHost, e->d2h_stream));
    CK(e, cudaMemcpyAsync(ln.out_nack, ln.d_out_nack, (size_t)st.n_nack * 8, cudaMemcpyDeviceToHost, e->d2h_stream));
  }
  CK(e, cudaStreamSynchronize(e->d2h_stream));
  if (n_out_p2b) *n_out_p2b = st.n_p2b;
  if (n_out_nack) *n_out_nack = st.n_nack;
  if (n_out_chosen) *n_out_chosen = st.n_chosen;
  if (watermark) *watermark = st.watermark;
  ln.busy = false;
  e->lane_tail ^= 1;
  e->lanes_in_flight--;
  return status;
}

// --------------------------------------------------------------------------- multi-GPU exchange

static int exchange_push(fpx_engine* e) {
  // the descriptor changes only between steps; epoch is owned by the device once publishing started
  CK(e, cudaSetDevice(e->cfg.device));
  CK(e, cudaStreamSynchronize(e->stream));
  CK(e, cudaMemcpy(&e->h_xch.epoch, &e->xch->epoch, 4, cudaMemcpyDeviceToHost));
  CK(e, cudaMemcpy(e->xch, &e->h_xch, sizeof(DevExchange), cudaMemcpyHostToDevice));
  return FPX_OK;
}

int fpx_exchange_export(fpx_engine* e, void* handle) {
  if (!e || !handle) return FPX_ERR_INVALID_ARG;
  static_assert(sizeof(cudaIpcMemHandle_t) == FPX_EXCHANGE_HANDLE_BYTES, "IPC handle size");
  CK(e, cudaSetDevice(e->cfg.device));
  CK(e, cudaIpcGetMemHandle((cudaIpcMemHandle_t*)handle, e->xch_table));
  return FPX_OK;
}

int fpx_exchange_attach(fpx_engine* e, int32_t shard, const void* handle) {
  if (!e || !handle || shard < 0 || shard >= e->g.shard_count || e->g.shard_count > kMaxShards) return FPX_ERR_INVALID_ARG;
  if (shard == e->g.shard_index) return FPX_OK;
  CK(e, cudaSetDevice(e->cfg.device));
  cudaIpcMemHandle_t h;
  memcpy(&h, handle, sizeof(h));
  void* p = nullptr;
  CK(e, cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
  if (e->xch_opened[shard]) cudaIpcCloseMemHandle(e->xch_opened[shard]);
  e->xch_opened[shard] = p;
  e->h_xch.tabs[shard] = (unsigned long long*)p;
  return exchange_push(e);
}

int fpx_exchange_attach_local(fpx_engine* e, int32_t shard, fpx_engine* peer) {
  if (!e || !peer || shard < 0 || shard >= e->g.shard_count || e->g.shard_count > kMaxShards ||
      peer->g.shard_index != shard || peer->g.shard_count != e->g.shard_count)
    return FPX_ERR_INVALID_ARG;
  if (peer == e) return FPX_OK;
  CK(e, cudaSetDevice(e->cfg.device));
  if (peer->cfg.device != e->cfg.device) {
    int can = 0;
    CK(e, cudaDeviceCanAccessPeer(&can, e->cfg.device, peer->cfg.device));
    if (!can) return FPX_ERR_UNSUPPORTED;
    cudaError_t pe = cudaDeviceEnablePeerAccess(peer->cfg.device, 0);
    if (pe != cudaSuccess && pe != cudaErrorPeerAccessAlreadyEnabled) CK(e, pe);
    (void)cudaGetLastError();
  }
  e->h_xch.tabs[shard] = peer->xch_table;
  return exchange_push(e);
}

uint32_t fpx_exchange_epoch(const fpx_engine* e) { return e ? e->xch_epoch : 0; }

int fpx_global_watermark_dev(fpx_engine* e, uint32_t epoch, int32_t timeout_ms, int32_t* d_out, int32_t* d_frontiers) {
  if (!e || timeout_ms < 0 || e->g.shard_count > kMaxShards) return FPX_ERR_INVALID_ARG;
  global_watermark_kernel<<<1, 32, 0, e->stream>>>(e->xch, e->xch_table, epoch, d_out, d_frontiers, e->st,
                                                   (unsigned long long)timeout_ms * 1000000ull);
  e->launches++;
  CK(e, cudaGetLastError());
  return FPX_OK;
}

int fpx_step_arm_ms(fpx_engine* e, int32_t ring_slot, float* arm_ms) {
  if (!e || e->step_ev.empty() || ring_slot < 0 || !arm_ms) return FPX_ERR_INVALID_ARG;
  cudaEvent_t* ev = e->step_ev.data() + (size_t)(ring_slot % kStepRing) * 4;
  CK(e, cudaEventSynchronize(ev[3]));
  CK(e, cudaEventElapsedTime(arm_ms, ev[1], ev[2]));
  return FPX_OK;
}

int fpx_sync(fpx_engine* e, fpx_sync_result* out) {
  if (!e) return FPX_ERR_INVALID_ARG;
  int status = FPX_OK;
  int64_t idx = -1;
  const int c = read_status(e, e->h_st, e->st, e->stream, &status, &idx);
  if (c != FPX_OK) return c;
  if (out) {
    out->status = status;
    out->reserved = 0;
    out->err_index = idx;
    out->n_p2b = e->h_st->n_p2b;
    out->n_nack = e->h_st->n_nack;
    out->n_chosen = e->h_st->n_chosen;
    out->watermark = e->h_st->watermark;
  }
  return status;
}

// --------------------------------------------------------------------------- host entry points

int fpx_proxyleader_arm(fpx_engine* e, const fpx_p2a* in, int32_t n, int64_t* err_index) {
  if (err_index) *err_index = -1;
  int c = check_n(e, in, n);
  if (c != FPX_OK || n == 0) return c;
  return staged_call(e, in, (size_t)n * 16, err_index, nullptr,
                     [&](void* d) { return fpx_proxyleader_arm_dev(e, (const fpx_p2a*)d, n); });
}

int fpx_acceptor_phase2a(fpx_engine* e, const fpx_p2a* in, int32_t n, fpx_p2b* out_p2b, int32_t* n_p2b,
                         fpx_nack* out_nack, int32_t* n_nack, int64_t* err_index) {
  if (err_index) *err_index = -1;
  if (n_p2b) *n_p2b = 0;
  if (n_nack) *n_nack = 0;
  int c = check_n(e, in, n);
  if (c != FPX_OK || n == 0) return c;
  if (!out_p2b || !out_nack || !n_p2b || !n_nack) return FPX_ERR_INVALID_ARG;
  CK(e, cudaSetDevice(e->cfg.device));
  // A batch may be cut at any index without changing its meaning (each piece is a
  // batch in delivery order), so the call is chunk-pipelined: H2D of chunk c+1 and
  // D2H of chunk c-1's replies overlap the kernel of chunk c on three streams.  The
  // replies of a chunk are copied back from their dense positions, which is where they
  // are as long as no Nack has been produced; otherwise the exact streams are copied
  // again at the end.
  const int32_t chunk = 1 << 19;
  int k = 0;
  for (int32_t off = 0; off < n; off += chunk, ++k) {
    int32_t len = std::min(chunk, n - off);
    cudaEvent_t ev_in = e->ev[(2 * k) % kMaxEvents], ev_k = e->ev[(2 * k + 1) % kMaxEvents];
    CK(e, cudaMemcpyAsync((char*)e->d_in + (size_t)off * 16, in + off, (size_t)len * 16, cudaMemcpyHostToDevice,
                          e->h2d_stream));
    CK(e, cudaEventRecord(ev_in, e->h2d_stream));
    CK(e, cudaStreamWaitEvent(e->stream, ev_in, 0));
    c = acceptor_launch(e, (const fpx_p2a*)e->d_in + off, len, (fpx_p2b*)e->d_out_a, (fpx_nack*)e->d_out_b, off > 0,
                        e->stream);
    if (c != FPX_OK) return c;
    CK(e, cudaEventRecord(ev_k, e->stream));
    CK(e, cudaStreamWaitEvent(e->d2h_stream, ev_k, 0));
    CK(e, cudaMemcpyAsync(out_p2b + off, (char*)e->d_out_a + (size_t)off * 16, (size_t)len * 16, cudaMemcpyDeviceToHost,
                          e->d2h_stream));
  }
  fpx_sync_result r;
  c = fpx_sync(e, &r);
  if (err_index) *err_index = r.err_index;
  CK(e, cudaStreamSynchronize(e->d2h_stream));
  if (c != FPX_OK) return c;
  *n_p2b = r.n_p2b;
  *n_nack = r.n_nack;
  if (r.n_nack) {  // leader change in this batch: the dense copies are not the streams
    if (r.n_p2b) CK(e, cudaMemcpyAsync(out_p2b, e->d_out_a, (size_t)r.n_p2b * 16, cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaMemcpyAsync(out_nack, e->d_out_b, (size_t)r.n_nack * 8, cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaStreamSynchronize(e->stream));
  }
  return FPX_OK;
}

int fpx_proxyleader_phase2b(fpx_engine* e, const fpx_p2b* in, int32_t n, fpx_chosen* out, int32_t* n_out,
                            int64_t* err_index) {
  if (err_index) *err_index = -1;
  if (n_out) *n_out = 0;
  int c = check_n(e, in, n);
  if (c != FPX_OK || n == 0) return c;
  if (!out || !n_out) return FPX_ERR_INVALID_ARG;
  fpx_sync_result r;
  c = staged_call(e, in, (size_t)n * 16, err_index, &r, [&](void* d) {
    return fpx_proxyleader_phase2b_dev(e, (const fpx_p2b*)d, n, (fpx_chosen*)e->d_out_b);
  });
  if (c != FPX_OK) return c;
  *n_out = r.n_chosen;
  if (r.n_chosen) {
    CK(e, cudaMemcpyAsync(out, e->d_out_b, (size_t)r.n_chosen * 8, cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaStreamSynchronize(e->stream));
  }
  return FPX_OK;
}


// --------------------------------------------------------------------------- vanilla Mencius

int fpx_vm_client_request_dev(fpx_engine* e, const fpx_p2a* d_in, int32_t n) {
  if (e && e->g.protocol != FPX_VANILLA_MENCIUS) return FPX_ERR_UNSUPPORTED;
  return arm_launch(e, d_in, n, 1);
}

int fpx_vm_client_request(fpx_engine* e, const fpx_p2a* in, int32_t n, int64_t* err_index) {
  if (err_index) *err_index = -1;
  int c = check_n(e, in, n);
  if (c != FPX_OK || n == 0) return c;
  if (e->g.protocol != FPX_VANILLA_MENCIUS) return FPX_ERR_UNSUPPORTED;
  return staged_call(e, in, (size_t)n * 16, err_index, nullptr,
                     [&](void* d) { return fpx_vm_client_request_dev(e, (const fpx_p2a*)d, n); });
}

// which: 0 handlePhase2a (d_reply dense), 1 handleChosen, 2 handleChosen with isRevocation
static int vm_launch(fpx_engine* e, const void* d_in, int32_t n, fpx_p2b* d_reply, int which) {
  int c = check_n(e, d_in, n);
  if (c != FPX_OK || n == 0) return c;
  if (e->g.protocol != FPX_VANILLA_MENCIUS) return FPX_ERR_UNSUPPORTED;
  if (which == 0 && !d_reply) return FPX_ERR_INVALID_ARG;
  VmParams P;
  P.g = e->g; P.in = (const int4*)d_in; P.out = (int4*)d_reply; P.n = n; P.votes = e->votes;
  P.rows = e->rows; P.st = e->st;
  P.tag = e->vm_tag++;
  if (which == 0) vm_phase2a_kernel<<<std::min((n + 256 * kVmUnroll - 1) / (256 * kVmUnroll), e->num_sms * FPX_VM_CTAS_PER_SM), 256, 0, e->stream>>>(P);
  else if (which == 1) vm_learn_chosen_kernel<false><<<(n + 255) / 256, 256, 0, e->stream>>>(P);
  else vm_learn_chosen_kernel<true><<<(n + 255) / 256, 256, 0, e->stream>>>(P);
  e->launches++;
  CK(e, cudaGetLastError());
  if (e->vm_tag == 0xffffffffu) {
    // Every batch tag has been used: the next call reuses tag 1, and a cell still claimed by the call of that
    // tag one cycle earlier would fail its Phase2a as a second claim of the batch.  Claims only mean something
    // inside one batch: reset them all behind this call's kernel.  Once per 2^32 - 2 calls.
    const size_t cells = (size_t)e->g.local_slots * e->g.voters;
    vm_claim_init_kernel<<<(unsigned)((cells + 255) / 256), 256, 0, e->stream>>>(e->votes, cells);
    e->launches++;
    CK(e, cudaGetLastError());
    e->vm_tag = 1;
  }
  return FPX_OK;
}

int fpx_vm_phase2a_dev(fpx_engine* e, const fpx_p2a* d_in, int32_t n, fpx_p2b* d_reply) {
  return vm_launch(e, d_in, n, d_reply, 0);
}

static int vm_call(fpx_engine* e, const void* in, int32_t n, fpx_p2b* reply, int64_t* err_index, int which) {
  if (err_index) *err_index = -1;
  int c = check_n(e, in, n);
  if (c != FPX_OK || n == 0) return c;
  if (e->g.protocol != FPX_VANILLA_MENCIUS) return FPX_ERR_UNSUPPORTED;
  if (which == 0 && !reply) return FPX_ERR_INVALID_ARG;
  return staged_call(e, in, (size_t)n * 16, err_index, nullptr, [&](void* d) {
    const int rc = vm_launch(e, d, n, (fpx_p2b*)e->d_out_a, which);
    if (rc == FPX_OK && which == 0) CK(e, cudaMemcpyAsync(reply, e->d_out_a, (size_t)n * 16, cudaMemcpyDeviceToHost, e->stream));
    return rc;
  });
}

int fpx_vm_phase2a(fpx_engine* e, const fpx_p2a* in, int32_t n, fpx_p2b* reply, int64_t* err_index) {
  return vm_call(e, in, n, reply, err_index, 0);
}
int fpx_vm_learn_chosen(fpx_engine* e, const fpx_p2b* in, int32_t n, int64_t* err_index) {
  return vm_call(e, in, n, nullptr, err_index, 1);
}
int fpx_vm_choose(fpx_engine* e, const fpx_p2b* in, int32_t n, int64_t* err_index) {
  return vm_call(e, in, n, nullptr, err_index, 2);
}
int fpx_vm_choose_dev(fpx_engine* e, const fpx_p2b* d_in, int32_t n) {
  return vm_launch(e, d_in, n, nullptr, 2);
}

int fpx_vm_step_dev(fpx_engine* e, const fpx_p2a* d_req, int32_t n_req, const fpx_p2a* d_p2a, int32_t n_p2a,
                    fpx_p2b* d_reply, const fpx_p2b* d_p2b, int32_t n_p2b, fpx_chosen* d_out_chosen, int32_t* d_watermark) {
  if (!e) return FPX_ERR_INVALID_ARG;
  if (e->g.protocol != FPX_VANILLA_MENCIUS) return FPX_ERR_UNSUPPORTED;
  // the client requests open the Phase 2 entries the votes of this step are tallied against, so they go first;
  // the Phase2a batch touches the other servers' cells only
  int c = fpx_vm_client_request_dev(e, d_req, n_req);
  if (c != FPX_OK) return c;
  c = vm_launch(e, d_p2a, n_p2a, d_reply, 0);
  if (c != FPX_OK) return c;
  return tally_launch(e, d_p2b, n_p2b, d_out_chosen, 1, d_watermark);
}

#include "fpx_engine_ranges.inc"
#include "fpx_engine_wire.inc"

int fpx_replica_chosen(fpx_engine* e, const fpx_chosen* in, int32_t n, int64_t* err_index) {
  if (err_index) *err_index = -1;
  int c = check_n(e, in, n);
  if (c != FPX_OK || n == 0) return c;
  return staged_call(e, in, (size_t)n * 8, err_index, nullptr,
                     [&](void* d) { return fpx_replica_chosen_dev(e, (const fpx_chosen*)d, n); });
}

int fpx_chosen_watermark(fpx_engine* e, int32_t* out) {
  if (!e || !out) return FPX_ERR_INVALID_ARG;
  CK(e, cudaSetDevice(e->cfg.device));
  int c = fpx_chosen_watermark_dev(e, nullptr);
  if (c != FPX_OK) return c;
  fpx_sync_result r;
  c = fpx_sync(e, &r);
  *out = r.watermark;
  return c;
}

int fpx_global_watermark(fpx_engine* e, uint32_t epoch, int32_t timeout_ms, int32_t* out, int32_t* frontiers) {
  if (!e || !out) return FPX_ERR_INVALID_ARG;
  CK(e, cudaSetDevice(e->cfg.device));
  int c = fpx_global_watermark_dev(e, epoch, timeout_ms, e->xch_out, e->xch_out + 1);
  if (c != FPX_OK) return c;
  fpx_sync_result r;
  c = fpx_sync(e, &r);
  if (c != FPX_OK) return c;
  int32_t host[1 + kMaxShards];
  CK(e, cudaMemcpy(host, e->xch_out, (size_t)(1 + e->g.shard_count) * 4, cudaMemcpyDeviceToHost));
  *out = host[0];
  if (frontiers) memcpy(frontiers, host + 1, (size_t)e->g.shard_count * 4);
  return FPX_OK;
}

int fpx_quorum_eval(fpx_engine* e, int32_t which, const uint32_t* masks, int32_t n, uint8_t* out) {
  if (!e || which < 0 || which > 3 || n < 0 || (n > 0 && (!masks || !out))) return FPX_ERR_INVALID_ARG;
  if (n == 0) return FPX_OK;
  CK(e, cudaSetDevice(e->cfg.device));
  CudaResources tmp(e->cfg.device);   // this call's temporaries
  uint32_t* d_m = nullptr;
  uint8_t* d_o = nullptr;
  CK(e, tmp.alloc(&d_m, (size_t)n * 4));
  CK(e, tmp.alloc(&d_o, (size_t)n));
  CK(e, cudaMemcpyAsync(d_m, masks, (size_t)n * 4, cudaMemcpyHostToDevice, e->stream));
  quorum_eval_kernel<<<(n + 255) / 256, 256, 0, e->stream>>>(e->g, which, d_m, n, d_o);
  e->launches++;
  CK(e, cudaMemcpyAsync(out, d_o, (size_t)n, cudaMemcpyDeviceToHost, e->stream));
  CK(e, cudaStreamSynchronize(e->stream));
  return FPX_OK;
}

int fpx_snapshot_acceptor(fpx_engine* e, int32_t group, int32_t acceptor, int32_t* round,
                          int32_t* max_voted_slot, int32_t first_slot, int32_t n_slots, int32_t* vote_round,
                          int32_t* vote_value) {
  if (!e || group < 0 || group >= e->g.groups || acceptor < 0 || acceptor >= e->g.per_group || n_slots < 0 ||
      (n_slots > 0 && (!vote_round || !vote_value)))
    return FPX_ERR_INVALID_ARG;
  CK(e, cudaSetDevice(e->cfg.device));
  CudaResources tmp(e->cfg.device);
  int key = group * e->g.per_group + acceptor;
  if (round) CK(e, cudaMemcpyAsync(round, e->acc_round + key, 4, cudaMemcpyDeviceToHost, e->stream));
  if (max_voted_slot)
    CK(e, cudaMemcpyAsync(max_voted_slot, e->acc_max_voted + key, 4, cudaMemcpyDeviceToHost, e->stream));
  if (n_slots > 0) {
    int32_t *d_r = nullptr, *d_v = nullptr;
    CK(e, tmp.alloc(&d_r, (size_t)n_slots * 4));
    CK(e, tmp.alloc(&d_v, (size_t)n_slots * 4));
    snapshot_votes_kernel<<<(n_slots + 255) / 256, 256, 0, e->stream>>>(e->g, e->votes, group, acceptor,
                                                                         first_slot, n_slots, d_r, d_v);
    e->launches++;
    CK(e, cudaMemcpyAsync(vote_round, d_r, (size_t)n_slots * 4, cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaMemcpyAsync(vote_value, d_v, (size_t)n_slots * 4, cudaMemcpyDeviceToHost, e->stream));
  }
  CK(e, cudaStreamSynchronize(e->stream));
  return FPX_OK;
}


int fpx_acceptor_phase1a(fpx_engine* e, int32_t group, int32_t acceptor, int32_t round, int32_t* nack_round) {
  if (!e || !nack_round || group < 0 || group >= e->g.groups || acceptor < 0 || acceptor >= e->g.per_group)
    return FPX_ERR_INVALID_ARG;
  if (round < 0 || round > FPX_MAX_ROUND) return FPX_ERR_ROUND_RANGE;
  CK(e, cudaSetDevice(e->cfg.device));
  int key = group * e->g.per_group + acceptor;
  int32_t cur = 0;
  CK(e, cudaMemcpyAsync(&cur, e->acc_round + key, 4, cudaMemcpyDeviceToHost, e->stream));
  CK(e, cudaStreamSynchronize(e->stream));
  if (round < cur) {            // Nack(round = round), Acceptor.scala:156-163
    *nack_round = cur;
    return FPX_OK;
  }
  *nack_round = -1;             // round = phase1a.round (:166)
  CK(e, cudaMemcpyAsync(e->acc_round + key, &round, 4, cudaMemcpyHostToDevice, e->stream));
  CK(e, cudaStreamSynchronize(e->stream));
  return FPX_OK;
}

int fpx_leader_safe_values(fpx_engine* e, uint32_t responders, int32_t first_slot, int32_t n_slots,
                           int32_t* vote_round, int32_t* value_id, int32_t* max_slot) {
  if (!e || n_slots < 0 || (n_slots > 0 && (!vote_round || !value_id)) || !max_slot) return FPX_ERR_INVALID_ARG;
  *max_slot = -1;
  if (n_slots == 0) return FPX_OK;
  CK(e, cudaSetDevice(e->cfg.device));
  CudaResources tmp(e->cfg.device);
  int32_t *d_r = nullptr, *d_v = nullptr, *d_m = nullptr;
  CK(e, tmp.alloc(&d_r, (size_t)n_slots * 4));
  CK(e, tmp.alloc(&d_v, (size_t)n_slots * 4));
  CK(e, tmp.alloc(&d_m, 4));
  CK(e, cudaMemsetAsync(d_m, 0xff, 4, e->stream));
  safe_values_kernel<<<(n_slots + 255) / 256, 256, 0, e->stream>>>(e->g, e->votes, responders, first_slot, n_slots,
                                                                    d_r, d_v, d_m);
  e->launches++;
  CK(e, cudaMemcpyAsync(vote_round, d_r, (size_t)n_slots * 4, cudaMemcpyDeviceToHost, e->stream));
  CK(e, cudaMemcpyAsync(value_id, d_v, (size_t)n_slots * 4, cudaMemcpyDeviceToHost, e->stream));
  CK(e, cudaMemcpyAsync(max_slot, d_m, 4, cudaMemcpyDeviceToHost, e->stream));
  CK(e, cudaStreamSynchronize(e->stream));
  return FPX_OK;
}

int fpx_snapshot_log(fpx_engine* e, int32_t first_slot, int32_t n_slots, int32_t* value_id) {
  if (!e || n_slots < 0 || (n_slots > 0 && !value_id)) return FPX_ERR_INVALID_ARG;
  if (n_slots == 0) return FPX_OK;
  CK(e, cudaSetDevice(e->cfg.device));
  CudaResources tmp(e->cfg.device);
  int32_t* d_v = nullptr;
  CK(e, tmp.alloc(&d_v, (size_t)n_slots * 4));
  snapshot_log_kernel<<<(n_slots + 255) / 256, 256, 0, e->stream>>>(e->g, e->rlog, first_slot, n_slots, d_v);
  e->launches++;
  CK(e, cudaMemcpyAsync(value_id, d_v, (size_t)n_slots * 4, cudaMemcpyDeviceToHost, e->stream));
  CK(e, cudaStreamSynchronize(e->stream));
  return FPX_OK;
}

}  // extern "C"

#include "fpx_engine_epaxos.inc"
#include "fpx_engine_epaxos_wire.inc"
#include "fpx_engine_f4.inc"
#include "fpx_engine_reads.inc"
#include "fpx_engine_wire_reads.inc"
#include "fpx_engine_wire_phase1.inc"
#include "fpx_engine_vm_revoke.inc"
