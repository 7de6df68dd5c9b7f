// fpx_epaxos.cuh -- EPaxos replica hot path (SURVEY 8(a) rows a6-a8).
//   S/epaxos/Replica.scala: handlePreAccept :1159-1289, handlePreAcceptOk :1291-1419,
//   preAcceptingSlowPath :796-813, handleAccept :1421-1512, handleAcceptOk :1514-1565,
//   transitionToPreAcceptPhase :633-729, transitionToAcceptPhase :732-793, commit :815-829.
//   S/epaxos/InstancePrefixSet.scala:121-126 -> S/compact/IntPrefixSet.scala:317-351 (dep-set union).
//
// One thread per message.  Batch contract (checked on the device by a validation pass AHEAD of the
// handler kernels: a violation is FPX_ERR_BATCH_ORDER with the index to split at and nothing of the
// call is applied, never a wrong answer):
//   E1  PreAccept / Accept / lead batches hold at most one message per instance;
//   E2  PreAcceptOk / AcceptOk batches hold at most one message per (instance,
//       replica); a response that REPLACES an earlier one with different content
//       (`responses(replicaIndex) = ok`, :1340) must be alone for its instance.
// Under E1/E2 handlers of different messages only interact through (a) the
// per-instance response count, resolved exactly like the MultiPaxos tally with
// first-delivery stamps, and (b) `largestBallot`, a running max that is only
// read when a Nack is built (resolved by a prefix pass over the batch).
// Dep sets are dense watermark vectors (topKDependencies = 1, Replica.scala:95);
// their union is the elementwise max (IntPrefixSet.addAll's values-empty branch,
// IntPrefixSet.scala:320-321).  General sets go through depset_union_kernel.
#pragma once
#include "fpx_common.cuh"
#include "fpx_scan.cuh"

namespace fpx {

constexpr int kEpMaxN = 8;          // replicas (n = 2f+1 <= 7)
constexpr int kEpCmdWords = 16;     // cmdLog row: 8 header + 8 deps
constexpr int kEpLeadWords = 96;    // leader row: twelve 32-byte sectors, every field group sector-aligned
// cmdLog row words
enum { C_KIND = 0, C_VALUE, C_BORD, C_BREP, C_VBORD, C_VBREP, C_SEQ, C_PAD, C_DEPS = 8 };
enum { EK_NONE = 0, EK_NOCOMMAND = 1, EK_PREACCEPTED = 2, EK_ACCEPTED = 3, EK_COMMITTED = 4 };
// leader row words: header | accept-phase deps | AcceptOk stamps | PreAcceptOk stamps | one 32-byte answer
// {seq, deps[7]} per replica.  A response touches the header sector, one stamp word and one answer sector;
// counting a quorum reads one stamp sector.
// A Preparing row (transitionToPreparePhase, :969-996) keeps its ballot in L_BORD / L_BREP, its PrepareOk
// first-delivery stamps in L_RSTAMP and replica k's PrepareOk {vb_ord, vb_rep, status, value} in sector k of L_RESP.
enum { L_KIND = 0, L_VALUE, L_BORD, L_BREP, L_FLAGS, L_ASEQ, L_PAD0, L_PAD1, L_ADEPS = 8, L_ASTAMP = 16, L_RSTAMP = 24, L_RESP = 32 };
enum { LK_NONE = 0, LK_PREACCEPTING = 1, LK_ACCEPTING = 2, LK_PREPARING = 3 };
constexpr int kEpRespWords = 8;     // {seq, deps[7]} (n <= 7)
enum { LF_AVOID = 1, LF_TIMER = 2 };
enum { REPLY_NONE = 0, REPLY_OK = 1, REPLY_NACK = 2, REPLY_COMMIT = 3 };
enum { EV_NONE = 0, EV_FAST_COMMIT = 1, EV_SLOW_ACCEPT = 2, EV_TIMER = 3, EV_COMMIT = 4 };
enum { EV_RECOVER_TIMER = 1 };                                   // Nack outcome
enum { EV_RESTART = 1 };                                         // PrepareOk outcome
enum { ST_NOT_SEEN = 0, ST_PRE_ACCEPTED = 1, ST_ACCEPTED = 2 };  // CommandStatus (EPaxos.proto:91-95)
// response kinds of the stamp / decide passes
enum { kRespPreAcceptOk = 0, kRespAcceptOk = 1, kRespPrepareOk = 2 };

struct EpGeometry {
  int32_t f, n, index, fast_quorum, slow_quorum;
  int32_t per_replica;   // instance numbers [0, per_replica)
};

struct EpState {
  int32_t* cmd;                    // [n*per_replica][kEpCmdWords]
  int32_t* lead;                   // [n*per_replica][kEpLeadWords]
  // scratch of the validation pass, tagged with the batch tag (a word of another tag is ignored)
  unsigned long long* claim;       // [n*per_replica]  (~batch_tag : min index) over the batch's records of the instance
  unsigned long long* rclaim;      // [n*per_replica][kEpMaxN]  the same per (instance, sender) of a response batch
  uint32_t* refused;               // [0] batch tag of the call the validation pass refused, 0 = none; stays until the
                                   //     status is collected.  [1] batch tag of the last call with a replacing response
  unsigned long long* largest;     // largestBallot as an order-preserving key
  unsigned long long* proc_ballot; // [max_batch] ballot key of record i if it "proceeded", else 0
  int32_t* vflag;                  // [max_batch] validation of a response batch: 0 not counted, 1 counted, 2 replacing
  DevStatus* st;
};

// (ordering, replicaIndex) -> key with tuple order (BallotHelpers.scala:11-21); both >= -1
__device__ __forceinline__ unsigned long long ballot_key(int ord, int rep) {
  return ((unsigned long long)(uint32_t)(ord + 1) << 32) | (uint32_t)(rep + 1);
}
__device__ __forceinline__ void key_ballot(unsigned long long k, int& ord, int& rep) {
  ord = (int)(uint32_t)(k >> 32) - 1;
  rep = (int)(uint32_t)k - 1;
}
__device__ __forceinline__ long long ep_instance(const EpGeometry& g, int rep, int num) {
  if ((uint32_t)rep >= (uint32_t)g.n || (uint32_t)num >= (uint32_t)g.per_replica) return -1;
  return (long long)num * g.n + rep;
}
// min index of this batch per key (instance, or instance and sender); returns the index that held the key
// before this one, -1 if none did
__device__ __forceinline__ long long ep_claim(unsigned long long* word, uint32_t tag, int i) {
  const unsigned long long mine = ((unsigned long long)(~tag) << 32) | (uint32_t)i;
  const unsigned long long old = atomicMin(word, mine);
  return (uint32_t)(old >> 32) == ~tag ? (long long)(uint32_t)old : -1;
}
// A call refused by its validation pass applies nothing: its handler kernels return at entry, and so do the
// kernels of every call queued behind it until the status has been collected (fpx_epaxos_sync).
__device__ __forceinline__ bool ep_refused(const EpState& s) { return __ldcg(s.refused) != 0; }
// the validation kernels of the calls queued behind a refused one return as well: the status is the refused call's
__device__ __forceinline__ bool ep_refused_before(const EpState& s, uint32_t tag) {
  const uint32_t r = __ldcg(s.refused);
  return r != 0 && r != tag;
}
__device__ __forceinline__ void ep_refuse(const EpState& s, uint32_t tag, int code, long long index) {
  report_error(s.st, code, index);
  *(volatile uint32_t*)s.refused = tag;
}

struct EpParams {
  EpGeometry g;
  EpState s;
  const int32_t* in;
  int32_t* out;
  int32_t n_rec;
  uint32_t tag;        // batch tag
  uint32_t seq_base;   // response stamps
};

// A CTA's tile of kEpTile fixed-width int32 rows staged in shared memory with coalesced 128-bit loads; row
// stride Wp = W | 1 words (odd: conflict-free when thread t reads row t).  256 * W * 4 bytes per tile: the
// tile starts 16-byte aligned.
constexpr int kEpTile = 256;
__device__ __forceinline__ void ep_stage_rows(const int32_t* in, long long tile0, int rows, int W, int Wp, int32_t* s_in) {
  const int words = rows * W;
  const int4* src = (const int4*)(in + tile0 * W);
  const uint32_t mW = 0xffffffffu / (uint32_t)W + 1u;           // e / W for e < 2^16
  for (int v = threadIdx.x; v < words / 4; v += kEpTile) {
    const int4 x = ld_stream(src + v);
    const int vals[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const uint32_t e = 4u * v + q, row = __umulhi(e, mW);
      s_in[row * Wp + (e - row * W)] = vals[q];
    }
  }
  for (int e = (words & ~3) + threadIdx.x; e < words; e += kEpTile) s_in[(e / W) * Wp + e % W] = in[tile0 * W + e];
}

// ---- The validation pass: one launch ahead of a call's handler kernels (two for PreAcceptOk / PrepareOk).  It
// reads {rep, num[, ballot, from]} of every row and the state the call starts from, and writes nothing but scratch
// tagged with the batch tag.  What it refuses -- an instance or sender out of range (FPX_ERR_SLOT_RANGE), a
// prepare-phase ballot past FPX_MAX_ROUND (FPX_ERR_ROUND_RANGE), a batch that breaks E1 / E2
// (FPX_ERR_BATCH_ORDER, the later index of the first colliding pair: both halves of a split there are smaller and
// the first is legal) -- is refused whole: no handler kernel of the call runs.
// E1 calls and handleNack (no contract, claims = false): rows of W words.
__global__ void __launch_bounds__(kEpTile) ep_validate_kernel(EpParams P, int W, bool claims, bool prepare_phase) {
  if (ep_refused_before(P.s, P.tag)) return;
  const int i = blockIdx.x * kEpTile + threadIdx.x;
  if (i >= P.n_rec) return;
  const int32_t* r = P.in + (size_t)i * W;
  const long long inst = ep_instance(P.g, r[0], r[1]);
  if (inst < 0) { ep_refuse(P.s, P.tag, FPX_ERR_SLOT_RANGE, i); return; }
  if (prepare_phase) {                                            // row i gets ordering L + 1 + i
    int L, rep;
    key_ballot(max(__ldcg(P.s.largest), ballot_key(0, P.g.index)), L, rep);
    if ((long long)L + 1 + i > FPX_MAX_ROUND) { ep_refuse(P.s, P.tag, FPX_ERR_ROUND_RANGE, i); return; }
  }
  if (claims) {
    const long long other = ep_claim(&P.s.claim[inst], P.tag, i);
    if (other >= 0) ep_refuse(P.s, P.tag, FPX_ERR_BATCH_ORDER, max((long long)i, other));
  }
}

// word w of a fresh leader row (transitionToPreAcceptPhase, :695-724): PreAccepting in the message's ballot, no
// AcceptOk / PreAcceptOk stamps except the leader's own PreAcceptOk, which is "before everything" (:716-724)
__device__ __forceinline__ int32_t ep_lead_word(const EpGeometry& g, const int32_t* r, int w) {
  if (w < L_ADEPS)
    return w == L_KIND ? LK_PREACCEPTING : w == L_VALUE ? r[4] : w == L_BORD ? r[2] : w == L_BREP ? r[3]
         : w == L_FLAGS ? (r[6] ? LF_AVOID : 0) : 0;
  if (w < L_ASTAMP) return 0;
  if (w < L_RSTAMP) return (int32_t)kStampEmpty;
  if (w < L_RESP) return w - L_RSTAMP == g.index ? 0 : (int32_t)kStampEmpty;
  const int k = (w - L_RESP) / kEpRespWords, j = (w - L_RESP) % kEpRespWords;
  if (k != g.index) return 0;
  return j == 0 ? r[5] : (j - 1 < g.n ? r[8 + j - 1] : 0);
}

// ---- transitionToPreAcceptPhase (:633-729).  in row: {rep, num, b_ord, b_rep, value, seq, avoid, pad, deps[n]}
// Thread t judges message t of the tile (cmdLog header as two 128-bit loads, cmdLog row written as four
// 128-bit words); the 384-byte leader rows are then written by whole warps, lane L the 16 bytes at word 4L:
// one fully coalesced store instruction per row instead of ~40 scalar ones.
__global__ void __launch_bounds__(kEpTile) ep_lead_kernel(EpParams P) {
  if (ep_refused(P.s)) return;
  const EpGeometry& g = P.g;
  extern __shared__ int32_t s_ep[];
  __shared__ long long s_inst[kEpTile];
  const int W = 8 + g.n, Wp = W | 1;
  const int tid = threadIdx.x;
  const long long tile0 = (long long)blockIdx.x * kEpTile;
  const int rows = (int)min((long long)kEpTile, P.n_rec - tile0);
  ep_stage_rows(P.in, tile0, rows, W, Wp, s_ep);
  __syncthreads();
  long long armed = -1;
  if (tid < rows) {
    const int32_t* r = s_ep + tid * Wp;
    const int i = (int)tile0 + tid;
    const long long inst = ep_instance(g, r[0], r[1]);
    if (inst >= 0) {                                              // always: the validation pass judged the range
      int4* c4 = (int4*)(P.s.cmd + inst * kEpCmdWords);
      const int4 h0 = __ldcg(c4), h1 = __ldcg(c4 + 1);          // {kind, value, bord, brep} {vbord, vbrep, seq, pad}
      const unsigned long long b = ballot_key(r[2], r[3]);
      const int kind = h0.x;
      bool bad = kind == EK_COMMITTED;                           // logger.fatal :663-667
      if (!bad && kind != EK_NONE) {
        bad = b < ballot_key(h0.z, h0.w);                        // checkLe
        if (!bad && kind != EK_NOCOMMAND) bad = b < ballot_key(h1.x, h1.y);
      }
      if (bad) {
        report_error(P.s.st, FPX_ERR_EPAXOS_STATE, i);
      } else {
        int dd[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) dd[k] = k < g.n ? r[8 + k] : 0;           // :684-693
        __stcg(c4, make_int4(EK_PREACCEPTED, r[4], r[2], r[3]));
        __stcg(c4 + 1, make_int4(r[2], r[3], r[5], 0));
        __stcg(c4 + 2, make_int4(dd[0], dd[1], dd[2], dd[3]));
        __stcg(c4 + 3, make_int4(dd[4], dd[5], dd[6], dd[7]));
        armed = inst;
      }
    }
  }
  s_inst[tid] = armed;
  __syncthreads();
  const int lane = tid & 31, warp = tid >> 5;
  for (int m = 0; m < 32; ++m) {
    const int t = warp * 32 + m;
    const long long inst = s_inst[t];
    if (inst < 0 || lane >= kEpLeadWords / 4) continue;
    const int32_t* r = s_ep + t * Wp;
    const int w = 4 * lane;
    __stcg((int4*)(P.s.lead + inst * kEpLeadWords) + lane,
           make_int4(ep_lead_word(g, r, w), ep_lead_word(g, r, w + 1), ep_lead_word(g, r, w + 2), ep_lead_word(g, r, w + 3)));
  }
}

// ---- handlePreAccept (:1159-1289) / handleAccept (:1421-1512)
// in row preaccept: {rep, num, b_ord, b_rep, value, seq, local_deps[n], msg_deps[n]}
// in row accept:    {rep, num, b_ord, b_rep, value, seq, deps[n]}
// out row: {kind, b_ord, b_rep, seq, deps[n]}
// A CTA takes a tile of 256 messages: the tile's input rows (one contiguous span) are staged in shared
// memory with coalesced 128-bit loads (row stride padded to an odd word count: conflict-free reads), the
// replies are staged the same way and leave with coalesced stores; the cmdLog row is one 64-byte line
// read and written as four 128-bit words; largestBallot is reduced per CTA before it touches memory.
__host__ __device__ __forceinline__ int ep_in_words(const EpGeometry& g, bool accept) { return accept ? 6 + g.n : 6 + 2 * g.n; }

// one atomicMax per CTA of a per-thread ballot key
__device__ __forceinline__ void ep_cta_max(unsigned long long m, unsigned long long* dst) {
  m = cta_reduce<kEpTile>(m, ScanMax());
  if (threadIdx.x == 0 && m) atomicMax(dst, m);
}

template <bool kAccept>
__global__ void __launch_bounds__(kEpTile) ep_acceptor_kernel(EpParams P) {
  if (ep_refused(P.s)) return;
  const EpGeometry& g = P.g;
  extern __shared__ int32_t s_ep[];
  const int W = ep_in_words(g, kAccept), Wp = W | 1;
  const int WO = 4 + g.n;                                       // odd: conflict-free as it is
  int32_t* s_in = s_ep;
  int32_t* s_out = s_ep + kEpTile * Wp;
  const int tid = threadIdx.x;
  const long long tile0 = (long long)blockIdx.x * kEpTile;
  const int rows = (int)min((long long)kEpTile, P.n_rec - tile0);
  {
    const int words = rows * W;
    const int4* src = (const int4*)(P.in + tile0 * W);          // 256 * W * 4 bytes per tile: 16-byte aligned
    const uint32_t mW = 0xffffffffu / (uint32_t)W + 1u;         // e / W for e < 2^16
    for (int v = tid; v < words / 4; v += kEpTile) {
      const int4 x = ld_stream(src + v);
      const int vals[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const uint32_t e = 4u * v + q, row = __umulhi(e, mW);
        s_in[row * Wp + (e - row * W)] = vals[q];
      }
    }
    for (int e = (words & ~3) + tid; e < words; e += kEpTile) s_in[(e / W) * Wp + e % W] = P.in[tile0 * W + e];
  }
  __syncthreads();
  const int i = (int)tile0 + tid;
  unsigned long long proceeded = 0;
  if (tid < rows) {
    const int32_t* r = s_in + tid * Wp;
    int32_t* o = s_out + tid * WO;
    o[0] = REPLY_NONE; o[1] = -1; o[2] = -1; o[3] = 0;
    for (int k = 0; k < g.n; ++k) o[4 + k] = 0;
    const long long inst = ep_instance(g, r[0], r[1]);
    if (inst >= 0) {                                              // always: the validation pass judged the range
      int4* c4 = (int4*)(P.s.cmd + inst * kEpCmdWords);
      const int4 h0 = __ldcg(c4), h1 = __ldcg(c4 + 1);          // {kind, value, bord, brep} {vbord, vbrep, seq, pad}
      const unsigned long long b = ballot_key(r[2], r[3]);
      const int kind = h0.x;
      bool done = false;
      if (kind == EK_COMMITTED) {                               // :1223-1234 / :1466-1477 reply Commit
        const int4 d0 = __ldcg(c4 + 2), d1 = __ldcg(c4 + 3);
        const int dd[8] = {d0.x, d0.y, d0.z, d0.w, d1.x, d1.y, d1.z, d1.w};
        o[0] = REPLY_COMMIT; o[3] = h1.z;
        for (int k = 0; k < g.n; ++k) o[4 + k] = dd[k];
        done = true;
      } else if (kind != EK_NONE) {
        if (b < ballot_key(h0.z, h0.w)) {                       // stale ballot: Nack(largestBallot)
          o[0] = REPLY_NACK;                                    // ballot filled by the fix-up pass
          atomicOr(&P.s.st->ts_flags, 1u);                      // this batch needs the fix-up
          done = true;
        } else {
          const unsigned long long vb = ballot_key(h1.x, h1.y);
          if (!kAccept && kind == EK_PREACCEPTED && b == vb) {  // :1195-1208 re-send the stored answer
            const int4 d0 = __ldcg(c4 + 2), d1 = __ldcg(c4 + 3);
            const int dd[8] = {d0.x, d0.y, d0.z, d0.w, d1.x, d1.y, d1.z, d1.w};
            o[0] = REPLY_OK; o[1] = r[2]; o[2] = r[3]; o[3] = h1.z;
            for (int k = 0; k < g.n; ++k) o[4 + k] = dd[k];
            done = true;
          } else if (!kAccept && kind == EK_ACCEPTED && b == vb) {
            o[1] = r[2]; o[2] = r[3]; done = true;              // :1219-1221 drop
          } else if (kAccept && kind == EK_ACCEPTED && b == vb) {
            o[0] = REPLY_OK; o[1] = r[2]; o[2] = r[3]; done = true;   // :1455-1464 re-send AcceptOk
          }
        }
      }
      if (!done) {
        // yield leadership to a higher ballot (:1240-1244 / :1482-1486)
        int32_t* l = P.s.lead + inst * kEpLeadWords;
        const int4 lh = __ldcg((const int4*)l);                 // {kind, value, bord, brep}
        if (lh.x != LK_NONE && b > ballot_key(lh.z, lh.w)) l[L_KIND] = LK_NONE;
        proceeded = b;                                          // largestBallot = max(..) (:1246 / :1489)
        int seq = r[5];
        int dd[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        o[0] = REPLY_OK; o[1] = r[2]; o[2] = r[3];
        if (!kAccept) {
          seq = max(0, seq);                                    // :1256 (local sequence number is 0, :599)
          for (int k = 0; k < g.n; ++k) {
            dd[k] = max(r[6 + k], r[6 + g.n + k]);              // deps.addAll(msg.deps) (:1257), dense
            o[4 + k] = dd[k];
          }
          o[3] = seq;
        } else {
          for (int k = 0; k < g.n; ++k) dd[k] = r[6 + k];
        }
        __stcg(c4, make_int4(kAccept ? EK_ACCEPTED : EK_PREACCEPTED, r[4], r[2], r[3]));
        __stcg(c4 + 1, make_int4(r[2], r[3], seq, 0));
        __stcg(c4 + 2, make_int4(dd[0], dd[1], dd[2], dd[3]));
        __stcg(c4 + 3, make_int4(dd[4], dd[5], dd[6], dd[7]));
      }
    }
    P.s.proc_ballot[i] = proceeded;
  }
  ep_cta_max(proceeded, P.s.largest + 1);   // largestBallot of the batch (its barrier also publishes s_out)
  // replies: coalesced
  int32_t* dst = P.out + tile0 * WO;
  for (int e = tid; e < rows * WO; e += kEpTile) __stcs(dst + e, s_out[e]);
}

// Nack(instance, largestBallot) carries largestBallot AS OF that delivery (:1166-1167): the max over the
// handle's value at batch start and the ballots of the records that proceeded before it -- an exclusive
// prefix max over the batch.  Three small passes, run only when the batch produced a Nack.  handlePrepare
// raises largestBallot before it builds its Nack (:1637, :1652): there every record contributes and the max is
// inclusive, floored at (0, index) (the reference's initial largestBallot, :458); the ballot goes to columns
// col, col+1 of the reply row.
constexpr int kEpScanTile = 1024;
__global__ void __launch_bounds__(kEpScanTile) ep_nack_tilemax_kernel(EpParams P, unsigned long long* tile_max) {
  if (!(__ldcg(&P.s.st->ts_flags) & 1u)) return;
  const int i = blockIdx.x * kEpScanTile + threadIdx.x;
  const unsigned long long m = cta_reduce<kEpScanTile>(i < P.n_rec ? P.s.proc_ballot[i] : 0ull, ScanMax());
  if (threadIdx.x == 0) tile_max[blockIdx.x] = m;
}
__global__ void __launch_bounds__(kEpScanTile) ep_nack_fixup_kernel(EpParams P, int WO, const unsigned long long* tile_max,
                                                                    int col, bool inclusive, unsigned long long floor) {
  if (!(__ldcg(&P.s.st->ts_flags) & 1u)) return;
  const int tid = threadIdx.x;
  // carry into this tile: largestBallot at batch start and every earlier tile
  unsigned long long c = tid == 0 ? max(P.s.largest[0], floor) : 0ull;
  for (int t = tid; t < (int)blockIdx.x; t += kEpScanTile) c = max(c, tile_max[t]);
  c = cta_reduce<kEpScanTile>(c, ScanMax());
  const int i = blockIdx.x * kEpScanTile + tid;
  const unsigned long long mine = i < P.n_rec ? P.s.proc_ballot[i] : 0ull;
  const unsigned long long excl = max(c, inclusive ? cta_scan<kEpScanTile, false>(mine, ScanMax())
                                                   : cta_scan<kEpScanTile, true>(mine, ScanMax()));
  if (i < P.n_rec) {
    int32_t* o = P.out + (size_t)i * WO;
    if (o[0] == REPLY_NACK) {
      int ord, rep;
      key_ballot(excl, ord, rep);
      o[col] = ord; o[col + 1] = rep;
    }
  }
}
__global__ void ep_largest_commit_kernel(EpState s) {
  // largest[1] accumulated this batch's proceeding ballots; fold into largest[0]
  s.largest[0] = max(s.largest[0], s.largest[1]);
  s.largest[1] = 0;
  s.st->ts_flags = 0;
}

// 32-bit response stamps: before they wrap, every recorded first-delivery stamp collapses to 0 ("before
// everything"), like renormalize_stamps_kernel does for the MultiPaxos rows
__global__ void ep_renormalize_kernel(EpState s, size_t n_inst) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_inst) return;
  int32_t* l = s.lead + i * kEpLeadWords;
  if (l[L_KIND] == LK_NONE) return;
  for (int k = 0; k < kEpMaxN; ++k) {
    if ((uint32_t)l[L_ASTAMP + k] != kStampEmpty) l[L_ASTAMP + k] = 0;
    if ((uint32_t)l[L_RSTAMP + k] != kStampEmpty) l[L_RSTAMP + k] = 0;
  }
}

// ---- handlePreAcceptOk (:1291-1419) / handleAcceptOk (:1514-1565), stamp pass
// in row preacceptok: {rep, num, b_ord, b_rep, from, seq, deps[n]};  acceptok: {rep, num, b_ord, b_rep, from, pad}
// mode[i] (scratch): 0 inactive, 1 first delivery of its replica, 2 replacing response.
// The tile's input rows are staged coalesced; per message: one 128-bit load of the leader header, one atomicMin
// on the replica's stamp word, and the answer {seq, deps} as two 128-bit words (one sector).
__device__ __forceinline__ void ep_load8(const int32_t* p, int (&v)[8]) {
  const int4 a = __ldcg((const int4*)p), b = __ldcg((const int4*)p + 1);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
__device__ __forceinline__ void ep_store8(int32_t* p, const int (&v)[8]) {
  __stcg((int4*)p, make_int4(v[0], v[1], v[2], v[3]));
  __stcg((int4*)p + 1, make_int4(v[4], v[5], v[6], v[7]));
}
// the answer {seq, deps[n], 0...} carried by PreAcceptOk row r; {vb_ord, vb_rep, status, value, 0...} by
// PrepareOk row r
template <int kWhich>
__device__ __forceinline__ void ep_answer_of(const EpGeometry& g, const int32_t* r, int (&v)[8]) {
  if (kWhich == kRespPrepareOk) {
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = k < 4 ? r[5 + k] : 0;
    return;
  }
  v[0] = r[5];
#pragma unroll
  for (int k = 0; k < 7; ++k) v[1 + k] = k < g.n ? r[6 + k] : 0;
}
// in-row words of the response handlers: PreAcceptOk 6+n, AcceptOk 6, PrepareOk 9
template <int kWhich>
__host__ __device__ __forceinline__ int ep_resp_in_words(const EpGeometry& g) {
  return kWhich == kRespAcceptOk ? 6 : kWhich == kRespPrepareOk ? 9 : 6 + g.n;
}

// Validation of a response batch (E2).  Only a response the handler would count takes part: the row leads the
// instance in the phase the response belongs to, in the response's ballot -- judged on the state the call starts
// from, which is what the stamp pass sees.  First launch: at most one such response per (instance, sender); vflag[i]
// = 1 counted, 2 counted and REPLACING (its sender's answer is already stored, with other content); the smallest
// counted index per instance goes to `claim`.  Second launch, once every claim is in (a grid-wide order: it cannot
// be the same launch): a replacing response must be the only counted one of its instance.  The pairs are
// (replacing, any other counted) -- with m the instance's smallest counted index, a replacing record i > m reports
// i, and when the replacing record IS m every other counted record reports itself: the minimum is the pair's
// later index either way.
template <int kWhich>
__global__ void __launch_bounds__(kEpTile) ep_validate_responses_kernel(EpParams P) {
  constexpr bool kAccept = kWhich == kRespAcceptOk, kPrepare = kWhich == kRespPrepareOk;
  if (ep_refused_before(P.s, P.tag)) return;
  const EpGeometry& g = P.g;
  const int i = blockIdx.x * kEpTile + threadIdx.x;
  if (i >= P.n_rec) return;
  const int32_t* r = P.in + (size_t)i * ep_resp_in_words<kWhich>(g);
  int flag = 0;
  const long long inst = ep_instance(g, r[0], r[1]);
  const int from = r[4];
  if (inst < 0 || (uint32_t)from >= (uint32_t)g.n) {
    ep_refuse(P.s, P.tag, FPX_ERR_SLOT_RANGE, i);
  } else {
    const int32_t* l = P.s.lead + inst * kEpLeadWords;
    const int4 h = __ldcg((const int4*)l);                                      // {kind, value, bord, brep}
    const bool leading = h.x == (kAccept ? LK_ACCEPTING : kPrepare ? LK_PREPARING : LK_PREACCEPTING);
    if (leading && ballot_key(r[2], r[3]) == ballot_key(h.z, h.w)) {
      flag = 1;
      ep_claim(&P.s.claim[inst], P.tag, i);
      const long long other = ep_claim(&P.s.rclaim[inst * kEpMaxN + from], P.tag, i);
      if (other >= 0) {
        ep_refuse(P.s, P.tag, FPX_ERR_BATCH_ORDER, max((long long)i, other));
      } else if (!kAccept && (uint32_t)__ldcg(&l[L_RSTAMP + from]) != kStampEmpty) {
        int v[8], have[8];
        ep_answer_of<kWhich>(g, r, v);
        ep_load8(l + L_RESP + from * kEpRespWords, have);
        bool same = true;
#pragma unroll
        for (int k = 0; k < 8; ++k) same = same && (k > g.n || have[k] == v[k]);
        if (!same) {
          flag = 2;
          *(volatile uint32_t*)(P.s.refused + 1) = P.tag;                       // the second launch has work
        }
      }
    }
  }
  P.s.vflag[i] = flag;
}
__global__ void __launch_bounds__(kEpTile) ep_validate_replace_kernel(EpParams P, int W) {
  if (__ldcg(P.s.refused + 1) != P.tag || ep_refused_before(P.s, P.tag)) return;
  const int i = blockIdx.x * kEpTile + threadIdx.x;
  if (i >= P.n_rec) return;
  const int flag = __ldcg(P.s.vflag + i);
  if (flag == 0) return;
  const int32_t* r = P.in + (size_t)i * W;
  const long long inst = ep_instance(P.g, r[0], r[1]);
  const uint32_t m = (uint32_t)__ldcg(&P.s.claim[inst]);                        // of this batch: record i claimed too
  if (m != (uint32_t)i && (flag == 2 || __ldcg(P.s.vflag + m) == 2)) ep_refuse(P.s, P.tag, FPX_ERR_BATCH_ORDER, i);
}

// the leader kinds the three response handlers count for: PreAcceptOk (:1295-1315), AcceptOk (:1518-1535),
// PrepareOk (:1763-1784)
template <int kWhich>
__global__ void __launch_bounds__(kEpTile) ep_response_stamp_kernel(EpParams P, int32_t* mode) {
  if (ep_refused(P.s)) return;
  constexpr bool kAccept = kWhich == kRespAcceptOk, kPrepare = kWhich == kRespPrepareOk;
  const EpGeometry& g = P.g;
  extern __shared__ int32_t s_ep[];
  const int W = ep_resp_in_words<kWhich>(g), Wp = W | 1;
  const int tid = threadIdx.x;
  const long long tile0 = (long long)blockIdx.x * kEpTile;
  const int rows = (int)min((long long)kEpTile, P.n_rec - tile0);
  ep_stage_rows(P.in, tile0, rows, W, Wp, s_ep);
  __syncthreads();
  if (tid >= rows) return;
  const int i = (int)tile0 + tid;
  const int32_t* r = s_ep + tid * Wp;
  int md = 0;
  const long long inst = ep_instance(g, r[0], r[1]);
  if (inst >= 0 && (uint32_t)r[4] < (uint32_t)g.n) {               // always: the validation pass judged the range
    int32_t* l = P.s.lead + inst * kEpLeadWords;
    const int4 h = __ldcg((const int4*)l);                                      // {kind, value, bord, brep}
    const bool leading = h.x == (kAccept ? LK_ACCEPTING : kPrepare ? LK_PREPARING : LK_PREACCEPTING);
    if (kPrepare && leading && ballot_key(r[2], r[3]) > ballot_key(h.z, h.w))
      report_error(P.s.st, FPX_ERR_CHECK_FAILED, i);                            // logger.checkLt (:1792)
    if (leading && ballot_key(r[2], r[3]) == ballot_key(h.z, h.w)) {            // :1325-1335 / :1543-1552 / :1785
      const uint32_t seq = P.seq_base + (uint32_t)i;
      const uint32_t old = atomicMin((uint32_t*)&l[(kAccept ? L_ASTAMP : L_RSTAMP) + r[4]], seq);
      if (old == kStampEmpty) {                                 // responses(replicaIndex) = ok (:1340 / :1796), new key
        md = 1;
        if (!kAccept) {
          int v[8];
          ep_answer_of<kWhich>(g, r, v);
          ep_store8(l + L_RESP + r[4] * kEpRespWords, v);
        }
      } else if (!kAccept && old < P.seq_base) {                // (a stamp of this batch: excluded by E2)
        int v[8], have[8];
        ep_answer_of<kWhich>(g, r, v);
        ep_load8(l + L_RESP + r[4] * kEpRespWords, have);
        bool same = true;
#pragma unroll
        for (int k = 0; k < 8; ++k) same = same && (k > g.n || have[k] == v[k]);
        if (!same) md = 2;                                      // replaces content; judged in the decide pass
      }
    }
  }
  mode[i] = md;
}

// preAcceptingSlowPath (:796-813) over the answers in[a] of leader row l, then transitionToAcceptPhase
// (:732-793): event {EV_SLOW_ACCEPT, seq, deps[n]} into o, cmdLog row c Accepted, l Accepting with only the
// leader's own AcceptOk.  h0 = the leader header {kind, value, bord, brep}.
__device__ __forceinline__ void ep_slow_path(const EpGeometry& g, int32_t* l, int32_t* c, const int4& h0,
                                             const int (&ans)[kEpMaxN - 1][8], const bool (&in)[kEpMaxN - 1], int32_t* o) {
  int sseq = INT_MIN;
  int sdeps[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
  for (int a = 0; a < kEpMaxN - 1; ++a) {
    if (!in[a]) continue;
    sseq = max(sseq, ans[a][0]);
#pragma unroll
    for (int k = 0; k < 7; ++k) if (k < g.n) sdeps[k] = max(sdeps[k], ans[a][1 + k]);   // dependencies.addAll (:804-807)
  }
  o[0] = EV_SLOW_ACCEPT; o[1] = sseq;
#pragma unroll
  for (int k = 0; k < 7; ++k) if (k < g.n) o[2 + k] = sdeps[k];
  // transitionToAcceptPhase (:732-793)
  __stcg((int4*)c, make_int4(EK_ACCEPTED, h0.y, h0.z, h0.w));
  __stcg((int4*)c + 1, make_int4(h0.z, h0.w, sseq, 0));
  ep_store8(c + C_DEPS, sdeps);
  l[L_ASEQ] = sseq;
  ep_store8(l + L_ADEPS, sdeps);
  int as[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) as[k] = k == g.index ? 0 : (int)kStampEmpty;   // own AcceptOk (:781-789)
  ep_store8(l + L_ASTAMP, as);
  l[L_KIND] = LK_ACCEPTING;
}

// out-row words of the response handlers: events {kind, seq, deps[n]}, PrepareOk {kind, b_ord, b_rep, value}
template <int kWhich>
__host__ __device__ __forceinline__ int ep_resp_out_words(const EpGeometry& g) {
  return kWhich == kRespPrepareOk ? 4 : 2 + g.n;
}

// handlePrepareOk's decision (:1804-1867) over the PrepareOks in[a] {vb_ord, vb_rep, status, value}: the
// maximum vote ballot, then the first PreAccepted response of that ballot -- lowest replica index first --
// or Noop.  The two branches before it cannot be taken in the reference and are not taken here: the
// `status == Some(Accepted)` test (:1813) compares an enum with an Option, and the fast-path candidates
// (:1836) require p.ballot == Ballot(0, _) while p.ballot is the Preparing ballot, of ordering >= 1.
__device__ __forceinline__ int ep_prepare_decide(const EpGeometry& g, const int (&ans)[kEpMaxN - 1][8],
                                                 const bool (&in)[kEpMaxN - 1]) {
  unsigned long long vmax = 0;
#pragma unroll
  for (int a = 0; a < kEpMaxN - 1; ++a)
    if (in[a]) vmax = max(vmax, ballot_key(ans[a][0], ans[a][1]));
  int value = FPX_VALUE_NOOP;
  bool found = false;
#pragma unroll
  for (int a = 0; a < kEpMaxN - 1; ++a) {
    if (found || !in[a] || ballot_key(ans[a][0], ans[a][1]) != vmax || ans[a][2] != ST_PRE_ACCEPTED) continue;
    value = ans[a][3];
    found = true;
  }
  return value;
}

// decide pass: events at the first crossing of the quorum thresholds.  out row: {event, seq, deps[n]} (PrepareOk:
// {kind, b_ord, b_rep, value}), staged in shared memory and stored coalesced.
template <int kWhich>
__global__ void __launch_bounds__(kEpTile) ep_response_decide_kernel(EpParams P, const int32_t* mode) {
  if (ep_refused(P.s)) return;
  constexpr bool kAccept = kWhich == kRespAcceptOk, kPrepare = kWhich == kRespPrepareOk;
  const EpGeometry& g = P.g;
  extern __shared__ int32_t s_ep[];
  const int W = ep_resp_in_words<kWhich>(g), Wp = W | 1;
  const int WO = ep_resp_out_words<kWhich>(g);                  // odd for events: conflict-free as it is
  int32_t* s_out = s_ep + kEpTile * Wp;
  const int tid = threadIdx.x;
  const long long tile0 = (long long)blockIdx.x * kEpTile;
  const int rows = (int)min((long long)kEpTile, P.n_rec - tile0);
  ep_stage_rows(P.in, tile0, rows, W, Wp, s_ep);
  __syncthreads();
  if (tid < rows) {
    const int i = (int)tile0 + tid;
    const int32_t* r = s_ep + tid * Wp;
    int32_t* o = s_out + tid * WO;
    for (int k = 0; k < WO; ++k) o[k] = 0;                      // o[0] = EV_NONE
    const int md = __ldcg(mode + i);
    if (md != 0) {
      const long long inst = ep_instance(g, r[0], r[1]);
      int32_t* l = P.s.lead + inst * kEpLeadWords;
      int32_t* c = P.s.cmd + inst * kEpCmdWords;
      const uint32_t seq = P.seq_base + (uint32_t)i;
      if (md == 2) {
        // a replacing response is alone for its instance in the batch (E2, judged by the validation pass): no
        // decision of this batch reads the answer it replaces; size unchanged: no threshold can be crossed
        int v[8];
        ep_answer_of<kWhich>(g, r, v);
        ep_store8(l + L_RESP + r[4] * kEpRespWords, v);
      } else {
        int st[8];
        ep_load8(l + (kAccept ? L_ASTAMP : L_RSTAMP), st);
        int before = 0;
#pragma unroll
        for (int k = 0; k < 8; ++k) before += (k < g.n && (uint32_t)st[k] < seq);
        const int after = before + 1;
        const int4 h0 = __ldcg((const int4*)l);                 // {kind, value, bord, brep}
        if (kPrepare) {
          if (before < g.slow_quorum && after >= g.slow_quorum) {                 // :1800-1802
            int ans[kEpMaxN - 1][8];
            bool in[kEpMaxN - 1];
#pragma unroll
            for (int a = 0; a < kEpMaxN - 1; ++a) {
              in[a] = a < g.n && (uint32_t)st[a] <= seq;
              if (in[a]) ep_load8(l + L_RESP + a * kEpRespWords, ans[a]);
            }
            // transitionToPreAcceptPhase(instance, ballot, value, avoidFastPath = true) (:1856-1867) is the
            // caller's fpx_epaxos_lead; until then the row leads nothing
            o[0] = EV_RESTART; o[1] = h0.z; o[2] = h0.w; o[3] = ep_prepare_decide(g, ans, in);
            l[L_KIND] = LK_NONE;
          }
        } else if (kAccept) {
          if (before < g.slow_quorum && after >= g.slow_quorum) {                 // :1558-1560
            int ad[8];
            ep_load8(l + L_ADEPS, ad);
            const int aseq = __ldcg(&l[L_ASEQ]);
            o[0] = EV_COMMIT; o[1] = aseq;
            #pragma unroll
            for (int k = 0; k < 7; ++k) if (k < g.n) o[2 + k] = ad[k];
            c[C_KIND] = EK_COMMITTED; c[C_VALUE] = h0.y; c[C_SEQ] = aseq;        // commit (:815-829)
#pragma unroll
            for (int k = 0; k < 8; ++k) if (k >= g.n) ad[k] = 0;
            ep_store8(c + C_DEPS, ad);
            l[L_KIND] = LK_NONE;
          }
        } else if (after >= g.slow_quorum) {                                      // :1345-1347
          const bool avoid = __ldcg(&l[L_FLAGS]) & LF_AVOID;
          bool slow = false, decide = false;
          if (!avoid && before < g.slow_quorum && g.slow_quorum < g.fast_quorum) {
            atomicOr((int*)&l[L_FLAGS], LF_TIMER);                               // :1353-1364
            o[0] = EV_TIMER;
          } else if (avoid) {
            slow = before < g.slow_quorum;                                       // :1369-1372
          } else {
            decide = after >= g.fast_quorum && before < g.fast_quorum;           // :1376
          }
          if (slow || decide) {
            // the answers delivered up to this one: {seq, deps} of every replica whose stamp is <= seq
            int ans[kEpMaxN - 1][8];
            bool in[kEpMaxN - 1];
#pragma unroll
            for (int a = 0; a < kEpMaxN - 1; ++a) {
              in[a] = a < g.n && (uint32_t)st[a] <= seq;
              if (in[a]) ep_load8(l + L_RESP + a * kEpRespWords, ans[a]);
            }
            int fseq = 0, fdeps[8] = {0, 0, 0, 0, 0, 0, 0, 0};
            bool fast = false;
            if (decide) {
              // popularItems over the non-leader (seq, deps) pairs, threshold fastQuorumSize - 1 (:1382-1396)
#pragma unroll
              for (int a = 0; a < kEpMaxN - 1; ++a) {
                if (fast || !in[a] || a == g.index) continue;
                int cnt = 0;
#pragma unroll
                for (int b2 = 0; b2 < kEpMaxN - 1; ++b2) {
                  if (!in[b2] || b2 == g.index) continue;
                  bool eq = true;
#pragma unroll
                  for (int k = 0; k < 8; ++k) eq = eq && (k > g.n || ans[a][k] == ans[b2][k]);
                  cnt += eq;
                }
                if (cnt >= g.fast_quorum - 1) {
                  fast = true; fseq = ans[a][0];
#pragma unroll
                  for (int k = 0; k < 7; ++k) fdeps[k] = k < g.n ? ans[a][1 + k] : 0;
                }
              }
              if (!fast) slow = true;
            }
            if (fast) {                                                          // :1401-1410 commit
              o[0] = EV_FAST_COMMIT; o[1] = fseq;
              #pragma unroll
              for (int k = 0; k < 7; ++k) if (k < g.n) o[2 + k] = fdeps[k];
              c[C_KIND] = EK_COMMITTED; c[C_VALUE] = h0.y; c[C_SEQ] = fseq;
              ep_store8(c + C_DEPS, fdeps);
              l[L_KIND] = LK_NONE;
            } else if (slow) {                                                   // preAcceptingSlowPath :796-813
              ep_slow_path(g, l, c, h0, ans, in, o);
            }
          }
        }
      }
    }
  }
  __syncthreads();
  int32_t* dst = P.out + tile0 * WO;
  for (int e = tid; e < rows * WO; e += kEpTile) __stcs(dst + e, s_out[e]);
}

// =========================================================================== recovery and the control path
// Reply rows staged in shared memory with an odd row stride WOp (conflict-free when thread t writes row t) leave
// as one coalesced span of rows * WO words.
__device__ __forceinline__ void ep_store_rows(int32_t* dst, const int32_t* s_out, int rows, int WO, int WOp) {
  for (int e = threadIdx.x; e < rows * WO; e += kEpTile) {
    const int row = e / WO;
    __stcs(dst + e, s_out[row * WOp + (e - row * WO)]);
  }
}

// ---- handleCommit (:1567-1575) -> commit (:815-831).  in row: {rep, num, value, seq, deps[n]}; no reply.
// CommittedEntry(triple) whatever the entry held (:826-827) and no leader state of any kind (:831).
__global__ void __launch_bounds__(kEpTile) ep_commit_kernel(EpParams P) {
  if (ep_refused(P.s)) return;
  const EpGeometry& g = P.g;
  extern __shared__ int32_t s_ep[];
  const int W = 4 + g.n, Wp = W | 1;
  const int tid = threadIdx.x;
  const long long tile0 = (long long)blockIdx.x * kEpTile;
  const int rows = (int)min((long long)kEpTile, P.n_rec - tile0);
  ep_stage_rows(P.in, tile0, rows, W, Wp, s_ep);
  __syncthreads();
  if (tid >= rows) return;
  const int32_t* r = s_ep + tid * Wp;
  const long long inst = ep_instance(g, r[0], r[1]);
  if (inst >= 0) {                                              // always: the validation pass judged the range
    int dd[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) dd[k] = k < g.n ? r[4 + k] : 0;
    int4* c4 = (int4*)(P.s.cmd + inst * kEpCmdWords);
    __stcg(c4, make_int4(EK_COMMITTED, r[2], -1, -1));
    __stcg(c4 + 1, make_int4(-1, -1, r[3], 0));
    __stcg(c4 + 2, make_int4(dd[0], dd[1], dd[2], dd[3]));
    __stcg(c4 + 3, make_int4(dd[4], dd[5], dd[6], dd[7]));
    P.s.lead[inst * kEpLeadWords + L_KIND] = LK_NONE;
  }
}

// ---- handleNack (:1577-1630).  in row: {rep, num, lb_ord, lb_rep}; out row: {kind}.  Every Nack raises
// largestBallot (:1578; a max, so the batch order does not matter); RECOVER_TIMER when a leader state of any kind
// has a ballot below the Nack's (:1580-1618), i.e. the caller (re)arms the recoverInstance timer (:1623-1629).
__global__ void __launch_bounds__(kEpTile) ep_nack_kernel(EpParams P) {
  if (ep_refused(P.s)) return;
  const EpGeometry& g = P.g;
  extern __shared__ int32_t s_ep[];
  const int W = 4, Wp = W | 1;
  const int tid = threadIdx.x;
  const long long tile0 = (long long)blockIdx.x * kEpTile;
  const int rows = (int)min((long long)kEpTile, P.n_rec - tile0);
  ep_stage_rows(P.in, tile0, rows, W, Wp, s_ep);
  __syncthreads();
  unsigned long long seen = 0;
  if (tid < rows) {
    const int i = (int)tile0 + tid;
    const int32_t* r = s_ep + tid * Wp;
    int kind = EV_NONE;
    const long long inst = ep_instance(g, r[0], r[1]);
    if (inst >= 0) {                                              // always: the validation pass judged the range
      seen = ballot_key(r[2], r[3]);
      const int4 lh = __ldcg((const int4*)(P.s.lead + inst * kEpLeadWords));   // {kind, value, bord, brep}
      if (lh.x != LK_NONE && ballot_key(lh.z, lh.w) < seen) kind = EV_RECOVER_TIMER;
    }
    __stcs(P.out + i, kind);
  }
  ep_cta_max(seen, P.s.largest);
}

// ---- transitionToPreparePhase (:969-996).  in row: {rep, num}; out row: {b_ord, b_rep}, the ballot of the
// Prepare to send.  largestBallot is read floored at (0, index) (its initial value in the reference, :458): row i
// gets (L + 1 + i, index), L the floored ordering at call start, and each transition raises largestBallot in
// turn (:976).  The row's leader state becomes Preparing in that ballot with no responses (the replica's own
// PrepareOk arrives as a message, :985); cmdLog is not touched.
__global__ void __launch_bounds__(kEpTile) ep_prepare_phase_kernel(EpParams P) {
  if (ep_refused(P.s)) return;
  const EpGeometry& g = P.g;
  const int i = blockIdx.x * kEpTile + threadIdx.x;
  int L, rep;
  key_ballot(max(__ldcg(P.s.largest), ballot_key(0, g.index)), L, rep);
  unsigned long long seen = 0;
  if (i < P.n_rec) {
    const int2 r = __ldcs((const int2*)P.in + i);
    const long long ord = (long long)L + 1 + i;
    int2 out = make_int2(-1, -1);
    const long long inst = ep_instance(g, r.x, r.y);
    if (inst >= 0 && ord <= FPX_MAX_ROUND) {                      // always: the validation pass judged both
      int4* l4 = (int4*)(P.s.lead + inst * kEpLeadWords);
      const int4 empty = make_int4((int)kStampEmpty, (int)kStampEmpty, (int)kStampEmpty, (int)kStampEmpty);
      __stcg(l4, make_int4(LK_PREPARING, 0, (int)ord, g.index));
      __stcg(l4 + 1, make_int4(0, 0, 0, 0));
      __stcg(l4 + L_ASTAMP / 4, empty); __stcg(l4 + L_ASTAMP / 4 + 1, empty);
      __stcg(l4 + L_RSTAMP / 4, empty); __stcg(l4 + L_RSTAMP / 4 + 1, empty);
      out = make_int2((int)ord, g.index);
      seen = ballot_key((int)ord, g.index);
    }
    __stcs((int2*)P.out + i, out);
  }
  ep_cta_max(seen, P.s.largest + 1);
}

// ---- handlePrepare (:1632-1757).  in row: {rep, num, b_ord, b_rep}
// out row: {kind, yielded, b_ord, b_rep, vb_ord, vb_rep, status, value, seq, deps[n]} -- PrepareOk (kind OK,
// b = the Prepare's ballot), Nack (kind NACK, b = largestBallot, filled by the fix-up pass), Commit (kind COMMIT,
// the triple).  Fields a reply does not carry are (-1, -1) ballots and zeros.
__global__ void __launch_bounds__(kEpTile) ep_prepare_kernel(EpParams P) {
  if (ep_refused(P.s)) return;
  const EpGeometry& g = P.g;
  extern __shared__ int32_t s_ep[];
  const int W = 4, Wp = W | 1, WO = 9 + g.n, WOp = WO | 1;
  int32_t* s_out = s_ep + kEpTile * Wp;
  const int tid = threadIdx.x;
  const long long tile0 = (long long)blockIdx.x * kEpTile;
  const int rows = (int)min((long long)kEpTile, P.n_rec - tile0);
  ep_stage_rows(P.in, tile0, rows, W, Wp, s_ep);
  __syncthreads();
  unsigned long long seen = 0;
  if (tid < rows) {
    const int i = (int)tile0 + tid;
    const int32_t* r = s_ep + tid * Wp;
    int32_t* o = s_out + tid * WOp;
    o[0] = REPLY_NONE; o[1] = 0; o[2] = -1; o[3] = -1; o[4] = -1; o[5] = -1; o[6] = ST_NOT_SEEN; o[7] = 0; o[8] = 0;
    for (int k = 0; k < g.n; ++k) o[9 + k] = 0;
    const long long inst = ep_instance(g, r[0], r[1]);
    if (inst >= 0) {                                              // always: the validation pass judged the range
      const unsigned long long b = ballot_key(r[2], r[3]);
      seen = b;                                                 // largestBallot = max(.., prepare.ballot) (:1637)
      int32_t* l = P.s.lead + inst * kEpLeadWords;
      const int4 lh = __ldcg((const int4*)l);                   // {kind, value, bord, brep}
      if (lh.x != LK_NONE && b > ballot_key(lh.z, lh.w)) {      // yield, before the stale check (:1645-1649)
        l[L_KIND] = LK_NONE;
        o[1] = 1;
      }
      int4* c4 = (int4*)(P.s.cmd + inst * kEpCmdWords);
      const int4 h0 = __ldcg(c4), h1 = __ldcg(c4 + 1);          // {kind, value, bord, brep} {vbord, vbrep, seq, pad}
      const int kind = h0.x;
      if (kind == EK_COMMITTED || kind == EK_PREACCEPTED || kind == EK_ACCEPTED) {
        const int4 d0 = __ldcg(c4 + 2), d1 = __ldcg(c4 + 3);
        const int dd[8] = {d0.x, d0.y, d0.z, d0.w, d1.x, d1.y, d1.z, d1.w};
        for (int k = 0; k < g.n; ++k) o[9 + k] = dd[k];
        o[7] = h0.y; o[8] = h1.z;
      }
      if (kind == EK_COMMITTED) {                               // :1746-1755 reply Commit(triple)
        o[0] = REPLY_COMMIT;
      } else if (kind != EK_NONE && b < ballot_key(h0.z, h0.w)) {   // :1676-1679 / :1700-1703 / :1724-1727
        o[0] = REPLY_NACK;
        o[7] = 0; o[8] = 0;
        for (int k = 0; k < g.n; ++k) o[9 + k] = 0;
        atomicOr(&P.s.st->ts_flags, 1u);                        // this batch needs the fix-up
      } else {
        o[0] = REPLY_OK; o[2] = r[2]; o[3] = r[3];
        if (kind == EK_PREACCEPTED || kind == EK_ACCEPTED) {    // :1705-1720 / :1729-1744
          o[4] = h1.x; o[5] = h1.y; o[6] = kind == EK_PREACCEPTED ? ST_PRE_ACCEPTED : ST_ACCEPTED;
          __stcg(c4, make_int4(kind, h0.y, r[2], r[3]));        // entry.copy(ballot = prepare.ballot)
        } else {                                                // NoCommandEntry(prepare.ballot) (:1669 / :1696)
          __stcg(c4, make_int4(EK_NOCOMMAND, 0, r[2], r[3]));
          __stcg(c4 + 1, make_int4(-1, -1, 0, 0));
          __stcg(c4 + 2, make_int4(0, 0, 0, 0));
          __stcg(c4 + 3, make_int4(0, 0, 0, 0));
        }
      }
    }
    P.s.proc_ballot[i] = seen;
  }
  ep_cta_max(seen, P.s.largest + 1);
  __syncthreads();
  ep_store_rows(P.out + tile0 * WO, s_out, rows, WO, WOp);
}

// ---- the defaultToSlowPath timer (:1015-1036) -> preAcceptingSlowPath (:796-813).  in row: {rep, num, b_ord,
// b_rep}; out row as PreAcceptOk events {kind, seq, deps[n]}.  Only a row still PreAccepting in that ballot with
// the timer armed (LF_TIMER, set where EV_TIMER was emitted) takes the slow path, over every answer it holds; in
// any other state the reference's stopTimers (:618-630) has cancelled the timer and the event is NONE.
__global__ void __launch_bounds__(kEpTile) ep_slow_path_timer_kernel(EpParams P) {
  if (ep_refused(P.s)) return;
  const EpGeometry& g = P.g;
  extern __shared__ int32_t s_ep[];
  const int W = 4, Wp = W | 1, WO = 2 + g.n;                    // odd: conflict-free as it is
  int32_t* s_out = s_ep + kEpTile * Wp;
  const int tid = threadIdx.x;
  const long long tile0 = (long long)blockIdx.x * kEpTile;
  const int rows = (int)min((long long)kEpTile, P.n_rec - tile0);
  ep_stage_rows(P.in, tile0, rows, W, Wp, s_ep);
  __syncthreads();
  if (tid < rows) {
    const int32_t* r = s_ep + tid * Wp;
    int32_t* o = s_out + tid * WO;
    for (int k = 0; k < WO; ++k) o[k] = 0;                      // o[0] = EV_NONE
    const long long inst = ep_instance(g, r[0], r[1]);
    if (inst >= 0) {                                              // always: the validation pass judged the range
      int32_t* l = P.s.lead + inst * kEpLeadWords;
      int32_t* c = P.s.cmd + inst * kEpCmdWords;
      const int4 h0 = __ldcg((const int4*)l);                   // {kind, value, bord, brep}
      if (h0.x == LK_PREACCEPTING && ballot_key(r[2], r[3]) == ballot_key(h0.z, h0.w) &&
          (__ldcg(&l[L_FLAGS]) & LF_TIMER)) {
        int st[8];
        ep_load8(l + L_RSTAMP, st);
        int ans[kEpMaxN - 1][8];
        bool in[kEpMaxN - 1];
#pragma unroll
        for (int a = 0; a < kEpMaxN - 1; ++a) {
          in[a] = a < g.n && (uint32_t)st[a] != kStampEmpty;
          if (in[a]) ep_load8(l + L_RESP + a * kEpRespWords, ans[a]);
        }
        ep_slow_path(g, l, c, h0, ans, in, o);
      }
    }
  }
  __syncthreads();
  ep_store_rows(P.out + tile0 * WO, s_out, rows, WO, WO);
}

// ---- dense dep-set union (all `values` empty): elementwise max over the R sets of a group.
// Pure streaming, 4n(R+1) bytes per group.  A CTA stages a tile of 256 groups of the flat
// [group][set][replica] int32 array in shared memory with fully coalesced 128-bit loads,
// then thread t reduces group t (conflict-free when R*n is odd, 2-way otherwise) and the
// tile's outputs go out coalesced.
constexpr int kUnionTile = 256;
__global__ void __launch_bounds__(kUnionTile) depset_union_dense_kernel(const int32_t* __restrict__ in, int n_groups,
                                                                        int R, int n, int32_t* __restrict__ out) {
  extern __shared__ int32_t s_tile[];             // kUnionTile * R * n  (+ kUnionTile * n outputs)
  const int W = R * n;
  int32_t* s_out = s_tile + kUnionTile * W;
  for (long long g0 = (long long)blockIdx.x * kUnionTile; g0 < n_groups; g0 += (long long)gridDim.x * kUnionTile) {
    const int groups = (int)min((long long)kUnionTile, n_groups - g0);
    const long long base = g0 * W;                // multiple of 4 ints: 16-byte aligned
    const int words = groups * W;
    const int4* src = (const int4*)(in + base);
    for (int v = threadIdx.x; v < words / 4; v += kUnionTile) {
      int4 x = ld_stream(src + v);
      *(int4*)(s_tile + 4 * v) = x;
    }
    for (int v = (words & ~3) + threadIdx.x; v < words; v += kUnionTile) s_tile[v] = in[base + v];
    __syncthreads();
    if ((int)threadIdx.x < groups) {
      const int32_t* p = s_tile + threadIdx.x * W;
      for (int k = 0; k < n; ++k) {
        int m = p[k];
        for (int r = 1; r < R; ++r) m = max(m, p[r * n + k]);   // dependencies.addAll (Replica.scala:804-807)
        s_out[threadIdx.x * n + k] = m;
      }
    }
    __syncthreads();
    for (int v = threadIdx.x; v < groups * n; v += kUnionTile) __stcs(out + g0 * n + v, s_out[v]);
    __syncthreads();
  }
}

// ---- general IntPrefixSet union (S/compact/IntPrefixSet.scala:253-259, 317-351, 426-431)
// Sets are CSR: watermark[j], values[off[j] .. off[j+1]) (canonical: every value >
// watermark).  Group q unions sets [goff[q], goff[q+1]).  Output: out_w[q],
// out_values[ooff[q] .. ooff[q] + out_n[q]) sorted ascending, ooff[q] = off[goff[q]].
// One thread per group; value lists on this path are tiny (the overflow of a
// prefix set), so an in-place insertion sort beats anything cooperative.
__global__ void depset_union_kernel(const int32_t* wm, const int32_t* off, const int32_t* values, const int32_t* goff,
                                    int n_groups, int32_t* out_w, int32_t* out_n, int32_t* out_values) {
  int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n_groups) return;
  int s0 = goff[q], s1 = goff[q + 1];
  int w = 0;
  for (int j = s0; j < s1; ++j) w = max(w, wm[j]);                           // maxWatermark
  int32_t* dst = out_values + off[s0];
  int m = 0;
  for (int j = s0; j < s1; ++j) {
    for (int t = off[j]; t < off[j + 1]; ++t) {
      int v = values[t];
      if (v < w) continue;                                                  // .filter(_ >= maxWatermark)
      int pos = m;                                                          // sorted insert, dedup (a Set)
      while (pos > 0 && dst[pos - 1] > v) --pos;
      if (pos > 0 && dst[pos - 1] == v) continue;
      for (int u = m; u > pos; --u) dst[u] = dst[u - 1];
      dst[pos] = v;
      ++m;
    }
  }
  int lo = 0;
  while (lo < m && dst[lo] == w) { ++lo; ++w; }                             // compact() (:426-431)
  if (lo)
    for (int u = lo; u < m; ++u) dst[u - lo] = dst[u];
  out_w[q] = w;
  out_n[q] = m - lo;
}

}  // namespace fpx
