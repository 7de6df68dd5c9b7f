// fpx_wire_phase1.cuh -- the new leader's Phase 1 from protobuf bytes (include/fpx.h fpx_leader_phase1b_wire and
// fpx_mencius_leader_phase1b_wire).
//
// S/multipaxos/MultiPaxos.proto: Phase1bSlotInfo :254-261, Phase1b :263-271, LeaderInbound :525-539 (phase1b = 1 of
// eight members).  Leader.handlePhase1b (S/multipaxos/Leader.scala:504-577) stores the Phase1bs of the leader's round
// until they form a read quorum, then re-proposes safeValue for every slot from chosenWatermark to maxSlot.  One
// Phase1b carries one info per voted slot (up to the whole window, 2^20 entries and tens of MB at cfg2), so the
// passes are:
//   walk    one CTA per message: the CTA stages kP1Window bytes at a time in shared memory and thread 0 walks the
//           tags and lengths (LeaderInbound, then Phase1b), recording each info's body span and the Phase1b scalars.
//           The info bodies of a phase1b member that a later member replaces are located, not parsed.
//           The walk is the only sequential part: its cost is per entry, a few shared loads.
//   parse   one thread per info entry: slot, vote_round, the vote_value's span; required fields checked.
//   select  one thread over the messages in delivery order: status, round filter, phase1bs(g)(a) = msg, quorum.
//   max     one thread per entry of the Phase1bs held at completion: maxPhase1bSlot by atomicMax.
//   first   one thread per entry: the first info of a slot in each Phase1b (info.find) by atomicMin into a dense
//           [slot - chosen_watermark][acceptor index] window.
//   emit    one thread per slot of [chosen_watermark, max_slot]: the arg-max over {vote_round, lowest acceptor} of
//           that window row, written as an fpx_p2a record and the vote value's span.
// Compartmentalized Mencius (S/mencius/Leader.scala:582-659) runs the same passes for one leader group: LeaderInbound
// has nine members, the quorum is f+1 in each of the group's AG acceptor groups, max_slot is seeded with recoverSlot
// and must be owned by the group, and the slots re-proposed are s0 = nextClassicRound(leader_group, chosenWatermark - 1)
// to max_slot by LG, slot s read from acceptor group (s / LG) % AG.  MultiPaxos is that with LG = 1, leader_group 0 and
// no recoverSlot: s0 = chosen_watermark, stride 1, group s % G.  The window row of slot s is (s - s0) / LG.
#pragma once
#include "fpx_wire.cuh"

namespace fpx {

constexpr int kP1Window = 16 * 1024;   // bytes of a message staged per step of the walk
constexpr int kP1Threads = 256;
constexpr int kP1MinInfo = 8;          // bytes of the smallest info field that can hold its three required fields
constexpr int32_t kP1NoEntry = 0x7f7f7f7f;

// per message, written by the walk
struct P1Msg {
  int32_t kind;                        // LeaderInbound member, the last on the wire (0: none)
  int32_t round, group, acceptor;      // Phase1b scalars (the last of each)
  int32_t n_info;                      // info entries of the Phase1b, at entries[floor((offs[m] - offs[0]) / 8) ...]
  int32_t bad;                         // malformed, or a required field missing
  int32_t pad[2];
};

struct P1Params {
  const uint8_t* bytes;                // 16-byte aligned
  const int32_t* offs;                 // n + 1
  int32_t n, n_bytes;
  int32_t round, chosen_watermark, value_id_base, out_capacity;
  int32_t groups, per_group, flexible, quorum;  // Mencius: groups = AG, the acceptor groups of one leader group
  int32_t mencius, lgroups, leader_group;  // MultiPaxos: 0, 1, 0
  int32_t recover_slot;                // seeds max_slot; MultiPaxos INT_MIN (no seed)
  long long s0;                        // the first slot re-proposed; MultiPaxos chosen_watermark
  P1Msg* msg;                          // n
  int4* ent;                           // walk: {body off, body len, -, -}; parse: {slot, vote_round, value off, len}
  int32_t* sel;                        // [groups * per_group]: the message held as phase1bs(g)(a), -1 none
  int32_t* first;                      // [out_capacity * per_group], kP1NoEntry
  int32_t* res;                        // {complete, max_slot, n_out}, Mencius and next_slot
  fpx_p2a* out;
  int2* spans;
  unsigned long long* err_word;
};

__device__ __forceinline__ long long p1_ent_base(const P1Params& P, int m) {
  return ((long long)P.offs[m] - P.offs[0]) / kP1MinInfo;
}

// a varint from the staged window (positions are buffer offsets; the window holds [wb, wb + kP1Window)); *hi: bits
// 32.. set.  Fails past lim.
__device__ __forceinline__ uint32_t p1_varint(const uint8_t* w, long long wb, long long& p, long long lim, bool& ok,
                                              bool* hi) {
  uint32_t v = 0;
  bool h = false;
  for (int i = 0; i < 10; ++i) {
    if (p >= lim) { ok = false; return 0; }
    const uint32_t b = w[p++ - wb];
    if (i < 4) v |= (b & 0x7f) << (7 * i);
    else if (i == 4) { v |= (b & 0x0f) << 28; h |= (b & 0x70) != 0; }
    else h |= (b & 0x7f) != 0;
    if (!(b & 0x80)) { *hi = h; return v; }
  }
  ok = false;
  return 0;
}

// Walk: one CTA per message.  Thread 0 keeps the walker's state across the window steps; a step stops when the next
// field header (at most 20 bytes: a tag and a ten-byte varint) may cross the window's end.  MEMBERS: LeaderInbound's
// oneof members, 8 (MultiPaxos) or 9 (Mencius) -- a constant in the per-entry loop.
template <int MEMBERS>
__global__ void __launch_bounds__(kP1Threads) p1_walk_kernel(P1Params P) {
  __shared__ __align__(16) uint8_t s_win[kP1Window];
  __shared__ long long s_wb;
  __shared__ int s_done;
  const int m = blockIdx.x;
  const long long total = P.offs[P.n], lo = P.offs[m], hi = P.offs[m + 1];
  const bool sane = P.offs[0] >= 0 && lo >= P.offs[0] && lo <= hi && hi <= total && total - P.offs[0] <= P.n_bytes;
  // walker state (thread 0)
  long long p = lo, end1 = 0;
  int level = 0;                       // 0: LeaderInbound, 1: inside a phase1b member
  P1Msg r{0, 0, 0, 0, 0, 0, {0, 0}};
  unsigned have = 0;
  bool ok = sane, short_info = false;
  const long long eb = sane ? p1_ent_base(P, m) : 0;
  long long wb = lo & ~15ll;
  for (;;) {
    if (sane) {
      const long long stop = min(hi, wb + kP1Window);
      for (long long k = (long long)threadIdx.x * 16; wb + k < stop; k += (long long)kP1Threads * 16) {
        if (wb + k + 16 <= (total & ~15ll)) *(uint4*)(s_win + k) = __ldg((const uint4*)(P.bytes + wb + k));
        else for (int j = 0; j < 16 && wb + k + j < total; ++j) s_win[k + j] = __ldg(P.bytes + wb + k + j);
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      const long long wend = wb + kP1Window;
      bool done = !ok;
      while (!done) {
        const long long lim = level ? end1 : hi;
        if (p == lim) {
          if (level) { level = 0; continue; }
          done = true;
          break;
        }
        if (lim - p > wend - p && wend - p < 20) break;     // the header may cross the window: restage at p
        bool h = false;
        const uint32_t tag = p1_varint(s_win, wb, p, lim, ok, &h);
        if (!ok || h || (tag >> 3) == 0) { ok = false; break; }
        const int f = (int)(tag >> 3), wt = (int)(tag & 7);
        uint32_t v = 0;
        if (wt == 0) {
          v = p1_varint(s_win, wb, p, lim, ok, &h);
          if (!ok) break;
          if (level && f >= 1 && f <= 3) {                  // group_index, acceptor_index, round: int32, last wins
            if (f == 1) r.group = (int)v; else if (f == 2) r.acceptor = (int)v; else r.round = (int)v;
            have |= 1u << (f - 1);
          }
        } else if (wt == 2) {
          v = p1_varint(s_win, wb, p, lim, ok, &h);
          if (!ok || h || (v >> 31) || lim - p < (long long)v) { ok = false; break; }
          if (level == 0 && f <= MEMBERS) {
            // oneof: another member replaces the one before; the same member again merges into it
            if (f == 1) {
              if (r.kind != 1) { r.round = r.group = r.acceptor = 0; r.n_info = 0; have = 0; short_info = false; }
              level = 1; end1 = p + v;
              r.kind = 1;
              continue;                                     // walk into the body
            }
            r.kind = f;
          } else if (level && f == 4) {                     // repeated Phase1bSlotInfo info
            // a body under 6 bytes cannot hold slot, vote_round and vote_value: it fails the required check if the
            // member stays; the others take kP1MinInfo bytes or more, which bounds the entries of the message
            if (v < 6) short_info = true;
            else P.ent[eb + r.n_info++] = make_int4((int)p, (int)v, 0, 0);
          }
          p += v;
        } else if (wt == 1 || wt == 5) {
          const int k = wt == 1 ? 8 : 4;
          if (lim - p < k) { ok = false; break; }
          p += k;
        } else {
          ok = false;                                       // group wire types
          break;
        }
      }
      if (!ok) done = true;
      s_done = done;
      s_wb = p & ~15ll;
    }
    __syncthreads();
    if (s_done) break;
    wb = s_wb;
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    // "Message missing required fields": the Phase1b's three scalars
    r.bad = !ok || (r.kind == 1 && (have != 7u || short_info));
    P.msg[m] = r;
  }
}

// Parse: one thread per info entry (grid-stride over the messages' entries).  A malformed info, a missing required
// field or a second vote_value (which protobuf would merge) marks its message bad.
__global__ void __launch_bounds__(kP1Threads) p1_parse_kernel(P1Params P) {
  for (int m = blockIdx.y; m < P.n; m += gridDim.y) {
    const P1Msg r = P.msg[m];
    if (r.kind != 1 || r.bad) continue;
    const long long eb = p1_ent_base(P, m);
    for (int k = blockIdx.x * kP1Threads + threadIdx.x; k < r.n_info; k += gridDim.x * kP1Threads) {
      const int4 sp = P.ent[eb + k];
      WireReader<false> b{0u, P.bytes, (uint32_t)sp.x, (uint32_t)(sp.x + sp.y), true};
      int slot = 0, vr = 0;
      unsigned have = 0;
      uint32_t voff = 0, vlen = 0;
      bool ok = true;
      while (ok && !b.done()) {
        const uint32_t tag = b.tag();
        if (!b.ok) { ok = false; break; }
        const int f = (int)(tag >> 3), wt = (int)(tag & 7);
        if (wt == 0 && (f == 1 || f == 2)) {
          const int v = (int)b.int32();
          if (f == 1) slot = v; else vr = v;
          have |= 1u << (f - 1);
        } else if (wt == 2 && f == 3) {
          const uint32_t n = b.small();
          if (!b.ok || b.end - b.p < n || (have & 4u)) { ok = false; break; }
          voff = b.p; vlen = n; have |= 4u;
          b.p += n;
        } else if (!b.skip(wt)) {
          ok = false;
        }
        ok = ok && b.ok;
      }
      if (!ok || have != 7u) P.msg[m].bad = 1;
      P.ent[eb + k] = make_int4(slot, vr, (int)voff, (int)vlen);
    }
  }
}

__device__ __forceinline__ bool p1_complete(const P1Params& P, uint32_t mask) {
  const uint32_t row = (1u << P.per_group) - 1u;
  for (int g = 0; g < P.groups; ++g) {
    const int c = __popc((mask >> (g * P.per_group)) & row);
    if (P.flexible ? c == P.per_group : c < P.quorum) return P.flexible;
  }
  return !P.flexible;
}

// Select: the messages in delivery order, one thread.  res = {complete, max_slot seed, 0(, -1)}.
__global__ void p1_select_kernel(P1Params P) {
  const int keys = P.groups * P.per_group;
  for (int k = 0; k < keys; ++k) P.sel[k] = -1;
  uint32_t mask = 0;
  int complete = -1;
  for (int m = 0; m < P.n; ++m) {
    const P1Msg r = P.msg[m];
    if (r.bad) { report_error(P.err_word, FPX_ERR_WIRE, m); break; }
    if (r.kind != 1) continue;                                  // not a phase1b
    if (r.round < P.round) continue;                            // stale: ignored (:517-525)
    if (r.round > P.round) { report_error(P.err_word, FPX_ERR_CHECK_FAILED, m); break; }   // logger.checkLt
    if ((uint32_t)r.group >= (uint32_t)P.groups || (uint32_t)r.acceptor >= (uint32_t)P.per_group) {
      report_error(P.err_word, FPX_ERR_BAD_ACCEPTOR, m);
      break;
    }
    const int key = r.group * P.per_group + r.acceptor;
    P.sel[key] = m;                                             // phase1bs(groupIndex)(acceptorIndex) = phase1b
    mask |= 1u << key;
    if (p1_complete(P, mask)) { complete = m; break; }
  }
  // maxPhase1bSlot of an empty Phase1b is -1; the entries raise it
  int seed = INT_MIN;
  if (complete >= 0)
    for (int k = 0; k < keys; ++k)
      if (P.sel[k] >= 0 && P.msg[P.sel[k]].n_info == 0) seed = -1;
  P.res[0] = complete;
  P.res[1] = complete >= 0 ? max(seed, P.recover_slot) : -1;   // Mencius: max(..., phase1.recoverSlot)
  P.res[2] = 0;
  if (P.mencius) P.res[3] = -1;
}

// the entries of the Phase1bs held at completion: f(entry, message)
template <class F>
__device__ __forceinline__ void p1_for_held(const P1Params& P, F&& f) {
  const int complete = __ldcg(&P.res[0]);
  if (complete < 0) return;
  for (int m = blockIdx.y; m <= complete; m += gridDim.y) {
    const P1Msg r = P.msg[m];
    if (r.kind != 1 || r.round != P.round || (uint32_t)r.group >= (uint32_t)P.groups ||
        (uint32_t)r.acceptor >= (uint32_t)P.per_group || __ldcg(&P.sel[r.group * P.per_group + r.acceptor]) != m)
      continue;
    const long long eb = p1_ent_base(P, m);
    for (int k = blockIdx.x * kP1Threads + threadIdx.x; k < r.n_info; k += gridDim.x * kP1Threads)
      f(eb + k, r);
  }
}

__global__ void __launch_bounds__(kP1Threads) p1_max_kernel(P1Params P) {
  int mx = INT_MIN;
  p1_for_held(P, [&](long long e, const P1Msg&) { mx = max(mx, P.ent[e].x); });
  mx = __reduce_max_sync(0xffffffffu, mx);
  if ((threadIdx.x & 31) == 0 && mx != INT_MIN) atomicMax(&P.res[1], mx);
}

// the slots s0, s0 + LG, ... up to max_slot
__device__ __forceinline__ long long p1_count(const P1Params& P, long long max_slot) {
  return max_slot >= P.s0 ? (max_slot - P.s0) / P.lgroups + 1 : 0;
}
// Mencius: nextSlot = nextClassicRound(leader_group, max_slot) (RoundSystem.scala:66-80), in 64 bits
__device__ __forceinline__ long long p1_next_slot(const P1Params& P, long long max_slot) {
  if (max_slot < 0) return P.leader_group;
  const long long base = P.lgroups * (max_slot / P.lgroups) + P.leader_group;
  return base > max_slot ? base : base + P.lgroups;
}
// why a completed call emits nothing (FPX_OK: it emits): the Mencius max_slot owner check (logger.check), a
// next_slot past int32, then more records than out_capacity
__device__ __forceinline__ int p1_refusal(const P1Params& P, long long max_slot) {
  if (P.mencius) {
    if (max_slot != -1 && max_slot % P.lgroups != P.leader_group) return FPX_ERR_CHECK_FAILED;
    if (p1_next_slot(P, max_slot) > INT_MAX) return FPX_ERR_SLOT_RANGE;
  }
  return p1_count(P, max_slot) > P.out_capacity ? FPX_ERR_INVALID_ARG : FPX_OK;
}

// the window rows [0, count) when the call completes and emits, else 0 rows
__device__ __forceinline__ long long p1_window(const P1Params& P) {
  if (__ldcg(&P.res[0]) < 0) return 0;
  const long long max_slot = __ldcg(&P.res[1]);
  return p1_refusal(P, max_slot) == FPX_OK ? p1_count(P, max_slot) : 0;
}

__global__ void __launch_bounds__(kP1Threads) p1_first_kernel(P1Params P) {
  const long long count = p1_window(P);
  if (count == 0) return;
  p1_for_held(P, [&](long long e, const P1Msg& r) {
    const int slot = P.ent[e].x;
    const long long d = (long long)slot - P.s0;               // < 2^31 once it is >= 0
    // a slot of another leader group counts toward max_slot only
    if (d < 0 || (uint32_t)d % (uint32_t)P.lgroups != 0) return;
    const long long k = (uint32_t)d / (uint32_t)P.lgroups;
    // safeValue reads phase1bs(slot % numAcceptorGroups) only (:552); Mencius acceptorGroupIndexBySlot (:342-345)
    if (k >= count || (slot / P.lgroups) % P.groups != r.group) return;
    atomicMin(&P.first[k * P.per_group + r.acceptor], (int32_t)e);
  });
}

__global__ void __launch_bounds__(kP1Threads) p1_emit_kernel(P1Params P) {
  const int complete = __ldcg(&P.res[0]);
  if (complete < 0) return;
  const long long max_slot = __ldcg(&P.res[1]);
  const int refused = p1_refusal(P, max_slot);
  if (refused != FPX_OK) {                                      // nothing written
    if (blockIdx.x == 0 && threadIdx.x == 0) report_error(P.err_word, refused, complete);
    return;
  }
  const long long count = p1_count(P, max_slot);
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    P.res[2] = (int32_t)count;
    if (P.mencius) P.res[3] = (int32_t)p1_next_slot(P, max_slot);
  }
  for (long long k = (long long)blockIdx.x * kP1Threads + threadIdx.x; k < count; k += (long long)gridDim.x * kP1Threads) {
    int best = -1, bvr = 0;
    for (int a = 0; a < P.per_group; ++a) {                    // ties in vote_round: the lowest acceptor index
      const int e = P.first[k * P.per_group + a];
      if (e == kP1NoEntry) continue;
      const int vr = P.ent[e].y;
      if (best < 0 || vr > bvr) { best = e; bvr = vr; }
    }
    const int slot = (int)(P.s0 + k * P.lgroups);
    int2 sp = make_int2(0, 0);
    int value = FPX_VALUE_NOOP;
    if (best >= 0) {
      const int4 en = P.ent[best];
      sp = make_int2(en.z, en.w);
      value = P.value_id_base + (int)k;
    }
    P.out[k] = fpx_p2a{slot, P.round, value, -1};
    P.spans[k] = sp;
  }
}


// ---------------------------------------------------------------------------
// The acceptor's side (include/fpx.h fpx_acceptor_phase1a_wire): Acceptor.handlePhase1a (S/multipaxos/Acceptor.scala:
// 148-182) per decoded AcceptorInbound record, its Phase1b or Nack as LeaderInbound bytes.  Passes:
//   parse   one thread per record: the Phase1a body {round, chosen_watermark}, the voter, the retired base;
//   apply   one thread per acceptor, its records in delivery order: Nack(round) below the acceptor's round, else
//           round = phase1a.round and a Phase1b -- skipped entirely when any record failed (nothing applied);
//   count   (slot tile, record): the acceptor's voted slots in [chosen_watermark, maxVotedSlot];
//   scan    tile_offsets_kernel over the (record, tile) counts: each info's place, grouped by message;
//   fill    (slot tile, record): one encode record per message header and per info, and the message's summed
//           body length (atomicAdd) which the header needs;
//   encode  the gathering encoder with P1bCodec over the n + infos records, then the messages' offsets.
// Compartmentalized Mencius (S/mencius/Acceptor.scala:166-200, fpx_mencius_acceptor_phase1a_wire) differs in what the
// passes read and write, not in the passes: acceptor (lg, ag) holds the slots lg + LG * ag mod LG * AG, so count and
// fill step by LG * AG from the first such slot >= chosen_watermark, up to the end of the live window (its
// Phase2aNoopRange votes do not raise acc_max_voted); the Phase1b's group_index is ag and the Nack is member 7.
// ---------------------------------------------------------------------------
constexpr int kP1aTile = 1024;       // slots per count / fill CTA (4 per thread)
enum { kP1aNone = 0, kP1aPhase1b = 1, kP1aNack = 2 };

struct P1aParams {
  Geometry g;
  const unsigned long long* votes;
  int32_t* acc_round;
  const int32_t* acc_max_voted;
  const uint8_t* bytes;                // the request batch
  int32_t n_bytes;
  const int32_t* kind;
  const int4* in;                      // fpx_wire_decode_inbound's records, a = group << 16 | acceptor
  int32_t n, tiles;                    // tiles: slot tiles of the live window
  int32_t* rnd;                        // [n] phase1a.round
  int32_t* lo;                         // [n] first slot of the Phase1b's infos
  int32_t* reply;                      // [n] kP1a*
  int32_t* nack;                       // [n] the acceptor's round (Nack)
  int32_t* bad;                        // a record failed: nothing is applied
  uint32_t* cnt;                       // [n * tiles + 1] infos per (record, tile), then their exclusive offsets
  int32_t* body;                       // [n] summed bytes of a Phase1b's infos
  int4* recs;                          // [n + infos] {slot, vote_round, value_id, message} / header {0, 0, 0, -1 - m}
  const int32_t* value_offs;
  int32_t num_values;
  unsigned long long* err_word;
  int32_t mencius;                     // slots of the acceptor's residue, to the live window's end
  int32_t stride;                      // 1, Mencius LG * AG
  int32_t wire_groups;                 // Phase1b.group_index = engine group % wire_groups (Mencius AG)
  int32_t nack_tag;                    // LeaderInbound.nack: 0x32 (= 6), Mencius 0x3a (= 7)
};

// (vote round, value) of acceptor (group, acceptor) at slot, round -1 for none (fpx_snapshot_acceptor's rule)
__device__ __forceinline__ int p1a_vote(const P1aParams& P, int group, int acceptor, int slot, int* value) {
  const int l = local_slot(P.g, slot);
  if (l < 0) return -1;
  const int v = voter_index(P.g, group, acceptor, slot);
  if (v < 0 || (!P.g.flexible && group != expected_group(P.g, slot))) return -1;
  const unsigned long long c = P.votes[cell_index(P.g, l, v)];
  if ((c >> 32) == 0) return -1;
  *value = (int)(uint32_t)c;
  return (int)(c >> 32) - 1;
}
__device__ __forceinline__ int p1a_first_held(const Geometry& g) { return g.base_local; }   // one shard

__global__ void __launch_bounds__(256) p1a_parse_kernel(P1aParams P) {
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= P.n) return;
  P.reply[i] = kP1aNone;
  if (P.kind[i] != 1) return;                                    // AcceptorInbound.phase1a = 1
  const int4 r = P.in[i];
  int code = FPX_OK, round = 0, cw = 0;
  if (r.z < 0 || r.w < 0 || (long long)r.z + r.w > P.n_bytes) {
    code = FPX_ERR_WIRE;
  } else {
    WireReader<false> b{0u, P.bytes, (uint32_t)r.z, (uint32_t)(r.z + r.w), true};
    unsigned have = 0;
    while (!b.done()) {
      const uint32_t tag = b.tag();
      if (!b.ok) break;
      const int f = (int)(tag >> 3), wt = (int)(tag & 7);
      if (wt == 0 && (f == 1 || f == 2)) {
        const int v = (int)b.int32();
        if (f == 1) round = v; else cw = v;
        have |= 1u << (f - 1);
      } else if (!b.skip(wt)) {
        break;
      }
    }
    if (!b.ok || have != 3u) code = FPX_ERR_WIRE;
  }
  const int group = r.x >> 16, acceptor = r.x & 0xffff;
  if (code == FPX_OK && ((uint32_t)group >= (uint32_t)P.g.groups || acceptor >= P.g.per_group)) code = FPX_ERR_INVALID_ARG;
  // votes below the retired base are gone: the reference would send them
  const int first = p1a_first_held(P.g);
  if (code == FPX_OK && cw < first && first > 0) code = FPX_ERR_SLOT_RANGE;
  if (code != FPX_OK) {
    report_error(P.err_word, code, i);
    *P.bad = 1;
    return;
  }
  P.rnd[i] = round;
  P.lo[i] = max(cw, first);
}

// one thread per acceptor key
__global__ void p1a_apply_kernel(P1aParams P) {
  const int k = threadIdx.x;
  if (k >= P.g.groups * P.g.per_group || __ldcg(P.bad)) return;
  int cur = P.acc_round[k];
  bool touched = false;
  for (int i = 0; i < P.n; ++i) {
    if (P.kind[i] != 1) continue;
    const int a = P.in[i].x;
    if ((a >> 16) * P.g.per_group + (a & 0xffff) != k) continue;
    const int r = P.rnd[i];
    if (r < cur) {                                               // Nack(round), Acceptor.scala:156-163
      P.reply[i] = kP1aNack; P.nack[i] = cur;
    } else {                                                     // round = phase1a.round (:166), Phase1b (:171-181)
      cur = r; touched = true;
      P.reply[i] = kP1aPhase1b;
    }
  }
  if (touched) P.acc_round[k] = cur;
}

// the Phase1b of record i covers slots lo, lo + stride, ... <= hi; tile t of it
__device__ __forceinline__ bool p1a_range(const P1aParams& P, int i, int* lo, int* hi) {
  if (__ldcg(P.bad) || P.reply[i] != kP1aPhase1b) return false;
  const int a = P.in[i].x;
  *lo = P.lo[i];
  if (P.mencius) {
    // the first slot >= lo of the acceptor's residue lg + LG * ag; noop-range votes leave acc_max_voted as it was
    const int group = a >> 16, r = group / P.g.agroups + P.g.lgroups * (group % P.g.agroups);
    const long long first = (long long)*lo + ((r - *lo % P.stride) % P.stride + P.stride) % P.stride;
    *hi = P.g.slot_capacity - 1;
    if (first > *hi) return false;
    *lo = (int)first;
  } else {
    *hi = P.acc_max_voted[(a >> 16) * P.g.per_group + (a & 0xffff)];
  }
  return *lo <= *hi;
}

__global__ void __launch_bounds__(256) p1a_count_kernel(P1aParams P) {
  const int i = blockIdx.y, t = blockIdx.x;
  int lo, hi;
  uint32_t c = 0;
  if (p1a_range(P, i, &lo, &hi)) {
    const int a = P.in[i].x;
    for (int u = 0; u < kP1aTile / 256; ++u) {
      const long long s = (long long)lo + ((long long)t * kP1aTile + u * 256 + threadIdx.x) * P.stride;
      int v;
      if (s <= hi && p1a_vote(P, a >> 16, a & 0xffff, (int)s, &v) >= 0) ++c;
    }
  }
  c = cta_reduce<256>(c, ScanSum());
  if (threadIdx.x == 0) P.cnt[(long long)i * P.tiles + t] = c;
}

__device__ __forceinline__ int p1a_value_len(const P1aParams& P, int v, bool* bad) {
  if (v == FPX_VALUE_NOOP) return 2;
  if ((uint32_t)v >= (uint32_t)P.num_values) { *bad = true; return 0; }
  const int len = P.value_offs[v + 1] - P.value_offs[v];
  if (len < 0) *bad = true;
  return len < 0 ? 0 : len;
}
// bytes of one info field (tag, length, body)
__device__ __forceinline__ int p1a_info_size(int slot, int vr, int vlen) {
  const int b = 2 + wire_int32_size(slot) + wire_int32_size(vr) + 1 + wire_varint_size((unsigned long long)vlen) + vlen;
  return 1 + wire_varint_size((unsigned long long)b) + b;
}

__global__ void __launch_bounds__(256) p1a_fill_kernel(P1aParams P) {
  const int i = blockIdx.y, t = blockIdx.x;
  const long long first = P.cnt[(long long)i * P.tiles];             // infos before message i
  if (t == 0 && threadIdx.x == 0) P.recs[i + first] = make_int4(0, 0, 0, -1 - i);
  int lo, hi;
  const bool live = p1a_range(P, i, &lo, &hi);
  const int a = P.in[i].x;
  uint32_t base = P.cnt[(long long)i * P.tiles + t];
  uint32_t sum = 0;
  for (int u = 0; u < kP1aTile / 256; ++u) {
    const long long s = (long long)lo + ((long long)t * kP1aTile + u * 256 + threadIdx.x) * P.stride;
    int v = 0, vr = -1;
    if (live && s <= hi) vr = p1a_vote(P, a >> 16, a & 0xffff, (int)s, &v);
    uint32_t tot;
    const uint32_t rank = cta_scan<256, true>(vr >= 0 ? 1u : 0u, ScanSum(), &tot);
    if (vr >= 0) {
      bool badv = false;
      const int vlen = p1a_value_len(P, v, &badv);
      if (badv) report_error(P.err_word, FPX_ERR_INVALID_ARG, i);
      sum += (uint32_t)p1a_info_size((int)s, vr, vlen);
      P.recs[i + 1 + base + rank] = make_int4((int)s, vr, v, i);
    }
    base += tot;
  }
  sum = cta_reduce<256>(sum, ScanSum());
  if (threadIdx.x == 0 && sum) atomicAdd(&P.body[i], (int)sum);
}

// the gathering encoder's codec over the header and info records
struct P1bEncParams {
  WireEnc enc;                         // enc.src: the value arena
  P1aParams A;
};
struct P1bMsg {
  int kind;                            // 0 nothing, 1 Phase1b header, 2 Nack, 3 info
  int f0, f1, f2;                      // header: group, acceptor, round; Nack: round; info: slot, vote_round
  int body;                            // header: the infos' bytes; info: the value's length
  int src;
  bool noop;
};
struct P1bCodec {
  using Params = P1bEncParams;
  using Msg = P1bMsg;
  static __device__ __forceinline__ bool stand_down(const Params& P) { return __ldcg(P.A.bad) != 0; }
  static __device__ __forceinline__ Msg msg(const Params& P, int r, int* code) {
    const int4 x = P.A.recs[r];
    Msg m{0, 0, 0, 0, 0, 0, false};
    if (x.w < 0) {
      const int i = -1 - x.w;
      const int rep = P.A.reply[i];
      if (rep == kP1aNack) { m.kind = 2; m.f0 = P.A.nack[i]; }
      else if (rep == kP1aPhase1b) {
        const int a = P.A.in[i].x;
        m.kind = 1; m.f0 = (a >> 16) % P.A.wire_groups; m.f1 = a & 0xffff; m.f2 = P.A.rnd[i]; m.body = __ldcg(&P.A.body[i]);
      }
      return m;
    }
    m.kind = 3; m.f0 = x.x; m.f1 = x.y;
    if (x.z == FPX_VALUE_NOOP) { m.noop = true; m.body = 2; return m; }
    bool bad = false;
    m.body = p1a_value_len(P.A, x.z, &bad);
    if (bad) { *code = FPX_ERR_INVALID_ARG; m.kind = 0; return m; }
    m.src = P.A.value_offs[x.z];
    return m;
  }
  static __device__ __forceinline__ int size(const Params&, const Msg& m) {
    if (m.kind == 1) {                 // the head only: the infos are records of their own
      const int b = 3 + wire_int32_size(m.f0) + wire_int32_size(m.f1) + wire_int32_size(m.f2) + m.body;
      return 1 + wire_varint_size((unsigned long long)b) + b - m.body;
    }
    if (m.kind == 2) return 2 + 1 + wire_int32_size(m.f0);
    if (m.kind == 3) return p1a_info_size(m.f0, m.f1, m.body);
    return 0;
  }
  static __device__ __forceinline__ int size_of(const Params& P, int r, int* code) { return size(P, msg(P, r, code)); }
  static __device__ __forceinline__ uint8_t* head(const Params& P, const Msg& m, uint8_t* p, int* gsrc, int* glen) {
    *gsrc = 0; *glen = 0;
    if (m.kind == 1) {                 // LeaderInbound{phase1b = 1 {group_index, acceptor_index, round, info...}}
      const int b = 3 + wire_int32_size(m.f0) + wire_int32_size(m.f1) + wire_int32_size(m.f2) + m.body;
      *p++ = 0x0a; p = wire_put_varint(p, (unsigned long long)b);
      p = wire_put_int32(p, 1, m.f0); p = wire_put_int32(p, 2, m.f1); p = wire_put_int32(p, 3, m.f2);
    } else if (m.kind == 2) {          // LeaderInbound{nack = 6 (Mencius 7) {round}}
      *p++ = (uint8_t)P.A.nack_tag; *p++ = (uint8_t)(1 + wire_int32_size(m.f0));
      p = wire_put_int32(p, 1, m.f0);
    } else if (m.kind == 3) {          // info = 4 {slot, vote_round, vote_value}
      const int b = 2 + wire_int32_size(m.f0) + wire_int32_size(m.f1) + 1 + wire_varint_size((unsigned long long)m.body) + m.body;
      *p++ = 0x22; p = wire_put_varint(p, (unsigned long long)b);
      p = wire_put_int32(p, 1, m.f0); p = wire_put_int32(p, 2, m.f1);
      *p++ = 0x1a; p = wire_put_varint(p, (unsigned long long)m.body);
      if (m.noop) { *p++ = 0x12; *p++ = 0x00; }
      else { *gsrc = m.src; *glen = m.body; }
    }
    return p;
  }
};

// message offsets from the records' offsets: message i starts at its header record
__global__ void p1a_offsets_kernel(P1aParams P, const int32_t* rec_offs, int32_t total_recs, int32_t* offsets) {
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i < P.n) offsets[i] = rec_offs[i + P.cnt[(long long)i * P.tiles]];
  if (i == P.n) offsets[i] = rec_offs[total_recs];
}

}  // namespace fpx
