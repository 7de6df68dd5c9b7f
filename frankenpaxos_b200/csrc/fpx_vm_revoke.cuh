// fpx_vm_revoke.cuh -- vanilla Mencius revocation, the servers' side (include/fpx.h fpx_vm_phase1a_wire,
// fpx_vm_entries): Server.handlePhase1a (S/vanillamencius/Server.scala:831-911) from ServerInbound bytes.
//
// Entries.  A vote cell is {hi: round + 1 | kCellChosen, lo: value}.  Phase2a always writes round == voteRound, so
// the cell holds a PendingEntry exactly.  A Phase1a adds two more kinds: VotelessEntry(round) and a PendingEntry
// whose round was raised above its voteRound.  Such a RAISED cell is {hi: round + 1, lo: kVmRaised} and its
// {voteRound (-1: voteless), value} sits in the side table vm_raise[cell], which only Phase1a writes.
// vm_phase2a_kernel needs no change for them: its round compare reads hi, a Nack leaves the cell as it was, and an
// accept overwrites lo with the proposal's value -- exactly where round == voteRound becomes true again.  (The
// cell's claim word cannot carry the raise: vm_phase2a rewrites the claim on a Nack too.)  kVmRaised is a value id
// the engine reserves (FPX_VALUE_RAISED); a ChosenEntry is {kCellChosen | kCellRevocation if isRevocation, value}.
//
// Phase1a passes:
//   parse   one thread per record: the body {round, start, stop}, the receiving server, the checks; walked slots
//           per record (ceil((stop - start) / n)), whose exclusive sum (tile_offsets_kernel) places the record's
//           encode records: one head, then one per walked slot;
//   apply   one CTA per server walks its records in delivery order -- they depend on each other only through the
//           rounds they raise and next_slot.  A record revoking the server itself first runs the log fill of
//           advanceWithSkips(stop - 1).  The walk takes 256 slots at a time: the first stale slot by a block
//           min-reduction, the raise below it, and one info (or an empty record) per slot;
//   encode  the gathering encoder over the head and info records; empty records take no bytes.
// Revocations are rare: a batch holds few Phase1a, each over up to 2 beta / n slots of one server.
#pragma once
#include "fpx_ranges.cuh"
#include "fpx_wire.cuh"

namespace fpx {

constexpr uint32_t kVmRaised = 0x80000001u;   // FPX_VALUE_RAISED: the cell's entry is in vm_raise
constexpr int kVmP1aThreads = 256;

// the entry of one (slot, server) cell; kind 0 None, 1 Voteless, 2 Pending, 3 Chosen
struct VmEntry {
  int kind, round, vote_round, value, revocation;
};
__device__ __forceinline__ VmEntry vm_entry(unsigned long long c, const unsigned long long* raise, size_t ri) {
  const uint32_t hi = (uint32_t)(c >> 32), lo = (uint32_t)c;
  if (c & kCellChosen) return {3, 0, 0, (int)lo, (c & kCellRevocation) ? 1 : 0};
  if (hi == 0) return {0, -1, -1, 0, 0};
  if (lo == kVmRaised && raise) {
    const unsigned long long s = raise[ri];
    const int vr = (int)(uint32_t)(s >> 32);
    return {vr < 0 ? 1 : 2, (int)hi - 1, vr, vr < 0 ? 0 : (int)(uint32_t)s, 0};
  }
  return {2, (int)hi - 1, (int)hi - 1, (int)lo, 0};
}

struct VmP1aParams {
  Geometry g;
  unsigned long long* votes;
  unsigned long long* raise;           // [local_slots * n]: {voteRound, value} of raised cells
  const uint32_t* rows;
  const uint8_t* bytes;
  int32_t n_bytes;
  const int32_t* kind;
  const int4* in;                      // fpx_wire_decode_vm_server_inbound's records, a = the receiving server
  int32_t n;
  int32_t* next_slot;                  // [servers] in / out
  int32_t *rnd, *start, *stop;         // [n] the Phase1a
  uint32_t* cnt;                       // [n + 1] walked slots per record, then their exclusive offsets and the total
  int32_t* reply;                      // [n] 0 none, 1 Phase1b, 2 Phase1Nack
  int32_t* nack;                       // [n] the Nack's round
  int32_t* body;                       // [n] the Phase1b's summed info bytes
  int4* recs;                          // [n + total]: head {3, i, 0, 0} at i + cnt[i], then one per walked slot:
                                       // {1 pending, slot, voteRound, value} | {2 chosen, slot, isRevocation, value}
                                       // | {0, ...} (nothing: past a Nack)
  int4* skips;                         // [n] fpx_vm_skip_rec of the log fill, slot_start == slot_stop: none
  const int32_t* value_offs;
  int32_t num_values;
  int32_t* bad;
  unsigned long long* err_word;
};

__device__ __forceinline__ int vm_value_len(const int32_t* value_offs, int32_t num_values, int v, bool* bad) {
  if (v == FPX_VALUE_NOOP) return 2;
  if ((uint32_t)v >= (uint32_t)num_values) { *bad = true; return 0; }
  const int len = value_offs[v + 1] - value_offs[v];
  if (len < 0) *bad = true;
  return len < 0 ? 0 : len;
}
// Phase1bSlotInfo{slot, pending_slot_info {vote_round, vote_value} | chosen_slot_info {value, is_revocation}}
__device__ __forceinline__ int vm_info_inner(int kind, int a, int vlen) {
  return kind == 1 ? 1 + wire_int32_size(a) + 1 + wire_varint_size((unsigned long long)vlen) + vlen
                   : 1 + wire_varint_size((unsigned long long)vlen) + vlen + 2;
}
__device__ __forceinline__ int vm_info_body(int kind, int slot, int a, int vlen) {
  const int in = vm_info_inner(kind, a, vlen);
  return 1 + wire_int32_size(slot) + 1 + wire_varint_size((unsigned long long)in) + in;
}
__device__ __forceinline__ int vm_info_size(int kind, int slot, int a, int vlen) {
  const int b = vm_info_body(kind, slot, a, vlen);
  return 1 + wire_varint_size((unsigned long long)b) + b;
}

__global__ void __launch_bounds__(256) vm_p1a_parse_kernel(VmP1aParams P) {
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= P.n) return;
  const int4 r = P.in[i];
  P.reply[i] = 0; P.cnt[i] = 0; P.body[i] = 0;
  P.skips[i] = make_int4(r.x, 0, 0, 1);
  if (P.kind[i] != 2) return;                                    // ServerInbound.phase1a = 2
  const Geometry& g = P.g;
  const int servers = g.per_group;
  int code = FPX_OK, round = 0, start = 0, stop = 0;
  if (r.z < 0 || r.w < 0 || (long long)r.z + r.w > P.n_bytes) {
    code = FPX_ERR_WIRE;
  } else {
    WireReader<false> b{0u, P.bytes, (uint32_t)r.z, (uint32_t)(r.z + r.w), true};
    unsigned have = 0;
    while (!b.done()) {
      const uint32_t tag = b.tag();
      if (!b.ok) break;
      const int f = (int)(tag >> 3), wt = (int)(tag & 7);
      if (wt == 0 && f >= 1 && f <= 3) {
        const int v = (int)b.int32();
        if (f == 1) round = v; else if (f == 2) start = v; else stop = v;
        have |= 1u << (f - 1);
      } else if (!b.skip(wt)) {
        break;
      }
    }
    if (!b.ok || have != 7u) code = FPX_ERR_WIRE;
  }
  const int server = r.x;
  long long count = 0;
  if (code == FPX_OK && (uint32_t)server >= (uint32_t)servers) code = FPX_ERR_INVALID_ARG;
  if (code == FPX_OK && (uint32_t)round > (uint32_t)FPX_MAX_ROUND) code = FPX_ERR_ROUND_RANGE;
  if (code == FPX_OK && start < 0) code = FPX_ERR_SLOT_RANGE;
  if (code == FPX_OK && start < stop) {
    // every walked slot live: the engine no longer holds a retired slot's entry
    count = ((long long)stop - start + servers - 1) / servers;
    if (local_slot(g, start) < 0 || local_slot(g, (int)(start + (count - 1) * servers)) < 0) code = FPX_ERR_SLOT_RANGE;
  }
  if (code == FPX_OK && start % servers == server) {
    // the revoked server itself: advanceWithSkips(stop - 1) fills [next_slot, stop - 1]; every slot of it live,
    // and the next_slot after it within int32 (the reference's Int would wrap)
    const int ns = P.next_slot[server];
    if (ns < 0 || ns % servers != server) code = FPX_ERR_INVALID_ARG;
    else if ((long long)stop - 1 >= ns &&
             (local_slot(g, ns) < 0 || local_slot(g, stop - 1) < 0 || (long long)stop - 1 + servers > INT_MAX))
      code = FPX_ERR_SLOT_RANGE;
  }
  if (code != FPX_OK) {
    report_error(P.err_word, code, i);
    *P.bad = 1;
    return;
  }
  P.rnd[i] = round; P.start[i] = start; P.stop[i] = stop;
  P.cnt[i] = (uint32_t)count;
}

// one CTA per server, its records in delivery order
__global__ void __launch_bounds__(kVmP1aThreads) vm_p1a_apply_kernel(VmP1aParams P) {
  __shared__ int s_stale, s_nack;
  if (__ldcg(P.bad)) return;
  const Geometry& g = P.g;
  const int s = blockIdx.x, servers = g.per_group, t = threadIdx.x;
  // 32-bit slot arithmetic throughout (a 64-bit division is a subroutine call, and its spills): the parse pass
  // bounds every slot here, next_slot after a fill included, by INT_MAX
  int ns = P.next_slot[s];
  bool moved = false;
  for (int i = 0; i < P.n; ++i) {
    if (P.kind[i] != 2 || P.in[i].x != s) continue;
    const int round = P.rnd[i], start = P.start[i], stop = P.stop[i];
    const long long head = (long long)i + P.cnt[i];
    const int count = (int)(P.cnt[i + 1] - P.cnt[i]);
    if (start % servers == s && stop > ns) {                     // stop - 1 >= ns
      // advanceWithSkips(stop - 1) (:577-620): own slots ns, ns + n, ... < newStop become ChosenEntry(Noop); each
      // must be vacant (logger.check(!log.contains), check(!phase2s.contains), :613-614)
      const int new_stop = (stop - 1) % servers == s ? stop : stop - 1;
      const int fills = (int)((uint32_t)(new_stop - ns + servers - 1) / (uint32_t)servers);
      for (int k = t; k < fills; k += kVmP1aThreads)
        if (!vm_fill_own(g, P.votes, P.rows, local_slot(g, ns + k * servers), s))
          report_error(P.err_word, FPX_ERR_CHECK_FAILED, i);
      if (t == 0) P.skips[i] = make_int4(s, ns, new_stop, 1);
      ns += fills * servers;
      moved = true;
      __syncthreads();
    } else if (t == 0) {
      P.skips[i] = make_int4(s, ns, ns, 1);
    }
    // the walk (:860-900): the first stale entry stops it with a Nack; the entries before it stay raised
    bool stopped = false;
    uint32_t sum = 0;
    if (t == 0) s_nack = 0;
    for (int c0 = 0; c0 < count; c0 += kVmP1aThreads) {
      if (t == 0) s_stale = INT_MAX;
      __syncthreads();
      const int k = c0 + t;
      const int slot = start + k * servers;
      const bool live = k < count && !stopped;
      VmEntry en{0, 0, 0, 0, 0};
      unsigned long long* cell = nullptr;
      size_t ri = 0;
      if (live) {
        const int l = local_slot(g, slot);
        cell = P.votes + cell_index(g, l, s);
        ri = (size_t)l * g.voters + s;
        en = vm_entry(__ldcg(cell), P.raise, ri);
        if ((en.kind == 1 || en.kind == 2) && en.round > round) atomicMin(&s_stale, (int)t);
      }
      __syncthreads();
      const int first = s_stale;
      int4 info = make_int4(0, slot, 0, 0);
      if (live && t < first) {
        if (en.kind == 3) {
          info = make_int4(2, slot, en.revocation, en.value);        // ChosenSlotInfo (:893-898)
        } else {
          if (en.kind == 2) {
            info = make_int4(1, slot, en.vote_round, en.value);      // PendingSlotInfo (:883-888)
            if (en.round < round && (uint32_t)__ldcg(cell) != kVmRaised)   // not raised before: its vote moves aside
              P.raise[ri] = ((unsigned long long)(uint32_t)en.vote_round << 32) | (uint32_t)en.value;
          } else if (en.kind == 0) {
            P.raise[ri] = 0xffffffff00000000ull;                     // VotelessEntry: voteRound -1
          }
          if (en.kind == 0 || en.round < round)                      // log.put(slot, ...(round = phase1a.round))
            *cell = ((unsigned long long)(uint32_t)(round + 1) << 32) | kVmRaised;
        }
        if (info.x) {
          bool bad = false;
          const int vlen = vm_value_len(P.value_offs, P.num_values, info.w, &bad);
          if (bad) report_error(P.err_word, FPX_ERR_INVALID_ARG, i);
          sum += (uint32_t)vm_info_size(info.x, slot, info.z, vlen);
        }
      }
      if (live && t == first) s_nack = en.round;                     // Phase1Nack(start, stop, entry.round)
      if (k < count) P.recs[head + 1 + k] = info;
      stopped = stopped || first != INT_MAX;
      __syncthreads();                                               // s_stale is read: the next chunk may reset it
    }
    if (stopped)                                                     // a Nack carries no infos
      for (int k = t; k < count; k += kVmP1aThreads) P.recs[head + 1 + k].x = 0;
    sum = cta_reduce<kVmP1aThreads>(sum, ScanSum());
    if (t == 0) {
      P.reply[i] = stopped ? 2 : 1;
      P.nack[i] = s_nack;
      P.body[i] = (int)sum;
    }
    __syncthreads();
  }
  if (t == 0 && moved) P.next_slot[s] = ns;
}

// the head records of the other kinds (non-Phase1a records get a zero-length reply)
__global__ void vm_p1a_heads_kernel(VmP1aParams P) {
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i < P.n) P.recs[(long long)i + P.cnt[i]] = make_int4(3, i, 0, 0);
}

struct VmP1bEncParams {
  WireEnc enc;                         // enc.src: the value arena
  VmP1aParams A;
};
struct VmP1bMsg {
  int kind;                            // 0 nothing, 1 Phase1b head, 2 Nack, 3 pending info, 4 chosen info
  int f0, f1, f2, f3;                  // head: server, round, start, stop; Nack: start, stop, round; info: slot, a
  int body;                            // head: the infos' bytes; info: the value's length
  int src;
  bool noop;
};
struct VmP1bCodec {
  using Params = VmP1bEncParams;
  using Msg = VmP1bMsg;
  static __device__ __forceinline__ bool stand_down(const Params& P) { return __ldcg(P.A.bad) != 0; }
  static __device__ __forceinline__ int head_body(const Msg& m) {
    return 4 + wire_int32_size(m.f0) + wire_int32_size(m.f1) + wire_int32_size(m.f2) + wire_int32_size(m.f3) + m.body;
  }
  static __device__ __forceinline__ Msg msg(const Params& P, int r, int* code) {
    const int4 x = P.A.recs[r];
    Msg m{0, 0, 0, 0, 0, 0, 0, false};
    if (x.x == 3) {
      const int i = x.y, rep = P.A.reply[i];
      if (rep == 1) {
        m.kind = 1; m.f0 = P.A.in[i].x; m.f1 = P.A.rnd[i]; m.f2 = P.A.start[i]; m.f3 = P.A.stop[i];
        m.body = __ldcg(&P.A.body[i]);
      } else if (rep == 2) {
        m.kind = 2; m.f0 = P.A.start[i]; m.f1 = P.A.stop[i]; m.f2 = P.A.nack[i];
      }
      return m;
    }
    if (x.x != 1 && x.x != 2) return m;
    m.kind = x.x + 2; m.f0 = x.y; m.f1 = x.z;
    if (x.w == FPX_VALUE_NOOP) { m.noop = true; m.body = 2; return m; }
    bool bad = false;
    m.body = vm_value_len(P.A.value_offs, P.A.num_values, x.w, &bad);
    if (bad) { *code = FPX_ERR_INVALID_ARG; m.kind = 0; return m; }
    m.src = P.A.value_offs[x.w];
    return m;
  }
  static __device__ __forceinline__ int size(const Params&, const Msg& m) {
    if (m.kind == 1) {                 // the head only: the infos are records of their own
      const int b = head_body(m);
      return 1 + wire_varint_size((unsigned long long)b) + b - m.body;
    }
    if (m.kind == 2) return 2 + 3 + wire_int32_size(m.f0) + wire_int32_size(m.f1) + wire_int32_size(m.f2);
    if (m.kind >= 3) return vm_info_size(m.kind - 2, m.f0, m.f1, m.body);
    return 0;
  }
  static __device__ __forceinline__ int size_of(const Params& P, int r, int* code) { return size(P, msg(P, r, code)); }
  static __device__ __forceinline__ uint8_t* head(const Params&, const Msg& m, uint8_t* p, int* gsrc, int* glen) {
    *gsrc = 0; *glen = 0;
    if (m.kind == 1) {                 // ServerInbound{phase1b = 3 {server_index, round, start, stop, info = 5...}}
      *p++ = 0x1a; p = wire_put_varint(p, (unsigned long long)head_body(m));
      p = wire_put_int32(p, 1, m.f0); p = wire_put_int32(p, 2, m.f1); p = wire_put_int32(p, 3, m.f2);
      p = wire_put_int32(p, 4, m.f3);
    } else if (m.kind == 2) {          // ServerInbound{phase1_nack = 8 {start, stop, round}}
      *p++ = 0x42; *p++ = (uint8_t)(3 + wire_int32_size(m.f0) + wire_int32_size(m.f1) + wire_int32_size(m.f2));
      p = wire_put_int32(p, 1, m.f0); p = wire_put_int32(p, 2, m.f1); p = wire_put_int32(p, 3, m.f2);
    } else if (m.kind >= 3) {          // info {slot = 1, pending_slot_info = 2 | chosen_slot_info = 3}
      const int k = m.kind - 2;
      const int in = vm_info_inner(k, m.f1, m.body);
      *p++ = 0x2a; p = wire_put_varint(p, (unsigned long long)vm_info_body(k, m.f0, m.f1, m.body));
      p = wire_put_int32(p, 1, m.f0);
      *p++ = k == 1 ? 0x12 : 0x1a; p = wire_put_varint(p, (unsigned long long)in);
      if (k == 1) { p = wire_put_int32(p, 1, m.f1); *p++ = 0x12; }   // vote_round, vote_value
      else *p++ = 0x0a;                                              // value
      p = wire_put_varint(p, (unsigned long long)m.body);
      int vlen = 0;
      if (m.noop) { *p++ = 0x12; *p++ = 0x00; }                      // CommandOrNoop{noop {}}
      else vlen = m.body;
      if (k == 2) { p[vlen] = 0x10; p[vlen + 1] = (uint8_t)m.f1; }   // is_revocation, after the value
      *gsrc = m.src; *glen = vlen;
    }
    return p;
  }
};

// message i starts at its head record
__global__ void vm_p1a_offsets_kernel(VmP1aParams P, const int32_t* rec_offs, int32_t total_recs, int32_t* offsets) {
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i < P.n) offsets[i] = rec_offs[(long long)i + P.cnt[i]];
  if (i == P.n) offsets[i] = rec_offs[total_recs];
}

// fpx_vm_entries: {kind, round, vote_round, value, is_revocation} of server `server` at slots [first, first + count)
__global__ void vm_entries_kernel(Geometry g, const unsigned long long* votes, const unsigned long long* raise,
                                  int server, int first, int count, int32_t* out) {
  const int k = blockIdx.x * 256 + threadIdx.x;
  if (k >= count) return;
  const int l = local_slot(g, first + k);
  const size_t ri = (size_t)l * g.voters + server;
  const VmEntry en = vm_entry(votes[cell_index(g, l, server)], raise, ri);
  int32_t* o = out + (size_t)k * 5;
  o[0] = en.kind; o[1] = en.round; o[2] = en.vote_round; o[3] = en.value; o[4] = en.revocation;
}

}  // namespace fpx
