// fpx_wire.cuh -- wire codec of the hot messages: scalapb / protobuf proto2 bytes <-> records.
//
// The reference spends most of a handler's time parsing the inbound protobuf and serialising
// the reply (SURVEY 8(a), "where the time goes"; every *InboundSerializer is ProtoSerializer,
// S/ProtoSerializer.scala:3-11).  The shapes are all-int32 plus one opaque value
// (S/multipaxos/MultiPaxos.proto: Phase2a :273-280, Phase2b :282-290, Chosen :292-298, Nack
// :455-460, LeaderInbound.nack = 6 :525-539, ProxyLeaderInbound :541-549, AcceptorInbound
// :551-561, ReplicaInbound.chosen = 1 :563-576), so a batch of received byte strings is decoded
// one thread per message and replies are encoded size -> scan -> emit, all HBM-bound byte work:
//   decode  the CTA stages its messages' contiguous byte span in shared memory with 128-bit
//           loads and parses from there (falls back to global loads for spans > kWireStage,
//           i.e. Phase2a batches, whose value bytes are skipped by length, not read);
//   encode  each CTA serialises 1024 replies into shared memory at the output's alignment
//           phase and copies the span out with 128-bit stores.
// Vanilla Mencius (S/vanillamencius/VanillaMencius.proto: ServerInbound :227-241, Phase2a :154-162,
// Skip :164-172, Phase2b :174-181, Chosen :183-190, Phase2Nack :209-215) goes through the same
// kernels: one more inbound of the decoder, Skip through the small-record encoder, and the reply
// stream, Chosen and Phase2a through the value-gathering one.
// Compartmentalized Mencius' replica (S/mencius/Mencius.proto: ReplicaInbound :363-371, Chosen :189-195,
// ChosenNoopRange :197-203) is the decoder's sixth inbound; its Phase2bNoopRange (:178-187), ChosenNoopRange and
// LeaderInbound.nack = 7 (:322-337) go through the small-record encoder.
// Parsing rules restated from the published proto2 wire format (DESIGN.md, wire codec): base-128
// varints of at most 10 bytes, int32 = low 32 bits, unknown fields skipped by wire type, a known
// number with another wire type is unknown, oneof = last member on the wire, a missing
// `required` field or any malformed byte fails the message (FPX_ERR_WIRE + its index).
#pragma once
#include "fpx_common.cuh"
#include "fpx_epaxos.cuh"
#include "fpx_scan.cuh"

namespace fpx {

constexpr int kWireStage = 24 * 1024;     // bytes of one CTA's message span staged in shared memory
constexpr int kWireDecThreads = 256;
constexpr int kWireEncPer = 4;            // replies per thread of the encoders
constexpr int kWireEncThreads = 256;
constexpr int kWireEncTile = kWireEncPer * kWireEncThreads;
constexpr int kWireMaxP2b = 46, kWireMaxNack = 13, kWireMaxP2bRange = 57, kWireMaxChosenRange = 24;

// Byte reader over one message.  kShared: positions index the CTA's staged window in shared memory
// (explicit ld.shared: a generic pointer would cost a generic load per byte); else they are offsets
// from the batch buffer in global memory.  All positions are 32-bit (the batch is < 2^31 bytes).
template <bool kShared>
struct WireReader {
  uint32_t sbase;            // shared-window address of window byte 0
  const uint8_t* g;          // batch buffer
  uint32_t p, end;
  bool ok;
  __device__ __forceinline__ uint32_t byte(uint32_t pos) const {
    if (kShared) {
      uint32_t v;
      asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(sbase + pos));
      return v;
    }
    return __ldg(g + pos);
  }
  __device__ __forceinline__ bool done() const { return p >= end; }
  // low 32 bits of a varint of at most 10 bytes; *hi_nonzero: bits 32.. were set (tags / lengths reject that)
  __device__ __forceinline__ uint32_t varint32(bool* hi_nonzero) {
    // one-byte varints (every tag, length and small field of the hot messages) without the loop
    if (p < end) {
      const uint32_t b0 = byte(p);
      if (b0 < 0x80u) { ++p; *hi_nonzero = false; return b0; }
    }
    uint32_t v = 0;
    bool hi = false;
#pragma unroll 1
    for (int i = 0; i < 10; ++i) {
      if (p >= end) { ok = false; return 0; }
      const uint32_t b = byte(p++);
      if (i < 4) v |= (b & 0x7f) << (7 * i);
      else if (i == 4) { v |= (b & 0x0f) << 28; hi |= (b & 0x70) != 0; }
      else hi |= (b & 0x7f) != 0;
      if (!(b & 0x80)) { *hi_nonzero = hi; return v; }
    }
    ok = false;                                  // malformed varint: more than 10 bytes
    return 0;
  }
  __device__ __forceinline__ uint32_t int32() { bool hi; return varint32(&hi); }      // (int) readRawVarint64
  // a tag: field number 1 .. 2^29-1 in bits 3.., i.e. any non-zero-field 32-bit value
  __device__ __forceinline__ uint32_t tag() {
    bool hi = false;
    uint32_t v = varint32(&hi);
    if (hi || (v >> 3) == 0) ok = false;
    return v;
  }
  // a length: anything >= 2^31 is longer than the batch
  __device__ __forceinline__ uint32_t small() {
    bool hi = false;
    uint32_t v = varint32(&hi);
    if (hi || (v >> 31)) ok = false;
    return v;
  }
  __device__ __forceinline__ bool skip(int wt) {
    if (wt == 0) { int32(); return ok; }
    if (wt == 1) { if (end - p < 8u) return ok = false; p += 8; return true; }
    if (wt == 5) { if (end - p < 4u) return ok = false; p += 4; return true; }
    if (wt == 2) {
      uint32_t n = small();
      if (!ok || end - p < n) return ok = false;
      p += n;
      return true;
    }
    return ok = false;
  }
};

// A oneof member on the path = n leading required int32 fields (numbered 1..n), plus for some members one
// nested value (a length-delimited field that is located, not parsed) and one required bool.
//   inbound 0  multipaxos ProxyLeaderInbound (MultiPaxos.proto:541-549)  phase2a = 1, phase2b = 2
//   inbound 1  multipaxos AcceptorInbound    (:551-561)                  phase2a = 2
//   inbound 2  mencius ProxyLeaderInbound    (Mencius.proto:339-350)     phase2a = 2, phase2a_noop_range = 3,
//                                                                        phase2b = 4, phase2b_noop_range = 5
//   inbound 3  mencius AcceptorInbound       (:352-361)                  phase2a = 2, phase2a_noop_range = 3
//   inbound 4  vanillamencius ServerInbound  (VanillaMencius.proto:227-241)  client_request = 1, phase2a = 4,
//                                            phase2b = 5, skip = 6, chosen = 7, phase2_nack = 9 (of 9 members)
//   inbound 5  mencius ReplicaInbound        (Mencius.proto:363-371)     chosen = 1, chosen_noop_range = 2
enum WireMember { kWmOpaque = 0, kWmP2a, kWmP2b4, kWmRange3, kWmMenciusP2b, kWmRangeVote5, kWmVmRequest, kWmVmP2a,
                  kWmVmChosen, kWmVmNack, kWmMrChosen, kWmRange2 };
// the decoder's instantiations: inbounds 0-3 (chosen at run time), 4, 5
enum { kWireInPath = 0, kWireInVm = 1, kWireInMenciusReplica = 2 };
template <int kIn>
__device__ __forceinline__ int wire_member(int inbound, int which) {
  constexpr bool kVm = kIn == kWireInVm;
  if (kIn == kWireInMenciusReplica)   // Chosen {slot, command_batch_or_noop}, ChosenNoopRange {start, end}
    return which == 1 ? kWmMrChosen : kWmRange2;
  if (kVm)   // vanilla Mencius: Phase2b {server_index, slot, round} has the mencius Phase2b's shape, Skip {server_index,
             // start, stop} that of a noop range
    return which == 1 ? kWmVmRequest : which == 4 ? kWmVmP2a : which == 5 ? kWmMenciusP2b : which == 6 ? kWmRange3
         : which == 7 ? kWmVmChosen : which == 9 ? kWmVmNack : kWmOpaque;
  if (inbound == 0) return which == 1 ? kWmP2a : which == 2 ? kWmP2b4 : kWmOpaque;
  if (inbound == 1) return which == 2 ? kWmP2a : kWmOpaque;
  if (inbound == 2)
    return which == 2 ? kWmP2a : which == 3 ? kWmRange3 : which == 4 ? kWmMenciusP2b : which == 5 ? kWmRangeVote5 : kWmOpaque;
  return which == 2 ? kWmP2a : which == 3 ? kWmRange3 : kWmOpaque;
}

// members of the inbound's oneof, numbered 1..count (MultiPaxos.proto:541-561, Mencius.proto:339-361; vanilla
// Mencius' ServerInbound, VanillaMencius.proto:227-241, has 9)
__device__ __forceinline__ int wire_member_count(int inbound) { return inbound == 0 ? 2 : inbound == 1 ? 4 : inbound == 2 ? 5 : 3; }

// Reader positions in, reader positions out (*value_pos: out->z is a position the caller rebases).
// *sender: the server field of a vanilla Mencius Phase2a, Phase2b or Skip (their field 1), else -1.
// kIn == kWireInVm: inbound 4 (the only one with a bool, a sender or a ClientRequest span: the other inbounds compile
// without them); kWireInMenciusReplica: inbound 5, {slot, 0, value_off, value_len} or {start, end, 0, 0}.
template <int kIn, bool kShared>
__device__ __forceinline__ bool wire_decode_one(int inbound, int lgroups, int agroups, WireReader<kShared> r, int* kind,
                                                int4* out, bool* value_pos, int* sender) {
  constexpr bool kVm = kIn == kWireInVm, kMr = kIn == kWireInMenciusReplica;
  int which = 0;
  uint32_t blo = 0, bhi = 0;
  while (!r.done()) {
    const uint32_t tag = r.tag();
    if (!r.ok) return false;
    const int wt = (int)(tag & 7);
    if (wt == 2) {
      const uint32_t n = r.small();
      if (!r.ok || r.end - r.p < n) return false;
      // oneof: the last member wins; a field number the message does not declare is an unknown field: skipped,
      // the earlier member stays (scalapb parseFrom)
      if ((tag >> 3) <= (uint32_t)(kVm ? 9 : kMr ? 2 : wire_member_count(inbound))) { which = (int)(tag >> 3); blo = r.p; bhi = r.p + n; }
      r.p += n;
    } else if (!r.skip(wt)) {
      return false;
    }
  }
  *kind = which;
  *out = make_int4(0, 0, 0, 0);
  *value_pos = false;
  *sender = -1;
  if (which == 0) return true;
  const int mk = wire_member<kIn>(inbound, which);
  if (mk == kWmOpaque) {
    *out = make_int4(0, 0, (int)blo, (int)(bhi - blo));
    *value_pos = true;
    return true;
  }
  const int n_ints = kMr ? (mk == kWmMrChosen ? 1 : 2)
                   : kVm ? (mk == kWmVmRequest ? 0 : mk == kWmVmChosen ? 1 : mk == kWmVmNack ? 2 : 3)
                         : (mk == kWmP2a ? 2 : mk == kWmP2b4 ? 4 : mk == kWmRangeVote5 ? 5 : 3);
  // the value's field number (0: none) and the required bool's (Chosen.isRevocation)
  const int vfield = kMr ? (mk == kWmMrChosen ? 2 : 0)
                   : kVm ? (mk == kWmVmP2a ? 4 : mk == kWmVmChosen ? 2 : mk == kWmVmRequest ? 1 : 0) : (mk == kWmP2a ? 3 : 0);
  const int bfield = kVm && mk == kWmVmChosen ? 3 : 0;
  WireReader<kShared> b = r;
  b.p = blo; b.end = bhi; b.ok = true;
  int v0 = 0, v1 = 0, v2 = 0, v3 = 0, v4 = 0;
  unsigned have = 0;
  uint32_t off = 0, len = 0;
  bool have_value = false, have_bool = false, bval = false;
  while (!b.done()) {
    const uint32_t tpos = b.p;
    const uint32_t tag = b.tag();
    if (!b.ok) return false;
    const int f = (int)(tag >> 3), wt = (int)(tag & 7);
    if (wt == 0 && f >= 1 && f <= n_ints) {
      const int v = (int)b.int32();
      if (!b.ok) return false;
      if (f == 1) v0 = v; else if (f == 2) v1 = v; else if (f == 3) v2 = v; else if (f == 4) v3 = v; else v4 = v;
      have |= 1u << (f - 1);
    } else if (kVm && wt == 0 && f == bfield) {
      bool hi = false;
      const uint32_t v = b.varint32(&hi);                        // readBool: the whole varint != 0
      if (!b.ok) return false;
      bval = v != 0 || hi; have_bool = true;
    } else if (wt == 2 && f == vfield) {
      const uint32_t n = b.small();
      if (!b.ok || b.end - b.p < n || have_value) return false;
      // the value bytes are not read; ClientRequest's span is the whole `command` field, tag and length
      // included: those bytes are CommandOrNoop().withCommand(command), both carry Command as field 1
      off = kVm && mk == kWmVmRequest ? tpos : b.p; len = b.p + n - off; have_value = true; b.p += n;
    } else if (!b.skip(wt)) {
      return false;
    }
  }
  // "Message missing required fields."
  if (have != (1u << n_ints) - 1u || (vfield && !have_value) || (bfield && !have_bool)) return false;
  if (kMr) {
    if (mk == kWmMrChosen) { *out = make_int4(v0, 0, (int)off, (int)len); *value_pos = true; }
    else *out = make_int4(v0, v1, 0, 0);
    return true;
  }
  if (kVm) {
    if (mk == kWmVmP2a || mk == kWmMenciusP2b || mk == kWmRange3) *sender = v0;
    if (mk == kWmVmP2a) { *out = make_int4(v1, v2, (int)off, (int)len); *value_pos = true; return true; }
    if (mk == kWmVmChosen) { *out = make_int4(v0, bval ? 1 : 0, (int)off, (int)len); *value_pos = true; return true; }
    if (mk == kWmVmRequest) { *out = make_int4(0, 0, (int)off, (int)len); *value_pos = true; return true; }
    if (mk == kWmVmNack) { *out = make_int4(v0, v1, 0, 0); return true; }
  }
  if (mk == kWmP2a) { *out = make_int4(v0, v1, (int)off, (int)len); *value_pos = true; }
  else if (mk == kWmP2b4) *out = make_int4(v0, v1, v2, v3);
  else if (mk == kWmRange3) *out = make_int4(v0, v1, v2, 0);               // {slot_start, slot_end, round, -}
  else if (mk == kWmMenciusP2b) *out = make_int4(0, v0, v1, v2);           // an fpx_p2b; the group follows from the slot
  else {                                                                    // Phase2bNoopRange -> an fpx_p2b_range
    int dst = -1;
    if (v0 >= 0 && v0 < agroups && v1 >= 0 && v1 < 0x10000 && lgroups > 0)
      dst = ((((v2 % lgroups) + lgroups) % lgroups) * agroups + v0) << 16 | v1;
    *out = make_int4(dst, v2, v3, v4);
  }
  return true;
}

struct WireDecodeParams {
  const uint8_t* bytes;     // 16-byte aligned
  const int32_t* offs;      // n + 1
  int32_t n;
  int32_t inbound;
  int32_t lgroups, agroups;   // mencius geometry (Phase2bNoopRange's dst)
  int32_t* kind;
  int4* out;
  int32_t* sender;          // vanilla Mencius only (else null): the message's server field, -1 if none
  DevStatus* st;
  // mencius ReplicaInbound only: out holds fpx_mencius_chosen rows, values[i] the Chosen value's {off, len}
  int32_t value_id_base;
  int2* values;
};

// The byte span of a decoder CTA's messages [m0, m1): staged in s_buf (kWireStage + 32 bytes) when it fits,
// window byte 0 = buffer byte `base`.  Every thread of the CTA calls it (it ends with __syncthreads).
struct WireSpan {
  long long lo, hi, base;
  bool sane, staged;
};
__device__ __forceinline__ WireSpan wire_stage_span(const uint8_t* bytes, const int32_t* offs, int n, int m0, int m1,
                                                    uint8_t* s_buf) {
  WireSpan w;
  w.lo = offs[m0]; w.hi = offs[m1];
  const long long total = offs[n];
  w.base = w.lo & ~15ll;
  w.sane = w.lo >= 0 && w.lo <= w.hi && w.hi <= total;   // garbage offsets never turn into wild reads
  w.staged = w.sane && w.hi - w.base <= kWireStage;
  if (w.staged) {
    // 128-bit loads while the chunk lies inside the buffer, bytes for the last partial chunk
    for (long long k = (long long)threadIdx.x * 16; w.base + k < w.hi; k += (long long)kWireDecThreads * 16) {
      if (w.base + k + 16 <= (total & ~15ll)) {
        *(uint4*)(s_buf + k) = __ldg((const uint4*)(bytes + w.base + k));
      } else {
        for (int j = 0; j < 16 && w.base + k + j < total; ++j) s_buf[k + j] = __ldg(bytes + w.base + k + j);
      }
    }
  }
  __syncthreads();
  return w;
}
// Message [a, b) of the span: false when it lies outside (offsets must be monotone), else f(reader, rebase) once, on
// the staged window with rebase = w.base (window -> buffer offsets) or on global memory with rebase = 0.
template <class F>
__device__ __forceinline__ bool wire_read(const WireSpan& w, const uint8_t* s_buf, const uint8_t* bytes, long long a,
                                          long long b, F&& f) {
  if (!(w.sane && a <= b && a >= w.lo && b <= w.hi)) return false;
  if (w.staged)
    f(WireReader<true>{(uint32_t)__cvta_generic_to_shared(s_buf), nullptr, (uint32_t)(a - w.base), (uint32_t)(b - w.base), true},
      (uint32_t)w.base);
  else
    f(WireReader<false>{0u, bytes, (uint32_t)a, (uint32_t)b, true}, 0u);
  return true;
}

// kIn: kWireInPath (inbounds 0-3), kWireInVm (the vanilla Mencius inbound 4: the other instantiations compile without
// its bool, sender and ClientRequest span) or kWireInMenciusReplica (inbound 5: dense fpx_mencius_chosen rows)
template <int kIn>
__global__ void __launch_bounds__(kWireDecThreads) wire_decode_kernel(WireDecodeParams P) {
  constexpr bool kVm = kIn == kWireInVm, kMr = kIn == kWireInMenciusReplica;
  const int inbound = kVm ? 4 : kMr ? 5 : P.inbound;
  __shared__ __align__(16) uint8_t s_buf[kWireStage + 32];
  const int m0 = blockIdx.x * kWireDecThreads;
  const int m1 = min(P.n, m0 + kWireDecThreads);
  const WireSpan w = wire_stage_span(P.bytes, P.offs, P.n, m0, m1, s_buf);
  const int i = m0 + threadIdx.x;
  if (i >= m1) return;
  int kind = 0, sender = -1;
  int4 rec = make_int4(0, 0, 0, 0);
  bool ok = false;
  wire_read(w, s_buf, P.bytes, P.offs[i], P.offs[i + 1], [&](auto r, uint32_t rebase) {
    bool value_pos = false;
    ok = wire_decode_one<kIn>(inbound, P.lgroups, P.agroups, r, &kind, &rec, &value_pos, &sender);
    if (ok && value_pos) rec.z += (int)rebase;
  });
  if (!ok) report_error(P.st, FPX_ERR_WIRE, i);
  if (kMr) {
    // Chosen(slot, v) -> {slot, slot + 1, value_id_base + i}, ChosenNoopRange(s, e) -> {s, e, Noop}; no member (or a
    // failed message) -> a row that covers no slot
    int4 row = make_int4(0, 0, FPX_VALUE_NOOP, 0);
    int2 val = make_int2(0, 0);
    if (ok && kind == 1) {
      row = make_int4(rec.x, (int)((uint32_t)rec.x + 1u), P.value_id_base + i, 0);
      val = make_int2(rec.z, rec.w);
    } else if (ok && kind == 2) {
      row = make_int4(rec.x, rec.y, FPX_VALUE_NOOP, 0);
    }
    P.kind[i] = ok ? kind : 0;
    P.out[i] = row;
    P.values[i] = val;
    return;
  }
  P.kind[i] = kind;
  P.out[i] = rec;
  if (kVm) P.sender[i] = ok ? sender : -1;
}

// ---------------------------------------------------------------------------
// EPaxos ReplicaInbound (S/epaxos/EPaxos.proto:220-235): one thread per message as above, with a nested parser.
// The members' fields are nested messages (Instance :35-41, Ballot :46-52, CommandOrNoop :80-88 over Command
// :61-78, InstancePrefixSetProto :97-103 over IntPrefixSetProto) or int32s.  Parsed as protobuf-java's
// mergeFrom builds the message: a member given again merges into the one before it (a nested Instance / Ballot
// too: the have-bits accumulate, a later scalar wins), another member starts afresh, and `required` is checked on
// the message that results.  Every member body on the wire is parsed, so malformed bytes anywhere fail.
// ---------------------------------------------------------------------------
// decoded row (12 + n int32, include/fpx.h fpx_epaxos_wire_decode)
enum { EW_IREP = 0, EW_INUM, EW_BORD, EW_BREP, EW_REPLICA, EW_VBORD, EW_VBREP, EW_STATUS, EW_VALUE, EW_SEQ, EW_FLAGS,
       EW_OVERFLOW, EW_DEPS };
// what a member's field is: nested messages first (wire type 2), then the int32 fields (wire type 0)
enum { kEfNone = 0, kEfInstance, kEfBallot, kEfVote, kEfValue, kEfDeps, kEfReplica, kEfStatus, kEfSeq };
// the roles of fields 1..8 of member `which`, a nibble each (field 1 lowest)
__device__ __forceinline__ uint32_t ep_wire_roles(int which) {
  switch (which) {
    case 1: return 0x4u;              // ClientRequest{command}: the value
    case 2:                           // PreAccept / Accept {instance, ballot, command_or_noop, sequence_number,
    case 4: return 0x58421u;          //   dependencies}
    case 3: return 0x58621u;          // PreAcceptOk {instance, ballot, replica_index, sequence_number, dependencies}
    case 5: return 0x6000210u;        // AcceptOk {instance = 2, ballot = 3, replica_index = 7}
    case 6: return 0x5841u;           // Commit {instance, command_or_noop, sequence_number, dependencies}
    case 7:                           // Prepare / Nack {instance, ballot (largest_ballot)}
    case 9: return 0x21u;
    case 8: return 0x58473612u;       // PrepareOk {ballot, instance, replica_index, vote_ballot, status,
                                      //   [command_or_noop, sequence_number, dependencies]}
    default: return 0u;
  }
}
// have-bits of the nested messages (EpWireMsg::sub)
enum { kSubInstance = 0x3, kSubBallot = 0xc, kSubVote = 0x30, kSubNumReplicas = 0x40 };

struct EpWireMsg {
  int irep, inum, bord, brep, vord, vrep, replica, status, seq;
  unsigned have;          // fields of the member given (bit f - 1)
  unsigned sub;           // kSub*
  int num_replicas, dcount, overflow;
  uint32_t voff, vlen;    // the value's span (reader positions)
  bool noop;
};
__device__ __forceinline__ EpWireMsg ep_wire_fresh() {
  EpWireMsg m;
  m.irep = m.inum = m.bord = m.brep = m.vord = m.vrep = -1;
  m.replica = m.status = m.seq = 0;
  m.have = m.sub = 0;
  m.num_replicas = m.dcount = m.overflow = 0;
  m.voff = m.vlen = 0;
  m.noop = false;
  return m;
}

// A message whose known fields are all skipped: bit f - 1 of *have for field f <= 4 given with its wire type
// (wt2: the length-delimited ones, wt0: the varints).  Command (wt2 0x9, wt0 0x6) and Noop (none).
template <bool kS>
__device__ __forceinline__ bool ep_wire_fields(WireReader<kS> b, unsigned wt2, unsigned wt0, unsigned* have) {
  while (!b.done()) {
    const uint32_t tag = b.tag();
    if (!b.ok) return false;
    const int f = (int)(tag >> 3), wt = (int)(tag & 7);
    if (f <= 4 && (((wt == 2 ? wt2 : wt == 0 ? wt0 : 0u) >> (f - 1)) & 1u)) *have |= 1u << (f - 1);
    if (!b.skip(wt)) return false;
  }
  return true;
}
// Instance / Ballot: two int32 fields, merged into (*x, *y) and have-bits << shift
template <bool kS>
__device__ __forceinline__ bool ep_wire_pair(WireReader<kS> b, int* x, int* y, unsigned* have, int shift) {
  while (!b.done()) {
    const uint32_t tag = b.tag();
    if (!b.ok) return false;
    const int f = (int)(tag >> 3), wt = (int)(tag & 7);
    if (wt == 0 && (f == 1 || f == 2)) {
      const int v = (int)b.int32();
      if (!b.ok) return false;
      if (f == 1) *x = v; else *y = v;
      *have |= 1u << (shift + f - 1);
    } else if (!b.skip(wt)) {
      return false;
    }
  }
  return true;
}
// CommandOrNoop {command = 1, noop = 2}: the last member wins, a Command given again merges
template <bool kS>
__device__ __forceinline__ bool ep_wire_value(WireReader<kS> b, bool* noop) {
  int which = 0;
  unsigned cmd = 0;
  while (!b.done()) {
    const uint32_t tag = b.tag();
    if (!b.ok) return false;
    const int f = (int)(tag >> 3), wt = (int)(tag & 7);
    if (wt == 2 && (f == 1 || f == 2)) {
      const uint32_t n = b.small();
      if (!b.ok || b.end - b.p < n) return false;
      WireReader<kS> s = b;
      s.end = b.p + n;
      if (f == 1 && which != 1) cmd = 0;
      unsigned none = 0;
      if (!(f == 1 ? ep_wire_fields(s, 0x9u, 0x6u, &cmd) : ep_wire_fields(s, 0u, 0u, &none))) return false;
      which = f;
      b.p += n;
    } else if (!b.skip(wt)) {
      return false;
    }
  }
  *noop = which == 2;
  return which != 1 || cmd == 0xfu;        // Command's four fields are required
}
// IntPrefixSetProto {watermark = 1, repeated value = 2}: `value` packed or not; *values counts them
template <bool kS>
__device__ __forceinline__ bool ep_wire_prefix_set(WireReader<kS> b, int* watermark, int* values) {
  bool have = false;
  while (!b.done()) {
    const uint32_t tag = b.tag();
    if (!b.ok) return false;
    const int f = (int)(tag >> 3), wt = (int)(tag & 7);
    if (f == 1 && wt == 0) {
      *watermark = (int)b.int32();
      have = true;
    } else if (f == 2 && wt == 0) {
      b.int32();
      ++*values;
    } else if (f == 2 && wt == 2) {
      const uint32_t n = b.small();
      if (!b.ok || b.end - b.p < n) return false;
      WireReader<kS> s = b;
      s.end = b.p + n;
      while (!s.done()) {
        s.int32();
        if (!s.ok) return false;
        ++*values;
      }
      b.p = s.p;
    } else {
      b.skip(wt);
    }
    if (!b.ok) return false;
  }
  return have;
}
// InstancePrefixSetProto {numReplicas = 1, repeated int_prefix_set = 2}: entry k's watermark -> deps[k] (k < n)
template <bool kS>
__device__ __forceinline__ bool ep_wire_deps(WireReader<kS> b, EpWireMsg& m, int32_t* deps, int n) {
  while (!b.done()) {
    const uint32_t tag = b.tag();
    if (!b.ok) return false;
    const int f = (int)(tag >> 3), wt = (int)(tag & 7);
    if (f == 1 && wt == 0) {
      m.num_replicas = (int)b.int32();
      if (!b.ok) return false;
      m.sub |= kSubNumReplicas;
    } else if (f == 2 && wt == 2) {
      const uint32_t len = b.small();
      if (!b.ok || b.end - b.p < len) return false;
      WireReader<kS> s = b;
      s.end = b.p + len;
      int wm = 0;
      if (!ep_wire_prefix_set(s, &wm, &m.overflow)) return false;
      if (m.dcount < n) deps[m.dcount] = wm;
      ++m.dcount;
      b.p += len;
    } else if (!b.skip(wt)) {
      return false;
    }
  }
  return true;
}
// one body of member `which`, merged into m
template <bool kS>
__device__ __forceinline__ bool ep_wire_member(WireReader<kS> b, int which, int n, EpWireMsg& m, int32_t* deps) {
  const uint32_t roles = ep_wire_roles(which);
  while (!b.done()) {
    const uint32_t tpos = b.p;
    const uint32_t tag = b.tag();
    if (!b.ok) return false;
    const int f = (int)(tag >> 3), wt = (int)(tag & 7);
    const int role = f <= 8 ? (int)((roles >> (4 * (f - 1))) & 15u) : kEfNone;
    if (role == kEfNone || wt != (role >= kEfReplica ? 0 : 2)) {    // unknown, or a known number with another type
      if (!b.skip(wt)) return false;
      continue;
    }
    const unsigned bit = 1u << (f - 1);
    if (role >= kEfReplica) {
      const int v = (int)b.int32();
      if (!b.ok) return false;
      if (role == kEfReplica) m.replica = v; else if (role == kEfStatus) m.status = v; else m.seq = v;
      m.have |= bit;
      continue;
    }
    const uint32_t len = b.small();
    if (!b.ok || b.end - b.p < len) return false;
    WireReader<kS> s = b;
    s.end = b.p + len;
    bool ok;
    if (role == kEfInstance) {
      ok = ep_wire_pair(s, &m.irep, &m.inum, &m.sub, 0);
    } else if (role == kEfBallot) {
      ok = ep_wire_pair(s, &m.bord, &m.brep, &m.sub, 2);
    } else if (role == kEfVote) {
      ok = ep_wire_pair(s, &m.vord, &m.vrep, &m.sub, 4);
    } else if (role == kEfDeps) {
      ok = ep_wire_deps(s, m, deps, n);
    } else if (m.have & bit) {
      ok = false;                     // a second command_or_noop (or ClientRequest.command) would merge: unsupported
    } else if (which == 1) {          // ClientRequest: the whole `command` field = CommandOrNoop().withCommand(command)
      unsigned cmd = 0;
      ok = ep_wire_fields(s, 0x9u, 0x6u, &cmd) && cmd == 0xfu;
      m.voff = tpos; m.vlen = s.end - tpos; m.noop = false;
    } else {
      ok = ep_wire_value(s, &m.noop);
      m.voff = s.p; m.vlen = len;
    }
    if (!ok) return false;
    m.have |= bit;
    b.p += len;
  }
  return true;
}
// One ReplicaInbound -> FPX_OK / FPX_ERR_WIRE / FPX_ERR_UNSUPPORTED (a set of another size, an unknown status)
template <bool kS>
__device__ __forceinline__ int ep_wire_decode_one(WireReader<kS> r, int n, int* kind, EpWireMsg& m, int32_t* deps) {
  int which = 0;
  while (!r.done()) {
    const uint32_t tag = r.tag();
    if (!r.ok) return FPX_ERR_WIRE;
    const int wt = (int)(tag & 7);
    if (wt == 2) {
      const uint32_t len = r.small();
      if (!r.ok || r.end - r.p < len) return FPX_ERR_WIRE;
      const int f = (int)(tag >> 3);
      if (f <= 9) {
        if (f != which) { m = ep_wire_fresh(); which = f; }
        WireReader<kS> s = r;
        s.end = r.p + len;
        if (!ep_wire_member(s, which, n, m, deps)) return FPX_ERR_WIRE;
      }
      r.p += len;
    } else if (!r.skip(wt)) {
      return FPX_ERR_WIRE;
    }
  }
  *kind = which;
  if (which == 0) return FPX_OK;
  // "Message missing required fields": the member's, PrepareOk's optional triple aside, and the nested ones
  const uint32_t roles = ep_wire_roles(which);
  unsigned need = 0, sub = 0;
  for (int f = 1; f <= 8; ++f) {
    const int role = (int)((roles >> (4 * (f - 1))) & 15u);
    if (role == kEfNone) continue;
    if (!(which == 8 && f >= 6)) need |= 1u << (f - 1);
    if (!(m.have >> (f - 1) & 1u)) continue;
    sub |= role == kEfInstance ? kSubInstance : role == kEfBallot ? kSubBallot : role == kEfVote ? kSubVote
         : role == kEfDeps ? kSubNumReplicas : 0u;
  }
  if ((m.have & need) != need || (m.sub & sub) != sub) return FPX_ERR_WIRE;
  // parsed, but not a set or status the engine holds
  if ((sub & kSubNumReplicas) && (m.num_replicas != n || m.dcount != n)) return FPX_ERR_UNSUPPORTED;
  if (which == 8 && (uint32_t)m.status > 2u) return FPX_ERR_UNSUPPORTED;
  return FPX_OK;
}

struct EpWireDecodeParams {
  const uint8_t* bytes;     // 16-byte aligned
  const int32_t* offs;      // n + 1
  int32_t n;
  int32_t replicas;
  int32_t value_id_base;
  int32_t* kind;
  int32_t* rows;            // n * (12 + replicas)
  int2* values;             // n {off, len}
  DevStatus* st;
  uint32_t* refused;        // the EPaxos handle's refusal word (EpState::refused)
  uint32_t tag;             // this call's batch tag
};

// A message that fails refuses the call like a handler's validation pass: the handle's calls queued behind it
// apply nothing until the status is collected.  Like those passes, it returns at once behind an earlier refusal.
__global__ void __launch_bounds__(kWireDecThreads) ep_wire_decode_kernel(EpWireDecodeParams P) {
  {
    const uint32_t rf = __ldcg(P.refused);
    if (rf != 0 && rf != P.tag) return;
  }
  __shared__ __align__(16) uint8_t s_buf[kWireStage + 32];
  const int m0 = blockIdx.x * kWireDecThreads;
  const int m1 = min(P.n, m0 + kWireDecThreads);
  const WireSpan w = wire_stage_span(P.bytes, P.offs, P.n, m0, m1, s_buf);
  const int i = m0 + threadIdx.x;
  if (i >= m1) return;
  const int n = P.replicas;
  int32_t* row = P.rows + (long long)i * (EW_DEPS + n);
  EpWireMsg m = ep_wire_fresh();
  int kind = 0, code = FPX_ERR_WIRE;
  wire_read(w, s_buf, P.bytes, P.offs[i], P.offs[i + 1], [&](auto r, uint32_t rebase) {
    code = ep_wire_decode_one(r, n, &kind, m, row + EW_DEPS);
    m.voff += rebase;
  });
  if (code != FPX_OK) {
    report_error(P.st, code, i);
    *(volatile uint32_t*)P.refused = P.tag;
    kind = 0;
    m = ep_wire_fresh();
  }
  const uint32_t roles = ep_wire_roles(kind);
  bool value = false, deps = false;
  for (int f = 1; f <= 8; ++f) {
    if (!(m.have >> (f - 1) & 1u)) continue;
    const int role = (int)((roles >> (4 * (f - 1))) & 15u);
    value |= role == kEfValue;
    deps |= role == kEfDeps;
  }
  P.kind[i] = kind;
  row[EW_IREP] = m.irep; row[EW_INUM] = m.inum; row[EW_BORD] = m.bord; row[EW_BREP] = m.brep;
  row[EW_REPLICA] = m.replica; row[EW_VBORD] = m.vord; row[EW_VBREP] = m.vrep; row[EW_STATUS] = m.status;
  row[EW_VALUE] = !value ? -1 : m.noop ? FPX_VALUE_NOOP : P.value_id_base + i;
  row[EW_SEQ] = m.seq;
  row[EW_FLAGS] = kind == 8 && (m.have & 0xe0u) == 0xe0u ? 1 : 0;      // PrepareOk's triple is there
  row[EW_OVERFLOW] = m.overflow;
  if (!deps)
    for (int k = 0; k < n; ++k) row[EW_DEPS + k] = 0;
  P.values[i] = value ? make_int2((int)m.voff, (int)m.vlen) : make_int2(0, 0);
}

// decoded rows -> the input rows of one handler call (the fpx_epaxos_* layouts); call = FPX_EP_CALL_*
__host__ __device__ constexpr int ep_wire_pack_kind(int call) {
  return call == 1 ? 2 : call == 2 ? 4 : call == 3 ? 3 : call == 4 ? 5 : call == 5 ? 6 : call == 6 ? 9 : call == 8 ? 7
       : call == 9 ? 8 : 0;
}
__host__ __device__ constexpr int ep_wire_pack_width(int call, int n) {
  return call == 1 ? 6 + 2 * n : call == 2 || call == 3 ? 6 + n : call == 4 ? 6 : call == 5 ? 4 + n : call == 9 ? 9 : 4;
}
struct EpWirePackParams {
  int32_t call, replicas;
  const int32_t* kind;        // [count], the batch's from `first` on
  const int32_t* rows;        // [count][12 + replicas]
  int32_t first, count;       // first: error indices are the batch's
  const int32_t* local_deps;  // [count][replicas] or null (zeros)
  int32_t* out;               // [count][ep_wire_pack_width]
  DevStatus* st;
  uint32_t* refused;
  uint32_t tag;
};
__global__ void __launch_bounds__(256) ep_wire_pack_kernel(EpWirePackParams P) {
  {
    const uint32_t rf = __ldcg(P.refused);
    if (rf != 0 && rf != P.tag) return;
  }
  const int j = blockIdx.x * 256 + threadIdx.x;
  if (j >= P.count) return;
  const int n = P.replicas, call = P.call;
  const int32_t* r = P.rows + (long long)j * (EW_DEPS + n);
  int32_t* o = P.out + (long long)j * ep_wire_pack_width(call, n);
  int code = FPX_OK;
  if (P.kind[j] != ep_wire_pack_kind(call)) code = FPX_ERR_INVALID_ARG;
  // sparse sets (overflow values) the handlers would read: fpx_epaxos_preaccept_sets' rule
  else if ((call == 1 || call == 2 || call == 3 || call == 5) && r[EW_OVERFLOW] > 0) code = FPX_ERR_UNSUPPORTED;
  if (code != FPX_OK) {
    report_error(P.st, code, (long long)P.first + j);
    *(volatile uint32_t*)P.refused = P.tag;
    return;
  }
  if (call == 5) {                                            // commit {rep, num, value_id, seq, deps}
    o[0] = r[EW_IREP]; o[1] = r[EW_INUM]; o[2] = r[EW_VALUE]; o[3] = r[EW_SEQ];
    for (int k = 0; k < n; ++k) o[4 + k] = r[EW_DEPS + k];
    return;
  }
  o[0] = r[EW_IREP]; o[1] = r[EW_INUM]; o[2] = r[EW_BORD]; o[3] = r[EW_BREP];
  if (call == 1 || call == 2) {                               // {.., value_id, seq, [local_deps,] deps}
    o[4] = r[EW_VALUE]; o[5] = r[EW_SEQ];
    int c = 6;
    if (call == 1) {
      for (int k = 0; k < n; ++k) o[6 + k] = P.local_deps ? P.local_deps[(long long)j * n + k] : 0;
      c += n;
    }
    for (int k = 0; k < n; ++k) o[c + k] = r[EW_DEPS + k];
  } else if (call == 3) {                                     // {.., from, seq, deps}
    o[4] = r[EW_REPLICA]; o[5] = r[EW_SEQ];
    for (int k = 0; k < n; ++k) o[6 + k] = r[EW_DEPS + k];
  } else if (call == 4) {                                     // {.., from, 0}
    o[4] = r[EW_REPLICA]; o[5] = 0;
  } else if (call == 9) {                                     // {.., from, vb_ord, vb_rep, status, value_id}
    o[4] = r[EW_REPLICA]; o[5] = r[EW_VBORD]; o[6] = r[EW_VBREP]; o[7] = r[EW_STATUS];
    o[8] = r[EW_FLAGS] & 1 ? r[EW_VALUE] : 0;                 // a NotSeen vote carries none: 0, as fpx_epaxos_prepare
  }
}

// ---------------------------------------------------------------------------
// encoders
// ---------------------------------------------------------------------------
__device__ __forceinline__ int wire_varint_size(unsigned long long v) {
  int n = 1;
  while (v >= 0x80) { v >>= 7; ++n; }
  return n;
}
__device__ __forceinline__ int wire_int32_size(int v) {   // negative int32 is sign-extended: 10 bytes
  // ceil(bits / 7) for bits = 1 .. 32 is ((bits + 6) * 37) >> 8
  return v < 0 ? 10 : ((38 - __clz(v | 1)) * 37) >> 8;
}
__device__ __forceinline__ uint8_t* wire_put_varint(uint8_t* p, unsigned long long v) {
  while (v >= 0x80) { *p++ = (uint8_t)(v | 0x80); v >>= 7; }
  *p++ = (uint8_t)v;
  return p;
}
__device__ __noinline__ uint8_t* wire_put_negative(uint8_t* p, int v) {   // sign-extended: ten bytes, rare
  return wire_put_varint(p, (unsigned long long)(long long)v);
}
__device__ __forceinline__ uint8_t* wire_put_int32(uint8_t* p, int field, int v) {
  *p++ = (uint8_t)(field << 3);
  if (v < 0) return wire_put_negative(p, v);
  // 1..5 bytes without a data-dependent loop: byte k is written iff the value has more than 7k bits
  const uint32_t u = (uint32_t)v;
  const int n = ((38 - __clz(v | 1)) * 37) >> 8;
  p[0] = (uint8_t)((u & 0x7f) | (n > 1 ? 0x80 : 0));
  if (n > 1) p[1] = (uint8_t)(((u >> 7) & 0x7f) | (n > 2 ? 0x80 : 0));
  if (n > 2) p[2] = (uint8_t)(((u >> 14) & 0x7f) | (n > 3 ? 0x80 : 0));
  if (n > 3) p[3] = (uint8_t)(((u >> 21) & 0x7f) | (n > 4 ? 0x80 : 0));
  if (n > 4) p[4] = (uint8_t)(u >> 28);
  return p + n;
}

// kWireVm*: vanilla Mencius ServerInbound (VanillaMencius.proto:227-241).  kWireVmReply is the dense reply
// stream of fpx_vm_phase2a (fpx_p2b {kind, server, slot, round|value}), one message per record by its kind.
// kWireMencius{Nack, P2bRange, ChosenRange}: compartmentalized Mencius (Mencius.proto) LeaderInbound.nack = 7,
// ProxyLeaderInbound.phase2b_noop_range = 5 and ReplicaInbound.chosen_noop_range = 2.  kWireMenciusPhase2a is
// kWirePhase2a under Mencius' ProxyLeaderInbound.phase2a = 2.
enum { kWirePhase2b = 0, kWireNack = 1, kWireChosen = 2, kWireMenciusPhase2b = 3, kWireVmReply = 4, kWireVmChosen = 5,
       kWireVmPhase2a = 6, kWireVmSkip = 7, kWireMenciusNack = 8, kWireMenciusP2bRange = 9, kWireMenciusChosenRange = 10,
       kWirePhase2a = 11, kWireMenciusPhase2a = 12 };
// the largest message of a small-record encoder (its shared-memory slot per record)
__host__ __device__ constexpr int wire_small_max(int kind) {
  return kind == kWireNack || kind == kWireMenciusNack ? kWireMaxNack : kind == kWireMenciusP2bRange ? kWireMaxP2bRange
       : kind == kWireMenciusChosenRange ? kWireMaxChosenRange : kWireMaxP2b;
}
// encoders whose messages carry a value from the arena: size -> scan -> wire_gather_emit_kernel
__host__ __device__ constexpr bool wire_gathers(int kind) {
  return kind == kWireChosen || kind == kWireVmReply || kind == kWireVmChosen || kind == kWireVmPhase2a ||
         kind == kWirePhase2a || kind == kWireMenciusPhase2a;
}

// What every encoder's params hold (as their member `enc`): n records in, n messages out.
struct WireEnc {
  int32_t n;
  uint8_t* out;               // 16-byte aligned
  int32_t out_capacity;
  int32_t* offs;              // n + 1
  uint32_t* tile_sum;         // [tiles] bytes per tile, then (after the scan) [tiles + 1] exclusive offsets
  const uint8_t* src;         // the gathered bytes: the value arena, or the request batch
  unsigned long long* err_word;
};

struct WireEncodeParams {
  WireEnc enc;
  const void* in;             // fpx_p2b (int4) | fpx_nack (int2) | fpx_chosen (int2) | fpx_p2a | fpx_vm_skip_rec
  // value-gathering encoders: the value bytes of value_id v are enc.src[value_offs[v] .. value_offs[v + 1])
  const int32_t* value_offs;
  int32_t num_values;
  int32_t servers;            // kWireVmPhase2a: sending_server = slot mod servers
  int32_t agroups;            // kWireMenciusP2bRange: acceptor_group_index = (dst >> 16) mod agroups
  // kWirePhase2a: value_id v is the span spans[v - span_base] = {off, len} of enc.src[0 .. span_bytes), for
  // v - span_base in [0, num_values); value_offs is not read
  const int2* spans;
  int32_t span_base, span_bytes;
};

// One message of a value-gathering encoder: outer oneof tag, int32 fields 1..nf, then (vfield != 0) the
// value under field vfield -- arena bytes, or a vanilla Mencius Noop -- then (revocation) the required
// `isRevocation` (field 3, `is_revocation`).  outer = 0: no bytes at all (a retired slot's Chosen, whose value the
// caller holds).
struct WireMsg {
  int outer, nf, vfield;
  int f0, f1, f2;
  int src, vlen;              // arena[src .. src + vlen); noop: CommandOrNoop{noop {}} = 12 00 instead
  bool noop, revocation, is_revocation;
};

// value_id v of a gathering encoder; Noop (FPX_VALUE_NOOP) where the shape has one, else out of range = bad
__device__ __forceinline__ bool wire_value(const WireEncodeParams& P, int v, bool noop_ok, WireMsg* m) {
  if (noop_ok && v == FPX_VALUE_NOOP) { m->noop = true; m->src = 0; m->vlen = 2; return true; }
  if ((uint32_t)v >= (uint32_t)P.num_values) return false;
  const int src = P.value_offs[v];
  const long long vlen = (long long)P.value_offs[v + 1] - src;
  if (vlen < 0) return false;
  m->src = src; m->vlen = (int)vlen;
  return true;
}

template <int KIND>
__device__ __forceinline__ WireMsg wire_msg(const WireEncodeParams& P, int i, bool* bad) {
  WireMsg m{0, 0, 0, 0, 0, 0, 0, 0, false, false, false};
  if (KIND == kWireChosen) {                        // ReplicaInbound{chosen = 1 {slot = 1, command_batch_or_noop = 2}}
    const int2 r = ((const int2*)P.in)[i];
    m.outer = 0x0a; m.nf = 1; m.f0 = r.x; m.vfield = 2;
    *bad = !wire_value(P, r.y, false, &m);
  } else if (KIND == kWireVmChosen) {               // ServerInbound{chosen = 7 {slot, command_or_noop, false}}
    const int2 r = ((const int2*)P.in)[i];
    m.outer = 0x3a; m.nf = 1; m.f0 = r.x; m.vfield = 2; m.revocation = true;
    *bad = !wire_value(P, r.y, true, &m);
  } else if (KIND == kWirePhase2a || KIND == kWireMenciusPhase2a) {
    // ProxyLeaderInbound{phase2a = 1 (Mencius 2) {slot, round, command_batch_or_noop}}
    const int4 r = ((const int4*)P.in)[i];
    m.outer = KIND == kWirePhase2a ? 0x0a : 0x12; m.nf = 2; m.f0 = r.x; m.f1 = r.y; m.vfield = 3;
    if (r.z == FPX_VALUE_NOOP) {
      m.noop = true; m.vlen = 2;
    } else {
      const uint32_t k = (uint32_t)r.z - (uint32_t)P.span_base;
      const int2 sp = k < (uint32_t)P.num_values ? P.spans[k] : make_int2(-1, -1);
      *bad = sp.x < 0 || sp.y < 0 || (long long)sp.x + sp.y > P.span_bytes;
      m.src = sp.x; m.vlen = sp.y;
    }
  } else if (KIND == kWireVmPhase2a) {              // ServerInbound{phase2a = 4 {sending_server, slot, round, value}}
    const int4 r = ((const int4*)P.in)[i];
    const int owner = r.x % P.servers;
    m.outer = 0x22; m.nf = 3; m.f0 = owner < 0 ? owner + P.servers : owner; m.f1 = r.x; m.f2 = r.y; m.vfield = 4;
    *bad = !wire_value(P, r.z, true, &m);
  } else {                                          // kWireVmReply
    const int4 r = ((const int4*)P.in)[i];
    if (r.x == FPX_VM_REPLY_PHASE2B) {              // phase2b = 5 {server_index, slot, round}
      m.outer = 0x2a; m.nf = 3; m.f0 = r.y; m.f1 = r.z; m.f2 = r.w;
    } else if (r.x == FPX_VM_REPLY_NACK) {          // phase2_nack = 9 {slot, round}
      m.outer = 0x4a; m.nf = 2; m.f0 = r.z; m.f1 = r.w;
    } else if (r.x == FPX_VM_REPLY_CHOSEN || r.x == FPX_VM_REPLY_CHOSEN_REVOCATION) {
      // chosen = 7 {slot, value in round, isRevocation}
      m.outer = 0x3a; m.nf = 1; m.f0 = r.z; m.vfield = 2; m.revocation = true;
      m.is_revocation = r.x == FPX_VM_REPLY_CHOSEN_REVOCATION;
      *bad = !wire_value(P, r.w, true, &m);
    } else if (r.x != FPX_VM_REPLY_CHOSEN_RETIRED) {
      *bad = true;
    }
  }
  return m;
}

__device__ __forceinline__ long long wire_msg_body(const WireMsg& m) {
  long long b = 0;
  if (m.nf > 0) b += 1 + wire_int32_size(m.f0);
  if (m.nf > 1) b += 1 + wire_int32_size(m.f1);
  if (m.nf > 2) b += 1 + wire_int32_size(m.f2);
  if (m.vfield) b += 1 + wire_varint_size((unsigned long long)m.vlen) + m.vlen;
  if (m.revocation) b += 2;
  return b;
}
__device__ __forceinline__ int wire_msg_size(const WireMsg& m) {
  if (!m.outer) return 0;
  const long long b = wire_msg_body(m);
  return (int)(1 + wire_varint_size((unsigned long long)b) + b);
}

template <int KIND>
__device__ __forceinline__ int wire_size_of(const WireEncodeParams& P, int i, int* code) {
  if (KIND == kWirePhase2b) {
    int4 r = ((const int4*)P.in)[i];
    // ProxyLeaderInbound{phase2b = 2}: 0x12, len (< 128: one byte), four int32 fields
    return 2 + 4 + wire_int32_size(r.x) + wire_int32_size(r.y) + wire_int32_size(r.z) + wire_int32_size(r.w);
  } else if (KIND == kWireMenciusPhase2b) {
    int4 r = ((const int4*)P.in)[i];
    // mencius ProxyLeaderInbound{phase2b = 4 {acceptor_index = 1, slot = 2, round = 3}}
    return 2 + 3 + wire_int32_size(r.y) + wire_int32_size(r.z) + wire_int32_size(r.w);
  } else if (KIND == kWireVmSkip) {
    int4 r = ((const int4*)P.in)[i];
    // ServerInbound{skip = 6 {server_index = 1, start_slot_inclusive = 2, stop_slot_exclusive = 3}}
    return 2 + 3 + wire_int32_size(r.x) + wire_int32_size(r.y) + wire_int32_size(r.z);
  } else if (KIND == kWireNack) {
    int2 r = ((const int2*)P.in)[i];
    return 2 + 1 + wire_int32_size(r.y);     // LeaderInbound{nack = 6 {round = 1}}
  } else if (KIND == kWireMenciusNack) {
    int2 r = ((const int2*)P.in)[i];
    return 2 + 1 + wire_int32_size(r.y);     // mencius LeaderInbound{nack = 7 {round = 1}}
  } else if (KIND == kWireMenciusP2bRange) {
    int4 r = ((const int4*)P.in)[i];
    // ProxyLeaderInbound{phase2b_noop_range = 5 {acceptor_group_index, acceptor_index, start, end, round}}
    return 2 + 5 + wire_int32_size((r.x >> 16) % P.agroups) + wire_int32_size(r.x & 0xffff) + wire_int32_size(r.y) +
           wire_int32_size(r.z) + wire_int32_size(r.w);
  } else if (KIND == kWireMenciusChosenRange) {
    int2 r = ((const int2*)P.in)[i];
    return 2 + 2 + wire_int32_size(r.x) + wire_int32_size(r.y);   // ReplicaInbound{chosen_noop_range = 2 {start, end}}
  } else {
    bool bad = false;
    const WireMsg m = wire_msg<KIND>(P, i, &bad);
    if (bad) *code = FPX_ERR_INVALID_ARG;
    return bad ? 0 : wire_msg_size(m);
  }
}

// An encoder is a codec C: wire_size_kernel<C> and wire_gather_emit_kernel<C> take its C::Params, which hold a WireEnc
// as `enc`, and ask it for
//   size_of(P, i, &code)          record i's message bytes; 0 when it sets *code (the record is bad)
//   msg(P, i, &code), size(P, m)  a gathering encoder's message descriptor of record i and its bytes
//   head(P, m, p, &gsrc, &glen)   writes message m at p but for the glen bytes gathered from enc.src + gsrc, and
//                                 returns where those go
//   stand_down(P)                 the call encodes nothing at all
// WireKindCodec<KIND>: the WireEncodeParams encoders; only the wire_gathers kinds are emitted through msg / head.
template <int KIND>
struct WireKindCodec {
  using Params = WireEncodeParams;
  using Msg = WireMsg;
  static __device__ __forceinline__ bool stand_down(const Params&) { return false; }
  static __device__ __forceinline__ int size_of(const Params& P, int i, int* code) { return wire_size_of<KIND>(P, i, code); }
  static __device__ __forceinline__ Msg msg(const Params& P, int i, int* code) {
    bool bad = false;
    const WireMsg m = wire_msg<KIND>(P, i, &bad);
    if (bad) *code = FPX_ERR_INVALID_ARG;
    return m;
  }
  static __device__ __forceinline__ int size(const Params&, const Msg& m) { return wire_msg_size(m); }
  // the head, a Noop and the trailing isRevocation; the arena's value bytes go between the last two
  static __device__ __forceinline__ uint8_t* head(const Params&, const Msg& m, uint8_t* p, int* gsrc, int* glen) {
    *p++ = (uint8_t)m.outer; p = wire_put_varint(p, (unsigned long long)wire_msg_body(m));
    if (m.nf > 0) p = wire_put_int32(p, 1, m.f0);
    if (m.nf > 1) p = wire_put_int32(p, 2, m.f1);
    if (m.nf > 2) p = wire_put_int32(p, 3, m.f2);
    int vlen = 0;
    if (m.vfield) {
      *p++ = (uint8_t)(m.vfield << 3 | 2); p = wire_put_varint(p, (unsigned long long)m.vlen);
      if (m.noop) { *p++ = 0x12; *p++ = 0x00; }                // CommandOrNoop{noop = 2 {}}
      else vlen = m.vlen;
    }
    if (m.revocation) { p[vlen] = 0x18; p[vlen + 1] = m.is_revocation; }   // Chosen.isRevocation = 3
    *gsrc = m.src; *glen = vlen;
    return p;
  }
};

// pass 1 of every encoder: bytes per tile of kWireEncTile records.  A thread reports its lowest bad record: the
// error word keeps the lowest index of all.
template <class C>
__global__ void __launch_bounds__(kWireEncThreads) wire_size_kernel(typename C::Params P) {
  if (C::stand_down(P)) return;
  __shared__ uint32_t s_w[kWireEncThreads / 32];
  uint32_t sum = 0;
  for (int u = 0; u < kWireEncPer; ++u) {
    const int i = blockIdx.x * kWireEncTile + (int)threadIdx.x * kWireEncPer + u;
    if (i < P.enc.n) {
      int code = FPX_OK;
      sum += (uint32_t)C::size_of(P, i, &code);
      if (code != FPX_OK) report_error(P.enc.err_word, code, i);
    }
  }
  sum = __reduce_add_sync(0xffffffffu, sum);
  if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = sum;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t t = 0;
    for (int w = 0; w < kWireEncThreads / 32; ++w) t += s_w[w];
    P.enc.tile_sum[blockIdx.x] = t;
  }
}

// pass 3 of the gathering encoders (after tile_offsets_kernel): a message's head by its record's thread, its gathered
// bytes by the warps of the CTA (lane-strided copy)
template <class C>
__global__ void __launch_bounds__(kWireEncThreads) wire_gather_emit_kernel(typename C::Params P) {
  if (C::stand_down(P)) return;
  __shared__ uint32_t s_dst[kWireEncTile];     // where each message's gathered bytes go
  __shared__ int32_t s_src[kWireEncTile], s_len[kWireEncTile];
  const uint32_t tiles = gridDim.x;
  if (__ldcg(&P.enc.tile_sum[tiles]) > (uint32_t)P.enc.out_capacity) {   // output buffer too small
    if (blockIdx.x == 0 && threadIdx.x == 0) report_error(P.enc.err_word, FPX_ERR_INVALID_ARG, 0);
    return;
  }
  const uint32_t gbase = __ldcg(&P.enc.tile_sum[blockIdx.x]);
  uint32_t run = 0;
  for (int u = 0; u < kWireEncPer; ++u) {
    const int i = blockIdx.x * kWireEncTile + u * kWireEncThreads + threadIdx.x;
    const int slotix = u * kWireEncThreads + threadIdx.x;
    int code = FPX_OK;
    typename C::Msg m{};
    if (i < P.enc.n) m = C::msg(P, i, &code);
    const uint32_t sz = i < P.enc.n && code == FPX_OK ? (uint32_t)C::size(P, m) : 0u;
    uint32_t tot;
    const uint32_t off = run + cta_scan<kWireEncThreads, true>(sz, ScanSum(), &tot);
    run += tot;
    s_len[slotix] = 0;
    if (i < P.enc.n) P.enc.offs[i] = (int32_t)(gbase + off);
    if (sz) {
      int gsrc = 0, glen = 0;
      const uint8_t* gdst = C::head(P, m, P.enc.out + gbase + off, &gsrc, &glen);
      s_dst[slotix] = (uint32_t)(gdst - P.enc.out);
      s_src[slotix] = gsrc;
      s_len[slotix] = glen;
    }
  }
  if (blockIdx.x == tiles - 1 && threadIdx.x == 0) P.enc.offs[P.enc.n] = (int32_t)(gbase + run);
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int k = warp; k < kWireEncTile; k += kWireEncThreads / 32) {
    const int len = s_len[k];
    const uint8_t* src = P.enc.src + s_src[k];
    uint8_t* dst = P.enc.out + s_dst[k];
    for (int j = lane; j < len; j += 32) dst[j] = __ldg(src + j);
  }
}

// pass 2 (Phase2b / Nack / vanilla Skip).  tile_sum[] holds the byte count of every tile (pass 1); a CTA finds its
// output offset by summing the counts of the tiles before it straight from L2 (<= a few thousand
// values: cheaper than a scan kernel or a look-back chain), serialises its tile into shared memory at
// the output's 16-byte phase and copies the span out with 128-bit stores.  Thread t owns the
// kWireEncPer consecutive records 4t .. 4t+3 of the tile: one CTA scan per tile.
template <int KIND>
__global__ void __launch_bounds__(kWireEncThreads) wire_emit_small_kernel(WireEncodeParams P, int tiles) {
  extern __shared__ __align__(16) uint8_t s_out[];   // 16 + tile * max message size
  const int tile = blockIdx.x;
  const int i0 = tile * kWireEncTile + (int)threadIdx.x * kWireEncPer;
  int4 rec[kWireEncPer];
  uint32_t sz[kWireEncPer];
  int rnd[kWireEncPer];       // kWireMenciusP2bRange: the fifth field
  uint32_t mine = 0;
#pragma unroll
  for (int u = 0; u < kWireEncPer; ++u) {
    const int i = i0 + u;
    sz[u] = 0;
    rec[u] = make_int4(0, 0, 0, 0);
    if (i < P.enc.n) {
      if (KIND == kWirePhase2b) {
        rec[u] = __ldcg((const int4*)P.in + i);      // second read of the records: L2
        sz[u] = 2 + 4 + wire_int32_size(rec[u].x) + wire_int32_size(rec[u].y) + wire_int32_size(rec[u].z) +
                wire_int32_size(rec[u].w);
      } else if (KIND == kWireMenciusPhase2b) {
        rec[u] = __ldcg((const int4*)P.in + i);
        sz[u] = 2 + 3 + wire_int32_size(rec[u].y) + wire_int32_size(rec[u].z) + wire_int32_size(rec[u].w);
      } else if (KIND == kWireVmSkip) {
        rec[u] = __ldcg((const int4*)P.in + i);
        sz[u] = 2 + 3 + wire_int32_size(rec[u].x) + wire_int32_size(rec[u].y) + wire_int32_size(rec[u].z);
      } else if (KIND == kWireMenciusP2bRange) {
        const int4 r = __ldcg((const int4*)P.in + i);
        rec[u] = make_int4((r.x >> 16) % P.agroups, r.x & 0xffff, r.y, r.z);   // fields 1-4; the round is field 5
        sz[u] = 2 + 5 + wire_int32_size(rec[u].x) + wire_int32_size(rec[u].y) + wire_int32_size(rec[u].z) +
                wire_int32_size(rec[u].w) + wire_int32_size(r.w);
        rnd[u] = r.w;
      } else if (KIND == kWireMenciusChosenRange) {
        const int2 r = __ldcg((const int2*)P.in + i);
        rec[u] = make_int4(r.x, r.y, 0, 0);
        sz[u] = 2 + 2 + wire_int32_size(r.x) + wire_int32_size(r.y);
      } else {
        int2 r = __ldcg((const int2*)P.in + i);
        rec[u].y = r.y;
        sz[u] = 2 + 1 + wire_int32_size(r.y);
      }
    }
    mine += sz[u];
  }
  // bytes of all tiles before this one (and, for the last tile, the grand total)
  unsigned long long gb = 0;
  for (int t = threadIdx.x; t < tile; t += kWireEncThreads) gb += __ldcg(&P.enc.tile_sum[t]);
  gb = cta_reduce<kWireEncThreads>(gb, ScanSum());
  uint32_t run;
  uint32_t off = cta_scan<kWireEncThreads, true>(mine, ScanSum(), &run);
  const bool fits = gb + run <= (unsigned long long)P.enc.out_capacity;
  if (!fits && gb <= (unsigned long long)P.enc.out_capacity && threadIdx.x == 0)
    report_error(P.enc.err_word, FPX_ERR_INVALID_ARG, 0);      // output buffer too small
  const uint32_t gbase = (uint32_t)gb;
  const uint32_t phase = gbase & 15u;
  uint8_t* p = s_out + phase + off;
#pragma unroll
  for (int u = 0; u < kWireEncPer; ++u) {
    const int i = i0 + u;
    if (i >= P.enc.n) break;
    P.enc.offs[i] = (int32_t)(gbase + off);
    off += sz[u];
    if (KIND == kWirePhase2b) {
      *p++ = 0x12; *p++ = (uint8_t)(sz[u] - 2);
      p = wire_put_int32(p, 1, rec[u].x); p = wire_put_int32(p, 2, rec[u].y); p = wire_put_int32(p, 3, rec[u].z);
      p = wire_put_int32(p, 4, rec[u].w);
    } else if (KIND == kWireMenciusPhase2b) {
      *p++ = 0x22; *p++ = (uint8_t)(sz[u] - 2);
      p = wire_put_int32(p, 1, rec[u].y); p = wire_put_int32(p, 2, rec[u].z); p = wire_put_int32(p, 3, rec[u].w);
    } else if (KIND == kWireVmSkip) {
      *p++ = 0x32; *p++ = (uint8_t)(sz[u] - 2);
      p = wire_put_int32(p, 1, rec[u].x); p = wire_put_int32(p, 2, rec[u].y); p = wire_put_int32(p, 3, rec[u].z);
    } else if (KIND == kWireMenciusP2bRange) {
      *p++ = 0x2a; *p++ = (uint8_t)(sz[u] - 2);
      p = wire_put_int32(p, 1, rec[u].x); p = wire_put_int32(p, 2, rec[u].y); p = wire_put_int32(p, 3, rec[u].z);
      p = wire_put_int32(p, 4, rec[u].w); p = wire_put_int32(p, 5, rnd[u]);
    } else if (KIND == kWireMenciusChosenRange) {
      *p++ = 0x12; *p++ = (uint8_t)(sz[u] - 2);
      p = wire_put_int32(p, 1, rec[u].x); p = wire_put_int32(p, 2, rec[u].y);
    } else if (KIND == kWireMenciusNack) {
      *p++ = 0x3a; *p++ = (uint8_t)(sz[u] - 2);
      p = wire_put_int32(p, 1, rec[u].y);
    } else {
      *p++ = 0x32; *p++ = (uint8_t)(sz[u] - 2);
      p = wire_put_int32(p, 1, rec[u].y);
    }
  }
  if (tile == tiles - 1 && threadIdx.x == 0) P.enc.offs[P.enc.n] = (int32_t)(gbase + run);
  __syncthreads();
  if (!fits) return;
  // global [gbase, gbase + run) <- shared [phase, phase + run): aligned 16-byte chunks in the middle
  const uint32_t end = phase + run;
  const uint32_t body_lo = phase ? 16u : 0u, body_hi = end & ~15u;
  uint8_t* g0 = P.enc.out + (gbase - phase);     // 16-byte aligned
  if (body_hi > body_lo) {
    for (uint32_t k = body_lo + threadIdx.x * 16u; k < body_hi; k += kWireEncThreads * 16u)
      *(uint4*)(g0 + k) = *(const uint4*)(s_out + k);
  }
  for (uint32_t k = phase + threadIdx.x; k < min(end, body_lo); k += kWireEncThreads) g0[k] = s_out[k];
  for (uint32_t k = max(body_hi, max(body_lo, phase)) + threadIdx.x; k < end; k += kWireEncThreads) g0[k] = s_out[k];
}

// ---------------------------------------------------------------------------
// EPaxos encoder: one canonical ReplicaInbound per record of a handler call's input and output rows (include/fpx.h
// fpx_epaxos_wire_encode).  The gathering encoder above with a codec of its own (EpWireCodec): the member's fields in
// number order by ep_wire_roles, the nested Instance / Ballot / InstancePrefixSetProto written inline, the
// CommandOrNoop's bytes gathered from the arena by the CTA's warps.
// ---------------------------------------------------------------------------
struct EpWireEncodeParams {
  WireEnc enc;                // enc.src: the arena
  int32_t call, replicas, self, per_replica;
  const int32_t* in;          // [n][w_in]   the call's input rows
  const int32_t* rows;        // [n][w_out]  its replies / events / ballots
  int32_t w_in, w_out;
  const int32_t* cmd;         // the handle's cmdLog: value_id of the value-less Commit / Accept records
  const int32_t* value_offs;
  int32_t num_values;
  const uint32_t* refused;    // a refused handler call leaves rows unspecified: nothing is encoded behind it
};
struct EpMsg {
  int member;                 // ReplicaInbound field number, 0: a zero-length message
  unsigned fields;            // bit f - 1: field f of the member is written
  int irep, inum, bord, brep, vord, vrep, replica, status, seq;
  const int32_t* deps;        // n watermarks
  int src, vlen;              // arena[src .. src + vlen)
  bool noop;
};
__device__ __forceinline__ EpMsg ep_enc_msg(const EpWireEncodeParams& P, int i, bool* bad) {
  EpMsg m{};
  const int32_t* in = P.in + (long long)i * P.w_in;
  const int32_t* o = P.rows + (long long)i * P.w_out;
  m.irep = in[0]; m.inum = in[1];
  int value = 0;
  bool cmd_value = false, has_value = false;
  const int call = P.call, kind = P.w_out ? o[0] : 0;
  if (call == 0) {                                              // lead -> PreAccept (Replica.scala:697-706)
    m.member = 2; m.bord = in[2]; m.brep = in[3]; value = in[4]; has_value = true; m.seq = in[5]; m.deps = in + 8;
  } else if (call == 1 || call == 2) {                          // handlePreAccept / handleAccept replies
    if (kind == REPLY_OK) {
      m.member = call == 1 ? 3 : 5; m.bord = o[1]; m.brep = o[2]; m.replica = P.self; m.seq = o[3]; m.deps = o + 4;
    } else if (kind == REPLY_NACK) {
      m.member = 9; m.bord = o[1]; m.brep = o[2];
    } else if (kind == REPLY_COMMIT) {
      m.member = 6; cmd_value = true; m.seq = o[3]; m.deps = o + 4;
    } else if (kind != REPLY_NONE) {
      *bad = true;
    }
  } else if (call == 3 || call == 4 || call == 10) {            // PreAcceptOk / AcceptOk / slow-path timer events
    if (kind == EV_FAST_COMMIT || kind == EV_COMMIT) {
      m.member = 6; cmd_value = true; m.seq = o[1]; m.deps = o + 2;
    } else if (kind == EV_SLOW_ACCEPT && call != 4) {
      m.member = 4; m.bord = in[2]; m.brep = in[3]; cmd_value = true; m.seq = o[1]; m.deps = o + 2;
    } else if (kind != EV_NONE && !(kind == EV_TIMER && call == 3)) {
      *bad = true;
    }
  } else if (call == 7) {                                       // transitionToPreparePhase -> Prepare
    m.member = 7; m.bord = o[0]; m.brep = o[1];
  } else if (call == 8) {                                       // handlePrepare replies
    if (kind == REPLY_OK) {
      m.member = 8; m.bord = o[2]; m.brep = o[3]; m.replica = P.self; m.vord = o[4]; m.vrep = o[5]; m.status = o[6];
      has_value = m.status != ST_NOT_SEEN; value = o[7]; m.seq = o[8]; m.deps = o + 9;
    } else if (kind == REPLY_NACK) {
      m.member = 9; m.bord = o[2]; m.brep = o[3];
    } else if (kind == REPLY_COMMIT) {
      m.member = 6; has_value = true; value = o[7]; m.seq = o[8]; m.deps = o + 9;
    } else if (kind != REPLY_NONE) {
      *bad = true;
    }
  }
  if (!m.member || *bad) { m.member = 0; return m; }
  m.fields = 0;
  const uint32_t roles = ep_wire_roles(m.member);
  for (int f = 1; f <= 8; ++f)
    if ((roles >> (4 * (f - 1))) & 15u) m.fields |= 1u << (f - 1);
  if (m.member == 8 && !has_value) m.fields &= 0x1fu;           // NotSeen: no triple (:1655-1744)
  if (cmd_value) {
    if ((uint32_t)m.irep >= (uint32_t)P.replicas || (uint32_t)m.inum >= (uint32_t)P.per_replica) { *bad = true; m.member = 0; return m; }
    value = __ldcg(P.cmd + ((long long)m.inum * P.replicas + m.irep) * kEpCmdWords + C_VALUE);
    has_value = true;
  }
  if (has_value && value == FPX_VALUE_NOOP) {
    m.noop = true; m.vlen = 2;
  } else if (has_value) {                                       // value_id v: arena[value_offs[v] .. value_offs[v + 1])
    if ((uint32_t)value >= (uint32_t)P.num_values) { *bad = true; m.member = 0; return m; }
    m.src = P.value_offs[value];
    const long long vl = (long long)P.value_offs[value + 1] - m.src;
    if (vl < 0) { *bad = true; m.member = 0; return m; }
    m.vlen = (int)vl;
  }
  return m;
}
// body bytes of m (kWrite: written at p; *vdst = where the arena's value bytes go, which the caller copies)
template <bool kWrite>
__device__ __forceinline__ int ep_msg_body(const EpMsg& m, int n, uint8_t* p, uint8_t** vdst) {
  const uint32_t roles = ep_wire_roles(m.member);
  int len = 0;
  for (int f = 1; f <= 8; ++f) {
    if (!((m.fields >> (f - 1)) & 1u)) continue;
    const int role = (int)((roles >> (4 * (f - 1))) & 15u);
    if (role == kEfInstance || role == kEfBallot || role == kEfVote) {
      const int a = role == kEfInstance ? m.irep : role == kEfBallot ? m.bord : m.vord;
      const int b = role == kEfInstance ? m.inum : role == kEfBallot ? m.brep : m.vrep;
      const int body = 2 + wire_int32_size(a) + wire_int32_size(b);     // <= 22
      if (kWrite) { *p++ = (uint8_t)(f << 3 | 2); *p++ = (uint8_t)body; p = wire_put_int32(p, 1, a); p = wire_put_int32(p, 2, b); }
      len += 2 + body;
    } else if (role >= kEfReplica) {
      const int v = role == kEfReplica ? m.replica : role == kEfStatus ? m.status : m.seq;
      len += 1 + wire_int32_size(v);
      if (kWrite) p = wire_put_int32(p, f, v);
    } else if (role == kEfValue) {
      len += 1 + wire_varint_size((unsigned long long)m.vlen) + m.vlen;
      if (kWrite) {
        *p++ = (uint8_t)(f << 3 | 2); p = wire_put_varint(p, (unsigned long long)m.vlen);
        if (m.noop) { *p++ = 0x12; *p++ = 0x00; }                        // CommandOrNoop{noop = 2 {}}
        else { *vdst = p; p += m.vlen; }
      }
    } else {                                                              // InstancePrefixSet.toProto, no values
      int body = 1 + wire_int32_size(n);
      for (int k = 0; k < n; ++k) body += 3 + wire_int32_size(m.deps[k]);
      len += 1 + wire_varint_size((unsigned long long)body) + body;
      if (kWrite) {
        *p++ = (uint8_t)(f << 3 | 2); p = wire_put_varint(p, (unsigned long long)body); p = wire_put_int32(p, 1, n);
        for (int k = 0; k < n; ++k) {
          const int w = m.deps[k];
          *p++ = 0x12; *p++ = (uint8_t)(1 + wire_int32_size(w)); p = wire_put_int32(p, 1, w);
        }
      }
    }
  }
  return len;
}
__device__ __forceinline__ int ep_msg_size(const EpMsg& m, int n) {
  if (!m.member) return 0;
  const int b = ep_msg_body<false>(m, n, nullptr, nullptr);
  return 1 + wire_varint_size((unsigned long long)b) + b;
}

struct EpWireCodec {
  using Params = EpWireEncodeParams;
  using Msg = EpMsg;
  static __device__ __forceinline__ bool stand_down(const Params& P) { return __ldcg(P.refused) != 0; }
  static __device__ __forceinline__ Msg msg(const Params& P, int i, int* code) {
    bool bad = false;
    const EpMsg m = ep_enc_msg(P, i, &bad);
    if (bad) *code = FPX_ERR_INVALID_ARG;
    return m;
  }
  static __device__ __forceinline__ int size(const Params& P, const Msg& m) { return ep_msg_size(m, P.replicas); }
  static __device__ __forceinline__ int size_of(const Params& P, int i, int* code) { return size(P, msg(P, i, code)); }
  static __device__ __forceinline__ uint8_t* head(const Params& P, const Msg& m, uint8_t* p, int* gsrc, int* glen) {
    *p++ = (uint8_t)(m.member << 3 | 2);
    p = wire_put_varint(p, (unsigned long long)ep_msg_body<false>(m, P.replicas, nullptr, nullptr));
    uint8_t* vdst = nullptr;
    ep_msg_body<true>(m, P.replicas, p, &vdst);
    if (!vdst) return p;
    *gsrc = m.src; *glen = m.vlen;
    return vdst;
  }
};

}  // namespace fpx
