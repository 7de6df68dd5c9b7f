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
// Parsing rules restated from the published proto2 wire format (DESIGN.md, wire codec): base-128
// varints of at most 10 bytes, int32 = low 32 bits, unknown fields skipped by wire type, a known
// number with another wire type is unknown, oneof = last member on the wire, a missing
// `required` field or any malformed byte fails the message (FPX_ERR_WIRE + its index).
#pragma once
#include "fpx_common.cuh"
#include "fpx_scan.cuh"

namespace fpx {

constexpr int kWireStage = 24 * 1024;     // bytes of one CTA's message span staged in shared memory
constexpr int kWireDecThreads = 256;
constexpr int kWireEncPer = 4;            // replies per thread of the encoders
constexpr int kWireEncThreads = 256;
constexpr int kWireEncTile = kWireEncPer * kWireEncThreads;
constexpr int kWireMaxP2b = 46, kWireMaxNack = 13;

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
enum WireMember { kWmOpaque = 0, kWmP2a, kWmP2b4, kWmRange3, kWmMenciusP2b, kWmRangeVote5, kWmVmRequest, kWmVmP2a,
                  kWmVmChosen, kWmVmNack };
template <bool kVm>
__device__ __forceinline__ int wire_member(int inbound, int which) {
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
// kVm: inbound 4 (the only one with a bool, a sender or a ClientRequest span: the other inbounds compile without them)
template <bool kShared, bool kVm>
__device__ __forceinline__ bool wire_decode_one(int inbound, int lgroups, int agroups, WireReader<kShared> r, int* kind,
                                                int4* out, bool* value_pos, int* sender) {
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
      if ((tag >> 3) <= (uint32_t)(kVm ? 9 : wire_member_count(inbound))) { which = (int)(tag >> 3); blo = r.p; bhi = r.p + n; }
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
  const int mk = wire_member<kVm>(inbound, which);
  if (mk == kWmOpaque) {
    *out = make_int4(0, 0, (int)blo, (int)(bhi - blo));
    *value_pos = true;
    return true;
  }
  const int n_ints = kVm ? (mk == kWmVmRequest ? 0 : mk == kWmVmChosen ? 1 : mk == kWmVmNack ? 2 : 3)
                         : (mk == kWmP2a ? 2 : mk == kWmP2b4 ? 4 : mk == kWmRangeVote5 ? 5 : 3);
  // the value's field number (0: none) and the required bool's (Chosen.isRevocation)
  const int vfield = kVm ? (mk == kWmVmP2a ? 4 : mk == kWmVmChosen ? 2 : mk == kWmVmRequest ? 1 : 0) : (mk == kWmP2a ? 3 : 0);
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
};

// kVm: the vanilla Mencius instantiation (inbound 4); the other inbounds' instantiation compiles without its bool,
// sender and ClientRequest span
template <bool kVm>
__global__ void __launch_bounds__(kWireDecThreads) wire_decode_kernel(WireDecodeParams P) {
  const int inbound = kVm ? 4 : P.inbound;
  __shared__ __align__(16) uint8_t s_buf[kWireStage + 32];
  const int m0 = blockIdx.x * kWireDecThreads;
  const int m1 = min(P.n, m0 + kWireDecThreads);
  const long long lo = P.offs[m0], hi = P.offs[m1];
  const long long total = P.offs[P.n];
  const long long base = lo & ~15ll;
  const bool sane = lo >= 0 && lo <= hi && hi <= total;   // garbage offsets never turn into wild reads
  const bool staged = sane && hi - base <= kWireStage;
  if (staged) {
    // 128-bit loads while the chunk lies inside the buffer, bytes for the last partial chunk
    for (long long k = (long long)threadIdx.x * 16; base + k < hi; k += (long long)kWireDecThreads * 16) {
      if (base + k + 16 <= (total & ~15ll)) {
        *(uint4*)(s_buf + k) = __ldg((const uint4*)(P.bytes + base + k));
      } else {
        for (int j = 0; j < 16 && base + k + j < total; ++j) s_buf[k + j] = __ldg(P.bytes + base + k + j);
      }
    }
  }
  __syncthreads();
  const int i = m0 + threadIdx.x;
  if (i >= m1) return;
  const long long a = P.offs[i], b = P.offs[i + 1];
  int kind = 0, sender = -1;
  int4 rec = make_int4(0, 0, 0, 0);
  bool ok = sane && a <= b && a >= lo && b <= hi;      // offsets must be monotone
  if (ok) {
    bool value_pos = false;
    if (staged) {
      WireReader<true> r{(uint32_t)__cvta_generic_to_shared(s_buf), nullptr, (uint32_t)(a - base), (uint32_t)(b - base), true};
      ok = wire_decode_one<true, kVm>(inbound, P.lgroups, P.agroups, r, &kind, &rec, &value_pos, &sender);
      if (ok && value_pos) rec.z += (int)base;                  // window -> buffer offsets
    } else {
      WireReader<false> r{0u, P.bytes, (uint32_t)a, (uint32_t)b, true};
      ok = wire_decode_one<false, kVm>(inbound, P.lgroups, P.agroups, r, &kind, &rec, &value_pos, &sender);
    }
  }
  if (!ok) report_error(P.st, FPX_ERR_WIRE, i);
  P.kind[i] = kind;
  P.out[i] = rec;
  if (kVm) P.sender[i] = ok ? sender : -1;
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
enum { kWirePhase2b = 0, kWireNack = 1, kWireChosen = 2, kWireMenciusPhase2b = 3, kWireVmReply = 4, kWireVmChosen = 5,
       kWireVmPhase2a = 6, kWireVmSkip = 7 };
// encoders whose messages carry a value from the arena: size -> scan -> wire_emit_valued_kernel
__host__ __device__ constexpr bool wire_gathers(int kind) {
  return kind == kWireChosen || kind == kWireVmReply || kind == kWireVmChosen || kind == kWireVmPhase2a;
}

struct WireEncodeParams {
  const void* in;             // fpx_p2b (int4) | fpx_nack (int2) | fpx_chosen (int2) | fpx_p2a | fpx_vm_skip_rec
  int32_t n;
  uint8_t* out;               // 16-byte aligned
  int32_t out_capacity;
  int32_t* offs;              // n + 1
  uint32_t* tile_sum;         // [tiles] bytes per tile, then (after the scan) [tiles + 1] exclusive offsets
  // value-gathering encoders: the value bytes of value_id v are arena[value_offs[v] .. value_offs[v + 1])
  const uint8_t* arena;
  const int32_t* value_offs;
  int32_t num_values;
  int32_t servers;            // kWireVmPhase2a: sending_server = slot mod servers
  DevStatus* st;
};

// One message of a value-gathering encoder: outer oneof tag, int32 fields 1..nf, then (vfield != 0) the
// value under field vfield -- arena bytes, or a vanilla Mencius Noop -- then (revocation) the required
// `isRevocation = false` (field 3).  outer = 0: no bytes at all (a retired slot's Chosen, whose value the
// caller holds).
struct WireMsg {
  int outer, nf, vfield;
  int f0, f1, f2;
  int src, vlen;              // arena[src .. src + vlen); noop: CommandOrNoop{noop {}} = 12 00 instead
  bool noop, revocation;
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
  WireMsg m{0, 0, 0, 0, 0, 0, 0, 0, false, false};
  if (KIND == kWireChosen) {                        // ReplicaInbound{chosen = 1 {slot = 1, command_batch_or_noop = 2}}
    const int2 r = ((const int2*)P.in)[i];
    m.outer = 0x0a; m.nf = 1; m.f0 = r.x; m.vfield = 2;
    *bad = !wire_value(P, r.y, false, &m);
  } else if (KIND == kWireVmChosen) {               // ServerInbound{chosen = 7 {slot, command_or_noop, false}}
    const int2 r = ((const int2*)P.in)[i];
    m.outer = 0x3a; m.nf = 1; m.f0 = r.x; m.vfield = 2; m.revocation = true;
    *bad = !wire_value(P, r.y, true, &m);
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
    } else if (r.x == FPX_VM_REPLY_CHOSEN) {        // chosen = 7 {slot, value in round, false}
      m.outer = 0x3a; m.nf = 1; m.f0 = r.z; m.vfield = 2; m.revocation = true;
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
__device__ __forceinline__ int wire_size_of(const WireEncodeParams& P, int i, bool* bad) {
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
  } else {
    const WireMsg m = wire_msg<KIND>(P, i, bad);
    return *bad ? 0 : wire_msg_size(m);
  }
}

// pass 1: bytes per tile of kWireEncTile replies
template <int KIND>
__global__ void __launch_bounds__(kWireEncThreads) wire_size_kernel(WireEncodeParams P) {
  __shared__ uint32_t s_w[kWireEncThreads / 32];
  uint32_t sum = 0;
  bool bad = false;
  int first_bad = INT_MAX;
  for (int u = 0; u < kWireEncPer; ++u) {
    int i = blockIdx.x * kWireEncTile + (int)threadIdx.x * kWireEncPer + u;
    if (i < P.n) {
      bool b = false;
      sum += (uint32_t)wire_size_of<KIND>(P, i, &b);
      if (b) { bad = true; first_bad = min(first_bad, i); }
    }
  }
  if (bad) report_error(P.st, FPX_ERR_INVALID_ARG, first_bad);
  sum = __reduce_add_sync(0xffffffffu, sum);
  if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = sum;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t t = 0;
    for (int w = 0; w < kWireEncThreads / 32; ++w) t += s_w[w];
    P.tile_sum[blockIdx.x] = t;
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
  uint32_t mine = 0;
#pragma unroll
  for (int u = 0; u < kWireEncPer; ++u) {
    const int i = i0 + u;
    sz[u] = 0;
    rec[u] = make_int4(0, 0, 0, 0);
    if (i < P.n) {
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
  for (int t = threadIdx.x; t < tile; t += kWireEncThreads) gb += __ldcg(&P.tile_sum[t]);
  gb = cta_reduce<kWireEncThreads>(gb, ScanSum());
  uint32_t run;
  uint32_t off = cta_scan<kWireEncThreads, true>(mine, ScanSum(), &run);
  const bool fits = gb + run <= (unsigned long long)P.out_capacity;
  if (!fits && gb <= (unsigned long long)P.out_capacity && threadIdx.x == 0)
    report_error(P.st, FPX_ERR_INVALID_ARG, 0);      // output buffer too small
  const uint32_t gbase = (uint32_t)gb;
  const uint32_t phase = gbase & 15u;
  uint8_t* p = s_out + phase + off;
#pragma unroll
  for (int u = 0; u < kWireEncPer; ++u) {
    const int i = i0 + u;
    if (i >= P.n) break;
    P.offs[i] = (int32_t)(gbase + off);
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
    } else {
      *p++ = 0x32; *p++ = (uint8_t)(sz[u] - 2);
      p = wire_put_int32(p, 1, rec[u].y);
    }
  }
  if (tile == tiles - 1 && threadIdx.x == 0) P.offs[P.n] = (int32_t)(gbase + run);
  __syncthreads();
  if (!fits) return;
  // global [gbase, gbase + run) <- shared [phase, phase + run): aligned 16-byte chunks in the middle
  const uint32_t end = phase + run;
  const uint32_t body_lo = phase ? 16u : 0u, body_hi = end & ~15u;
  uint8_t* g0 = P.out + (gbase - phase);     // 16-byte aligned
  if (body_hi > body_lo) {
    for (uint32_t k = body_lo + threadIdx.x * 16u; k < body_hi; k += kWireEncThreads * 16u)
      *(uint4*)(g0 + k) = *(const uint4*)(s_out + k);
  }
  for (uint32_t k = phase + threadIdx.x; k < min(end, body_lo); k += kWireEncThreads) g0[k] = s_out[k];
  for (uint32_t k = max(body_hi, max(body_lo, phase)) + threadIdx.x; k < end; k += kWireEncThreads) g0[k] = s_out[k];
}

// pass 3 of the value-gathering encoders (wire_gathers): a message's head (and a Noop, and the trailing
// isRevocation) by its thread, its value bytes by the warps of the CTA (lane-strided copy)
template <int KIND>
__global__ void __launch_bounds__(kWireEncThreads) wire_emit_valued_kernel(WireEncodeParams P) {
  __shared__ uint32_t s_dst[kWireEncTile];     // where each message's value bytes go
  __shared__ int32_t s_src[kWireEncTile], s_len[kWireEncTile];
  const uint32_t tiles = gridDim.x;
  if (__ldcg(&P.tile_sum[tiles]) > (uint32_t)P.out_capacity) {   // output buffer too small
    if (blockIdx.x == 0 && threadIdx.x == 0) report_error(P.st, FPX_ERR_INVALID_ARG, 0);
    return;
  }
  const uint32_t gbase = __ldcg(&P.tile_sum[blockIdx.x]);
  uint32_t run = 0;
  for (int u = 0; u < kWireEncPer; ++u) {
    const int i = blockIdx.x * kWireEncTile + u * kWireEncThreads + threadIdx.x;
    const int slotix = u * kWireEncThreads + threadIdx.x;
    bool bad = false;
    WireMsg m{};
    if (i < P.n) m = wire_msg<KIND>(P, i, &bad);
    const uint32_t sz = i < P.n && !bad ? (uint32_t)wire_msg_size(m) : 0u;
    uint32_t tot;
    const uint32_t off = run + cta_scan<kWireEncThreads, true>(sz, ScanSum(), &tot);
    run += tot;
    s_len[slotix] = 0;
    if (i < P.n) P.offs[i] = (int32_t)(gbase + off);
    if (i < P.n && sz) {
      uint8_t* p = P.out + gbase + off;
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
      if (m.revocation) { p[vlen] = 0x18; p[vlen + 1] = 0x00; }   // Chosen.isRevocation = 3: false
      s_dst[slotix] = (uint32_t)(p - P.out);
      s_src[slotix] = m.src;
      s_len[slotix] = vlen;
    }
  }
  if (blockIdx.x == tiles - 1 && threadIdx.x == 0) P.offs[P.n] = (int32_t)(gbase + run);
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int m = warp; m < kWireEncTile; m += kWireEncThreads / 32) {
    const int len = s_len[m];
    const uint8_t* src = P.arena + s_src[m];
    uint8_t* dst = P.out + s_dst[m];
    for (int k = lane; k < len; k += 32) dst[k] = __ldg(src + k);
  }
}

}  // namespace fpx
