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

// A oneof member on the path = n leading required int32 fields (numbered 1..n) plus, for Phase2a, one
// nested value (field 3) that is located, not parsed.
//   inbound 0  multipaxos ProxyLeaderInbound (MultiPaxos.proto:541-549)  phase2a = 1, phase2b = 2
//   inbound 1  multipaxos AcceptorInbound    (:551-561)                  phase2a = 2
//   inbound 2  mencius ProxyLeaderInbound    (Mencius.proto:339-350)     phase2a = 2, phase2a_noop_range = 3,
//                                                                        phase2b = 4, phase2b_noop_range = 5
//   inbound 3  mencius AcceptorInbound       (:352-361)                  phase2a = 2, phase2a_noop_range = 3
enum WireMember { kWmOpaque = 0, kWmP2a, kWmP2b4, kWmRange3, kWmMenciusP2b, kWmRangeVote5 };
__device__ __forceinline__ int wire_member(int inbound, int which) {
  if (inbound == 0) return which == 1 ? kWmP2a : which == 2 ? kWmP2b4 : kWmOpaque;
  if (inbound == 1) return which == 2 ? kWmP2a : kWmOpaque;
  if (inbound == 2)
    return which == 2 ? kWmP2a : which == 3 ? kWmRange3 : which == 4 ? kWmMenciusP2b : which == 5 ? kWmRangeVote5 : kWmOpaque;
  return which == 2 ? kWmP2a : which == 3 ? kWmRange3 : kWmOpaque;
}

// members of the inbound's oneof, numbered 1..count (MultiPaxos.proto:541-561, Mencius.proto:339-361)
__device__ __forceinline__ int wire_member_count(int inbound) { return inbound == 0 ? 2 : inbound == 1 ? 4 : inbound == 2 ? 5 : 3; }

// Reader positions in, reader positions out (*value_pos: out->z is a position the caller rebases).
template <bool kShared>
__device__ __forceinline__ bool wire_decode_one(int inbound, int lgroups, int agroups, WireReader<kShared> r, int* kind,
                                                int4* out, bool* value_pos) {
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
      if ((tag >> 3) <= (uint32_t)wire_member_count(inbound)) { which = (int)(tag >> 3); blo = r.p; bhi = r.p + n; }
      r.p += n;
    } else if (!r.skip(wt)) {
      return false;
    }
  }
  *kind = which;
  *out = make_int4(0, 0, 0, 0);
  *value_pos = false;
  if (which == 0) return true;
  const int mk = wire_member(inbound, which);
  if (mk == kWmOpaque) {
    *out = make_int4(0, 0, (int)blo, (int)(bhi - blo));
    *value_pos = true;
    return true;
  }
  const int n_ints = mk == kWmP2a ? 2 : mk == kWmP2b4 ? 4 : mk == kWmRangeVote5 ? 5 : 3;
  WireReader<kShared> b = r;
  b.p = blo; b.end = bhi; b.ok = true;
  int v0 = 0, v1 = 0, v2 = 0, v3 = 0, v4 = 0;
  unsigned have = 0;
  uint32_t off = 0, len = 0;
  bool have_value = false;
  while (!b.done()) {
    const uint32_t tag = b.tag();
    if (!b.ok) return false;
    const int f = (int)(tag >> 3), wt = (int)(tag & 7);
    if (wt == 0 && f >= 1 && f <= n_ints) {
      const int v = (int)b.int32();
      if (!b.ok) return false;
      if (f == 1) v0 = v; else if (f == 2) v1 = v; else if (f == 3) v2 = v; else if (f == 4) v3 = v; else v4 = v;
      have |= 1u << (f - 1);
    } else if (wt == 2 && mk == kWmP2a && f == 3) {
      const uint32_t n = b.small();
      if (!b.ok || b.end - b.p < n || have_value) return false;
      off = b.p; len = n; have_value = true; b.p += n;          // the value bytes are not read
    } else if (!b.skip(wt)) {
      return false;
    }
  }
  if (have != (1u << n_ints) - 1u || (mk == kWmP2a && !have_value)) return false;   // "Message missing required fields."
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
  DevStatus* st;
};

__global__ void __launch_bounds__(kWireDecThreads) wire_decode_kernel(WireDecodeParams P) {
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
  int kind = 0;
  int4 rec = make_int4(0, 0, 0, 0);
  bool ok = sane && a <= b && a >= lo && b <= hi;      // offsets must be monotone
  if (ok) {
    bool value_pos = false;
    if (staged) {
      WireReader<true> r{(uint32_t)__cvta_generic_to_shared(s_buf), nullptr, (uint32_t)(a - base), (uint32_t)(b - base), true};
      ok = wire_decode_one<true>(P.inbound, P.lgroups, P.agroups, r, &kind, &rec, &value_pos);
      if (ok && value_pos) rec.z += (int)base;                  // window -> buffer offsets
    } else {
      WireReader<false> r{0u, P.bytes, (uint32_t)a, (uint32_t)b, true};
      ok = wire_decode_one<false>(P.inbound, P.lgroups, P.agroups, r, &kind, &rec, &value_pos);
    }
  }
  if (!ok) report_error(P.st, FPX_ERR_WIRE, i);
  P.kind[i] = kind;
  P.out[i] = rec;
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

enum { kWirePhase2b = 0, kWireNack = 1, kWireChosen = 2, kWireMenciusPhase2b = 3 };

struct WireEncodeParams {
  const void* in;             // fpx_p2b (int4) | fpx_nack (int2) | fpx_chosen (int2)
  int32_t n;
  uint8_t* out;               // 16-byte aligned
  int32_t out_capacity;
  int32_t* offs;              // n + 1
  uint32_t* tile_sum;         // [tiles] bytes per tile, then (after the scan) [tiles + 1] exclusive offsets
  // Chosen only: the value bytes of value_id v are arena[value_offs[v] .. value_offs[v + 1])
  const uint8_t* arena;
  const int32_t* value_offs;
  int32_t num_values;
  DevStatus* st;
};

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
  } else if (KIND == kWireNack) {
    int2 r = ((const int2*)P.in)[i];
    return 2 + 1 + wire_int32_size(r.y);     // LeaderInbound{nack = 6 {round = 1}}
  } else {
    int2 r = ((const int2*)P.in)[i];
    if ((uint32_t)r.y >= (uint32_t)P.num_values) { *bad = true; return 0; }
    long long vlen = (long long)P.value_offs[r.y + 1] - P.value_offs[r.y];
    if (vlen < 0) { *bad = true; return 0; }
    long long body = 1 + wire_int32_size(r.x) + 1 + wire_varint_size((unsigned long long)vlen) + vlen;
    return (int)(1 + wire_varint_size((unsigned long long)body) + body);
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

// pass 2 (Phase2b / Nack).  tile_sum[] holds the byte count of every tile (pass 1); a CTA finds its
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

// pass 3 (Chosen): header by its thread, value bytes by the warps of the CTA (lane-strided copy)
__global__ void __launch_bounds__(kWireEncThreads) wire_emit_chosen_kernel(WireEncodeParams P) {
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
    const uint32_t sz = i < P.n ? (uint32_t)wire_size_of<kWireChosen>(P, i, &bad) : 0u;
    uint32_t tot;
    const uint32_t off = run + cta_scan<kWireEncThreads, true>(sz, ScanSum(), &tot);
    run += tot;
    s_len[slotix] = 0;
    if (i < P.n && !bad) {
      P.offs[i] = (int32_t)(gbase + off);
      int2 r = ((const int2*)P.in)[i];
      const int src = P.value_offs[r.y], vlen = P.value_offs[r.y + 1] - src;
      const unsigned long long body = 1ull + wire_int32_size(r.x) + 1 + wire_varint_size((unsigned long long)vlen) + vlen;
      uint8_t hdr[24];
      uint8_t* p = hdr;
      *p++ = 0x0a; p = wire_put_varint(p, body);               // ReplicaInbound.chosen = 1
      p = wire_put_int32(p, 1, r.x);                           // Chosen.slot = 1
      *p++ = 0x12; p = wire_put_varint(p, (unsigned long long)vlen);   // Chosen.command_batch_or_noop = 2
      const int hl = (int)(p - hdr);
      uint8_t* g = P.out + gbase + off;
      for (int k = 0; k < hl; ++k) g[k] = hdr[k];
      s_dst[slotix] = gbase + off + (uint32_t)hl;
      s_src[slotix] = src;
      s_len[slotix] = vlen;
    } else if (i < P.n) {
      P.offs[i] = (int32_t)(gbase + off);
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
