// wire_vm_oracle.cc -- CPU oracle of the vanilla Mencius wire codec.  TEST INFRASTRUCTURE.
//
// Restates the published proto2 wire format (protocol-buffers "Encoding": base-128 varints of at most
// 10 bytes, tag = field << 3 | wire type, int32 sign-extended to 64 bits, known fields written in
// field-number order, unknown fields skipped by wire type, a known number with another wire type is
// unknown, the last oneof member on the wire wins, a missing `required` field fails the parse, a bool
// is varint != 0) for the shapes of S/vanillamencius/VanillaMencius.proto: ServerInbound :227-241,
// CommandOrNoop :84-93, ClientRequest :95-100, Phase2a :154-162, Skip :164-172, Phase2b :174-181,
// Chosen :183-190, Phase2Nack :209-215.  Written straight from the format, one message at a time; the
// GPU codec (fpx_wire.cuh) is compared against it.  Pinned by tests/golden/wire_vanilla_mencius.json.
#include <stdint.h>
#include <string.h>

namespace {
constexpr int kWireError = -15, kInvalidArg = -1;
constexpr int32_t kNoop = INT32_MIN;

struct Reader {
  const uint8_t* p; const uint8_t* end;
  bool ok = true;
  bool done() const { return p >= end; }
  uint64_t varint() {
    uint64_t v = 0;
    for (int i = 0; i < 10; ++i) {
      if (p >= end) { ok = false; return 0; }
      uint8_t b = *p++;
      v |= (uint64_t)(b & 0x7f) << (7 * i);
      if (!(b & 0x80)) return v;
    }
    ok = false;
    return 0;
  }
  bool skip(int wt) {
    switch (wt) {
      case 0: varint(); return ok;
      case 1: if (end - p < 8) return ok = false; p += 8; return true;
      case 5: if (end - p < 4) return ok = false; p += 4; return true;
      case 2: { uint64_t n = varint(); if (!ok || (uint64_t)(end - p) < n) return ok = false; p += n; return true; }
      default: return ok = false;                   // group wire types
    }
  }
};

// One ServerInbound.  out = 4 ints, see include/fpx.h (fpx_wire_decode_vm_server_inbound).
int decode_one(const uint8_t* base, int64_t lo, int64_t hi, int32_t* kind, int32_t* out, int32_t* sender) {
  Reader r{base + lo, base + hi};
  int which = 0; const uint8_t* blo = nullptr; const uint8_t* bhi = nullptr;
  while (!r.done()) {
    uint64_t tag = r.varint();
    if (!r.ok || (tag >> 3) == 0 || (tag >> 3) > 0x1fffffff) return kWireError;
    int wt = (int)(tag & 7);
    if (wt == 2) {
      uint64_t n = r.varint();
      if (!r.ok || (uint64_t)(r.end - r.p) < n) return kWireError;
      if ((tag >> 3) <= 9) { which = (int)(tag >> 3); blo = r.p; bhi = r.p + n; }
      r.p += n;
    } else if (!r.skip(wt)) {
      return kWireError;
    }
  }
  *kind = which;
  out[0] = out[1] = out[2] = out[3] = 0;
  *sender = -1;
  if (which == 0) return 0;
  if (which == 2 || which == 3 || which == 8) {     // Phase1a, Phase1b, Phase1Nack: for the host
    out[2] = (int32_t)(blo - base); out[3] = (int32_t)(bhi - blo);
    return 0;
  }
  // per member: int32 fields 1..n_ints, the length-delimited value field, the bool field
  const int n_ints = which == 1 ? 0 : which == 7 ? 1 : which == 9 ? 2 : 3;
  const int vfield = which == 1 ? 1 : which == 4 ? 4 : which == 7 ? 2 : 0;
  const int bfield = which == 7 ? 3 : 0;
  Reader b{blo, bhi};
  int32_t v[3] = {0, 0, 0}; unsigned have = 0;
  int64_t off = 0, len = 0; bool have_value = false, have_bool = false, bval = false;
  while (!b.done()) {
    const uint8_t* tpos = b.p;
    uint64_t tag = b.varint();
    if (!b.ok || (tag >> 3) == 0 || (tag >> 3) > 0x1fffffff) return kWireError;
    int f = (int)(tag >> 3), wt = (int)(tag & 7);
    if (wt == 0 && f >= 1 && f <= n_ints) {
      v[f - 1] = (int32_t)b.varint(); have |= 1u << (f - 1);
      if (!b.ok) return kWireError;
    } else if (wt == 0 && f == bfield) {
      bval = b.varint() != 0; have_bool = true;
      if (!b.ok) return kWireError;
    } else if (wt == 2 && f == vfield) {
      uint64_t n = b.varint();
      if (!b.ok || (uint64_t)(b.end - b.p) < n) return kWireError;
      if (have_value) return kWireError;            // a second value would be merged: not supported
      // ClientRequest: the whole `command` field, tag included (= CommandOrNoop().withCommand(command))
      const uint8_t* start = which == 1 ? tpos : b.p;
      off = start - base; len = (int64_t)(b.p + n - start); have_value = true; b.p += n;
    } else if (!b.skip(wt)) {
      return kWireError;
    }
  }
  if (have != (1u << n_ints) - 1u || (vfield && !have_value) || (bfield && !have_bool)) return kWireError;
  switch (which) {
    case 1: out[2] = (int32_t)off; out[3] = (int32_t)len; break;
    case 4: out[0] = v[1]; out[1] = v[2]; out[2] = (int32_t)off; out[3] = (int32_t)len; *sender = v[0]; break;
    case 5: out[1] = v[0]; out[2] = v[1]; out[3] = v[2]; *sender = v[0]; break;
    case 6: out[0] = v[0]; out[1] = v[1]; out[2] = v[2]; *sender = v[0]; break;
    case 7: out[0] = v[0]; out[1] = bval ? 1 : 0; out[2] = (int32_t)off; out[3] = (int32_t)len; break;
    case 9: out[0] = v[0]; out[1] = v[1]; break;
    default: out[2] = (int32_t)(blo - base); out[3] = (int32_t)(bhi - blo); break;   // unknown members
  }
  return 0;
}

int varint_size(uint64_t v) { int n = 1; while (v >= 0x80) { v >>= 7; ++n; } return n; }
int int32_size(int32_t v) { return varint_size((uint64_t)(int64_t)v); }
uint8_t* put_varint(uint8_t* p, uint64_t v) { while (v >= 0x80) { *p++ = (uint8_t)(v | 0x80); v >>= 7; } *p++ = (uint8_t)v; return p; }
uint8_t* put_int32(uint8_t* p, int field, int32_t v) { *p++ = (uint8_t)(field << 3); return put_varint(p, (uint64_t)(int64_t)v); }

struct Values { const uint8_t* arena; const int32_t* offs; int num; };

// one message: ServerInbound{outer: {int32 fields 1..nf, [vfield: CommandOrNoop], [isRevocation = false]}}
struct Msg { int outer, nf; int32_t f[3]; int vfield; int32_t value; bool revocation; };

// bytes of m at p (p == nullptr: only the size); kInvalidArg for a value_id outside the arena
int64_t put_msg(uint8_t* p, const Msg& m, const Values& vals) {
  const uint8_t* src = nullptr; int64_t vlen = 0;
  static const uint8_t kNoopBytes[2] = {0x12, 0x00};   // CommandOrNoop{noop = 2 {}}
  if (m.vfield) {
    if (m.value == kNoop) { src = kNoopBytes; vlen = 2; }
    else if (m.value < 0 || m.value >= vals.num) return kInvalidArg;
    else { src = vals.arena + vals.offs[m.value]; vlen = vals.offs[m.value + 1] - vals.offs[m.value]; }
  }
  int64_t body = 0;
  for (int k = 0; k < m.nf; ++k) body += 1 + int32_size(m.f[k]);
  if (m.vfield) body += 1 + varint_size((uint64_t)vlen) + vlen;
  if (m.revocation) body += 2;
  const int64_t total = 1 + varint_size((uint64_t)body) + body;
  if (!p) return total;
  *p++ = (uint8_t)m.outer; p = put_varint(p, (uint64_t)body);
  for (int k = 0; k < m.nf; ++k) p = put_int32(p, k + 1, m.f[k]);
  if (m.vfield) { *p++ = (uint8_t)(m.vfield << 3 | 2); p = put_varint(p, (uint64_t)vlen); memcpy(p, src, (size_t)vlen); p += vlen; }
  if (m.revocation) { *p++ = 0x18; *p++ = 0x00; }
  return total;
}

// kind: 0 reply stream (int4 {kind, server, slot, round|value}), 1 Chosen (int2 {slot, value}),
// 2 Phase2a (int4 {slot, round, value, dst}), 3 Skip (int4 {server, start, stop, own}).  Returns the total
// bytes, or a negative status with *err = the record.
int64_t encode(int kind, const int32_t* in, int n, int servers, const Values& vals, uint8_t* out, int32_t* offsets,
               int64_t* err) {
  *err = -1;
  int64_t pos = 0;
  for (int i = 0; i < n; ++i) {
    offsets[i] = (int32_t)pos;
    Msg m{0, 0, {0, 0, 0}, 0, 0, false};
    if (kind == 0) {
      const int32_t* r = in + 4 * i;
      if (r[0] == 0) m = Msg{0x2a, 3, {r[1], r[2], r[3]}, 0, 0, false};         // phase2b = 5
      else if (r[0] == 1) m = Msg{0x4a, 2, {r[2], r[3], 0}, 0, 0, false};       // phase2_nack = 9
      else if (r[0] == 2) m = Msg{0x3a, 1, {r[2], 0, 0}, 2, r[3], true};        // chosen = 7
      else if (r[0] == 3) continue;                                             // retired: no bytes
      else { *err = i; return kInvalidArg; }
    } else if (kind == 1) {
      const int32_t* r = in + 2 * i;
      m = Msg{0x3a, 1, {r[0], 0, 0}, 2, r[1], true};
    } else if (kind == 2) {
      const int32_t* r = in + 4 * i;
      const int32_t owner = ((r[0] % servers) + servers) % servers;
      m = Msg{0x22, 3, {owner, r[0], r[1]}, 4, r[2], false};                    // phase2a = 4
    } else {
      const int32_t* r = in + 4 * i;
      m = Msg{0x32, 3, {r[0], r[1], r[2]}, 0, 0, false};                        // skip = 6
    }
    const int64_t sz = put_msg(out ? out + pos : nullptr, m, vals);
    if (sz < 0) { *err = i; return sz; }
    pos += sz;
  }
  offsets[n] = (int32_t)pos;
  return pos;
}
}  // namespace

extern "C" {
int fpo_wire_decode_vm(const uint8_t* bytes, const int32_t* offsets, int n, int32_t* kind, int32_t* out, int32_t* sender,
                       int64_t* err) {
  *err = -1;
  for (int i = 0; i < n; ++i) {
    int st = decode_one(bytes, offsets[i], offsets[i + 1], &kind[i], out + 4 * i, &sender[i]);
    if (st != 0) { *err = i; return st; }
  }
  return 0;
}
int64_t fpo_wire_encode_vm(int kind, const int32_t* in, int n, int servers, const uint8_t* arena, const int32_t* value_offsets,
                           int num_values, uint8_t* out, int32_t* offsets, int64_t* err) {
  return encode(kind, in, n, servers, Values{arena, value_offsets, num_values}, out, offsets, err);
}
}
