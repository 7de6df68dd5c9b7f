// wire_mencius_oracle.cc -- CPU oracle of Compartmentalized Mencius' noop-range and replica wire codec, and of the
// replica's mixed Chosen / ChosenNoopRange call.  TEST INFRASTRUCTURE.
//
// Restates the published proto2 wire format (protocol-buffers "Encoding": base-128 varints of at most 10 bytes,
// tag = field << 3 | wire type, int32 sign-extended to 64 bits, known fields written in field-number order, unknown
// fields skipped by wire type, a known number with another wire type is unknown, the last oneof member on the wire
// wins, a missing `required` field fails the parse) for the shapes of S/mencius/Mencius.proto: Phase2bNoopRange
// :178-187, Chosen :189-195, ChosenNoopRange :197-203, Nack :266-271, LeaderInbound :322-337 (nack = 7),
// ProxyLeaderInbound :339-350, ReplicaInbound :363-371.  Written one message at a time; the GPU codec
// (fpx_wire.cuh) is compared against it.  Pinned by tests/golden/wire_mencius.json.
//
// The replica: Replica.handleChosen (S/mencius/Replica.scala:402-420) and handleChosenNoopRange (:464-486) restated
// per message -- for slot <- start until end by numLeaderGroups: in the log -> return, else log.put -- plus the
// split rule of fpx_mencius_replica_inbound (include/fpx.h).
#include <stdint.h>
#include <string.h>

#include <vector>

namespace {
constexpr int kWireError = -15, kSlotRange = -6;
constexpr int32_t kNoop = INT32_MIN;
constexpr int kMaxRangeBatch = 65535;

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

// One ReplicaInbound -> kind, the fpx_mencius_chosen row (4 ints) and the value span (2 ints).
int decode_one(const uint8_t* base, int64_t lo, int64_t hi, int32_t value_id, int32_t* kind, int32_t* row,
               int32_t* val) {
  row[0] = row[1] = 0; row[2] = kNoop; row[3] = 0; val[0] = val[1] = 0;
  *kind = 0;
  Reader r{base + lo, base + hi};
  int which = 0; const uint8_t* blo = nullptr; const uint8_t* bhi = nullptr;
  while (!r.done()) {
    uint64_t tag = r.varint();
    if (!r.ok || (tag >> 3) == 0 || (tag >> 3) > 0x1fffffff) return kWireError;
    int wt = (int)(tag & 7);
    if (wt == 2) {
      uint64_t n = r.varint();
      if (!r.ok || (uint64_t)(r.end - r.p) < n) return kWireError;
      if ((tag >> 3) <= 2) { which = (int)(tag >> 3); blo = r.p; bhi = r.p + n; }
      r.p += n;
    } else if (!r.skip(wt)) {
      return kWireError;
    }
  }
  if (which == 0) return 0;
  const int n_ints = which == 1 ? 1 : 2, vfield = which == 1 ? 2 : 0;
  Reader b{blo, bhi};
  int32_t v[2] = {0, 0}; unsigned have = 0;
  int64_t off = 0, len = 0; bool have_value = false;
  while (!b.done()) {
    uint64_t tag = b.varint();
    if (!b.ok || (tag >> 3) == 0 || (tag >> 3) > 0x1fffffff) return kWireError;
    int f = (int)(tag >> 3), wt = (int)(tag & 7);
    if (wt == 0 && f >= 1 && f <= n_ints) {
      v[f - 1] = (int32_t)b.varint(); have |= 1u << (f - 1);
      if (!b.ok) return kWireError;
    } else if (wt == 2 && f == vfield) {
      uint64_t n = b.varint();
      if (!b.ok || (uint64_t)(b.end - b.p) < n) return kWireError;
      if (have_value) return kWireError;            // a second value would be merged: not supported
      off = b.p - base; len = (int64_t)n; have_value = true; b.p += n;
    } else if (!b.skip(wt)) {
      return kWireError;
    }
  }
  if (have != (1u << n_ints) - 1u || (vfield && !have_value)) return kWireError;
  *kind = which;
  if (which == 1) {
    row[0] = v[0]; row[1] = (int32_t)((uint32_t)v[0] + 1u); row[2] = value_id;
    val[0] = (int32_t)off; val[1] = (int32_t)len;
  } else {
    row[0] = v[0]; row[1] = v[1];
  }
  return 0;
}

int varint_size(uint64_t v) { int n = 1; while (v >= 0x80) { v >>= 7; ++n; } return n; }
int int32_size(int32_t v) { return varint_size((uint64_t)(int64_t)v); }
uint8_t* put_varint(uint8_t* p, uint64_t v) { while (v >= 0x80) { *p++ = (uint8_t)(v | 0x80); v >>= 7; } *p++ = (uint8_t)v; return p; }
uint8_t* put_int32(uint8_t* p, int field, int32_t v) { *p++ = (uint8_t)(field << 3); return put_varint(p, (uint64_t)(int64_t)v); }

// outer{int32 fields 1..nf}
int64_t put_msg(uint8_t* p, int outer, int nf, const int32_t* f) {
  int64_t body = 0;
  for (int k = 0; k < nf; ++k) body += 1 + int32_size(f[k]);
  const int64_t total = 1 + varint_size((uint64_t)body) + body;
  if (!p) return total;
  *p++ = (uint8_t)outer; p = put_varint(p, (uint64_t)body);
  for (int k = 0; k < nf; ++k) p = put_int32(p, k + 1, f[k]);
  return total;
}

// slots the record covers (0 unless 0 <= start <= end <= cap)
int64_t covers(const int32_t* r, int lg, int64_t cap) {
  if (r[0] < 0 || r[1] < r[0] || r[1] > cap) return 0;
  return ((int64_t)r[1] - r[0] + lg - 1) / lg;
}
}  // namespace

extern "C" {
int fpo_wire_decode_mencius_replica(const uint8_t* bytes, const int32_t* offsets, int n, int32_t value_id_base,
                                    int32_t* kind, int32_t* rows, int32_t* values, int64_t* err) {
  *err = -1;
  int st = 0;
  for (int i = 0; i < n; ++i) {
    int s = decode_one(bytes, offsets[i], offsets[i + 1], value_id_base + i, &kind[i], rows + 4 * i, values + 2 * i);
    if (s != 0 && st == 0) { st = s; *err = i; }
  }
  return st;
}

// what: 0 Phase2bNoopRange (fpx_p2b_range {dst, start, end, round}), 1 ChosenNoopRange ({start, end}), 2 the Mencius
// Nack ({leader, round}).  Returns the total bytes.
int64_t fpo_wire_encode_mencius(int what, const int32_t* in, int n, int agroups, uint8_t* out, int32_t* offsets) {
  int64_t pos = 0;
  for (int i = 0; i < n; ++i) {
    offsets[i] = (int32_t)pos;
    int64_t sz;
    if (what == 0) {
      const int32_t* r = in + 4 * i;
      const int32_t f[5] = {(r[0] >> 16) % agroups, r[0] & 0xffff, r[1], r[2], r[3]};
      sz = put_msg(out ? out + pos : nullptr, 0x2a, 5, f);          // ProxyLeaderInbound.phase2b_noop_range = 5
    } else if (what == 1) {
      sz = put_msg(out ? out + pos : nullptr, 0x12, 2, in + 2 * i);  // ReplicaInbound.chosen_noop_range = 2
    } else {
      sz = put_msg(out ? out + pos : nullptr, 0x3a, 1, in + 2 * i + 1);   // LeaderInbound.nack = 7
    }
    pos += sz;
  }
  offsets[n] = (int32_t)pos;
  return pos;
}

// fpx_mencius_replica_inbound's split: the first range (>= 2 slots) that shares a slot with an earlier range, or the
// first range past kMaxRangeBatch; n if none.
int fpo_mencius_split(const int32_t* in, int n, int lg, int64_t cap) {
  std::vector<int> ranges;
  for (int i = 0; i < n; ++i) {
    const int32_t* r = in + 4 * i;
    if (covers(r, lg, cap) < 2) continue;
    if ((int)ranges.size() == kMaxRangeBatch) return i;
    for (int j : ranges) {
      const int32_t* q = in + 4 * j;
      if (q[0] % lg == r[0] % lg && (q[0] > r[0] ? q[0] : r[0]) < (q[1] < r[1] ? q[1] : r[1])) return i;
    }
    ranges.push_back(i);
  }
  return n;
}

// The records [0, n) applied one message at a time to log[0, cap) (-1 = absent; slots below `retired` count as
// present).  Returns the status of the first record with a bad slot (its index in *err), else 0.
int fpo_mencius_apply(const int32_t* in, int n, int lg, int64_t cap, int64_t retired, int32_t* log, int64_t* err) {
  *err = -1;
  int st = 0;
  for (int i = 0; i < n; ++i) {
    const int32_t* r = in + 4 * i;
    if (r[0] < 0 || r[1] < r[0] || r[1] > cap) {
      if (st == 0) { st = kSlotRange; *err = i; }
      continue;
    }
    for (int64_t s = r[0]; s < r[1]; s += lg) {
      if (s < retired || log[s] != -1) break;       // already in the log: return
      log[s] = r[2];
    }
  }
  return st;
}
}
