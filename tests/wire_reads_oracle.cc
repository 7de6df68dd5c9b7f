// wire_reads_oracle.cc -- CPU oracle of the MultiPaxos replica and read-path wire codec.  TEST INFRASTRUCTURE.
//
// Restates the published proto2 wire format (base-128 varints of at most 10 bytes, tag = field << 3 | wire type,
// int32 = low 32 bits, sign-extended to 10 bytes when written, fields written in number order, unknown fields
// skipped by wire type, a known number with another wire type is unknown, the last oneof member on the wire wins,
// a member / nested message given again is merged, a missing `required` field fails the parse) for the shapes of
// S/multipaxos/MultiPaxos.proto: CommandId :188-196, Command :198-204, MaxSlotRequest / MaxSlotReply :316-331,
// BatchMaxSlotRequest / BatchMaxSlotReply :333-349, the read requests :351-396, ClientInbound :489-500,
// ReadBatcherInbound :513-523, ReplicaInbound :563-576.  One message at a time, straight from the format; the GPU
// codec (fpx_wire_reads.cuh) is compared against it.  Pinned by tests/golden/wire_multipaxos_reads.json.
#include <stdint.h>
#include <string.h>

#include <vector>

namespace {
constexpr int kOk = 0, kWireError = -15, kInvalidArg = -1, kOverflow = -8;

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
  // a tag: field number >= 1, the value within 32 bits
  bool tag(int* f, int* wt) {
    uint64_t t = varint();
    if (!ok || (t >> 3) == 0 || t > 0xffffffffull) return ok = false;
    *f = (int)(t >> 3); *wt = (int)(t & 7);
    return true;
  }
  // a length-delimited field: [*lo, *lo + *n)
  bool bytes(const uint8_t** lo, uint64_t* n) {
    *n = varint();
    if (!ok || (uint64_t)(end - p) < *n) return ok = false;
    *lo = p; p += *n;
    return true;
  }
  bool skip(int wt) {
    switch (wt) {
      case 0: varint(); return ok;
      case 1: if (end - p < 8) return ok = false; p += 8; return true;
      case 5: if (end - p < 4) return ok = false; p += 4; return true;
      case 2: { const uint8_t* lo; uint64_t n; return bytes(&lo, &n); }
      default: return ok = false;                   // group wire types
    }
  }
};

struct CommandId {
  unsigned have = 0;
  int32_t pseudo = 0, id = 0;
  const uint8_t* addr = nullptr;
  uint64_t alen = 0;
};
bool parse_command_id(Reader b, CommandId* c) {                        // merged into *c
  int f, wt;
  while (!b.done()) {
    if (!b.tag(&f, &wt)) return false;
    if (f == 1 && wt == 2) { if (!b.bytes(&c->addr, &c->alen)) return false; c->have |= 1; }
    else if ((f == 2 || f == 3) && wt == 0) {
      int32_t v = (int32_t)b.varint();
      if (!b.ok) return false;
      (f == 2 ? c->pseudo : c->id) = v; c->have |= 1u << (f - 1);
    } else if (!b.skip(wt)) return false;
  }
  return true;
}
bool parse_command(Reader b) {
  CommandId cid;
  unsigned have = 0;
  int f, wt;
  while (!b.done()) {
    if (!b.tag(&f, &wt)) return false;
    if ((f == 1 || f == 2) && wt == 2) {
      const uint8_t* lo; uint64_t n;
      if (!b.bytes(&lo, &n)) return false;
      if (f == 1 && !parse_command_id(Reader{lo, lo + n}, &cid)) return false;
      have |= 1u << (f - 1);
    } else if (!b.skip(wt)) return false;
  }
  return have == 3 && cid.have == 7;
}

// the bodies of the final run of the oneof's members 1..members (every member of the run, in wire order)
bool oneof_run(Reader r, int members, int* which, std::vector<std::pair<const uint8_t*, uint64_t>>* bodies) {
  *which = 0; bodies->clear();
  int f, wt;
  while (!r.done()) {
    if (!r.tag(&f, &wt)) return false;
    if (wt == 2) {
      const uint8_t* lo; uint64_t n;
      if (!r.bytes(&lo, &n)) return false;
      if (f <= members) {
        if (f != *which) { *which = f; bodies->clear(); }
        bodies->push_back({lo, n});
      }
    } else if (!r.skip(wt)) return false;
  }
  return true;
}

struct ReplicaMsg {
  int kind = 0;
  int32_t slot = 0;
  int64_t voff = 0, vlen = 0;
  std::vector<std::pair<int64_t, int64_t>> cmds;                     // {off, len} of each Command
};
int decode_replica_one(const uint8_t* base, int64_t lo, int64_t hi, ReplicaMsg* m) {
  *m = ReplicaMsg();
  std::vector<std::pair<const uint8_t*, uint64_t>> bodies;
  int which;
  if (!oneof_run(Reader{base + lo, base + hi}, 7, &which, &bodies)) return kWireError;
  m->kind = which;
  if (which == 0) return kOk;
  const int cf = which == 4 || which == 7 ? 1 : 2;
  const bool has_slot = which != 4 && which != 7, singular = which >= 2 && which <= 4;
  unsigned have = 0;
  for (auto& bd : bodies) {
    Reader b{bd.first, bd.first + bd.second};
    int f, wt;
    while (!b.done()) {
      if (!b.tag(&f, &wt)) return kWireError;
      if (f == 1 && wt == 0 && has_slot) {
        m->slot = (int32_t)b.varint();
        if (!b.ok) return kWireError;
        have |= 1;
      } else if (which == 1 && f == 2 && wt == 2) {
        const uint8_t* v; uint64_t n;
        if (!b.bytes(&v, &n) || (have & 2)) return kWireError;       // a second value: the codec's deviation
        m->voff = v - base; m->vlen = (int64_t)n; have |= 2;
      } else if (which != 1 && f == cf && wt == 2) {
        const uint8_t* c; uint64_t n;
        if (!b.bytes(&c, &n) || (singular && (have & 2))) return kWireError;   // a second Command: deviation
        if (!parse_command(Reader{c, c + n})) return kWireError;
        m->cmds.push_back({c - base, (int64_t)n});
        have |= 2;
      } else if (!b.skip(wt)) return kWireError;
    }
  }
  bool req = which <= 3 ? have == 3 : which == 4 ? (have & 2) != 0 : which <= 6 ? (have & 1) != 0 : true;
  if (!req) return kWireError;
  if (!has_slot) m->slot = -1;
  return kOk;
}

// The codec's offset rule: message i lies inside the span of its tile of 256 messages, and that span inside the
// batch.  With monotone offsets this is a <= b; with others it refuses what the codec refuses.
bool in_window(const int32_t* offs, int32_t n, int32_t i) {
  const int32_t t0 = i / 256 * 256, t1 = t0 + 256 < n ? t0 + 256 : n;
  const int64_t lo = offs[t0], hi = offs[t1], a = offs[i], b = offs[i + 1];
  return lo >= 0 && lo <= hi && hi <= offs[n] && a <= b && a >= lo && b <= hi;
}

void report(int* st, int64_t* idx, int code, int64_t i) {
  if (*st == kOk || i < *idx) { *st = code; *idx = i; }
}
}  // namespace

extern "C" {

// fpx_wire_decode_replica_inbound.  chosen[2k], chosen_values[2k], reads[2k], read_commands[2k]; counts[3].
int fpo_wire_decode_replica(const uint8_t* bytes, const int32_t* offs, int32_t n, int32_t value_id_base,
                            int32_t handle_base, int32_t reads_cap, int32_t* kind, int32_t* chosen,
                            int32_t* chosen_values, int32_t* reads, int32_t* read_commands, int32_t* counts,
                            int64_t* err_index) {
  int st = kOk;
  int64_t idx = -1;
  std::vector<ReplicaMsg> msgs(n);
  int split = n, first_chosen = -1;
  for (int32_t i = 0; i < n; ++i) {
    const int c = in_window(offs, n, i) ? decode_replica_one(bytes, offs[i], offs[i + 1], &msgs[i])
                                                          : kWireError;
    if (c != kOk) { report(&st, &idx, c, i); msgs[i] = ReplicaMsg(); }
    kind[i] = msgs[i].kind;
    if (msgs[i].kind == 1 && first_chosen < 0) first_chosen = i;
    if (msgs[i].kind >= 2 && first_chosen >= 0 && split == n) split = i;
  }
  int32_t nc = 0, nr = 0;
  for (int32_t i = 0; i < split; ++i) {
    const ReplicaMsg& m = msgs[i];
    if (m.kind == 1) {
      chosen[2 * nc] = m.slot; chosen[2 * nc + 1] = (int32_t)((uint32_t)value_id_base + (uint32_t)i);
      chosen_values[2 * nc] = (int32_t)m.voff; chosen_values[2 * nc + 1] = (int32_t)m.vlen;
      ++nc;
    } else if (m.kind >= 2) {
      if ((int64_t)nr + (int64_t)m.cmds.size() > reads_cap) { report(&st, &idx, kOverflow, i); nr += (int32_t)m.cmds.size(); continue; }
      for (auto& c : m.cmds) {
        reads[2 * nr] = m.slot; reads[2 * nr + 1] = (int32_t)((uint32_t)handle_base + (uint32_t)nr);
        read_commands[2 * nr] = (int32_t)c.first; read_commands[2 * nr + 1] = (int32_t)c.second;
        ++nr;
      }
    }
  }
  counts[0] = nc; counts[1] = nr; counts[2] = split;
  *err_index = idx;
  return st;
}

// fpx_reads_wire_decode.  out[4i] = {key, id, voter, slot}, spans[2i].
int fpo_reads_wire_decode(const uint8_t* bytes, const int32_t* offs, int32_t n, int32_t batcher, int32_t key_cap,
                          int32_t* kind, int32_t* out, int32_t* spans, int64_t* err_index) {
  int st = kOk;
  int64_t idx = -1;
  std::vector<std::pair<const uint8_t*, uint64_t>> bodies;
  for (int32_t i = 0; i < n; ++i) {
    int which = 0;
    int32_t v[4] = {0, 0, 0, 0};
    CommandId cid;
    unsigned have = 0;
    bool ok = in_window(offs, n, i) &&
              oneof_run(Reader{bytes + offs[i], bytes + offs[i + 1]}, batcher ? 4 : 5, &which, &bodies);
    if (ok && which == 4) {
      for (auto& bd : bodies) {
        Reader b{bd.first, bd.first + bd.second};
        int f, wt;
        while (ok && !b.done()) {
          if (!b.tag(&f, &wt)) { ok = false; break; }
          if (!batcher && f == 1 && wt == 2) {
            const uint8_t* lo; uint64_t len;
            ok = b.bytes(&lo, &len) && parse_command_id(Reader{lo, lo + len}, &cid);
            have |= 1;
          } else if (f >= (batcher ? 1 : 2) && f <= 4 && wt == 0) {
            v[f - 1] = (int32_t)b.varint();
            ok = b.ok;
            have |= 1u << (f - 1);
          } else {
            ok = b.skip(wt);
          }
        }
      }
      ok = ok && have == 15 && (batcher || cid.have == 7);
    }
    int32_t* o = out + 4 * i;
    o[0] = -1; o[1] = o[2] = o[3] = 0;
    spans[2 * i] = spans[2 * i + 1] = 0;
    if (!ok) { report(&st, &idx, kWireError, i); kind[i] = 0; continue; }
    kind[i] = which;
    if (which == 0) continue;
    spans[2 * i] = (int32_t)(bodies.back().first - bytes); spans[2 * i + 1] = (int32_t)bodies.back().second;
    if (which != 4) continue;
    const int32_t g = batcher ? 0 : v[1], a = v[2];
    const int32_t voter = (uint32_t)g < 0x8000u && (uint32_t)a < 0x8000u ? (g << 16 | a) : -1;
    if (batcher) {
      int32_t key = v[1] % key_cap;
      o[0] = key < 0 ? key + key_cap : key; o[1] = v[1];
    } else {
      o[0] = cid.pseudo; o[1] = cid.id;
    }
    o[2] = voter; o[3] = v[3];
  }
  *err_index = idx;
  return st;
}

}  // extern "C"

namespace {
struct Out {
  uint8_t* p;                    // null: count only
  int64_t n = 0;
  void byte(uint8_t b) { if (p) p[n] = b; ++n; }
  void varint(uint64_t v) { while (v >= 0x80) { byte((uint8_t)(v | 0x80)); v >>= 7; } byte((uint8_t)v); }
  void int32(int f, int32_t v) { byte((uint8_t)(f << 3)); varint((uint64_t)(int64_t)v); }
  void raw(const uint8_t* s, int64_t len) { if (p) memcpy(p + n, s, (size_t)len); n += len; }
};
int64_t varint_size(uint64_t v) { int64_t n = 1; while (v >= 0x80) { v >>= 7; ++n; } return n; }
int64_t int32_size(int32_t v) { return varint_size((uint64_t)(int64_t)v); }
}  // namespace

extern "C" {

// fpx_wire_encode_max_slot_replies (out null: sizes only).  in[4i] = {voter, max_voted_slot, body_off, body_len}.
// Returns the total byte count, or a negative status with *err_index.
int64_t fpo_wire_encode_max_slot_replies(const uint8_t* bytes, int32_t n_bytes, const int32_t* kind, const int32_t* in,
                                         int32_t n, int32_t groups, int32_t per_group, uint8_t* out, int32_t* offs,
                                         int64_t* err_index) {
  Out o{out};
  *err_index = -1;
  int st = kOk;
  int64_t idx = -1;
  for (int32_t i = 0; i < n; ++i) {
    offs[i] = (int32_t)o.n;
    const int32_t* r = in + 4 * i;
    const int k = kind[i];
    if (k != 3 && k != 4) continue;
    bool ok = r[2] >= 0 && r[3] >= 0 && (int64_t)r[2] + r[3] <= n_bytes;
    CommandId cid;
    unsigned have = 0;
    int32_t x[2] = {0, 0};
    if (ok) {
      Reader b{bytes + r[2], bytes + r[2] + r[3]};
      int f, wt;
      while (ok && !b.done()) {
        if (!b.tag(&f, &wt)) { ok = false; break; }
        if (k == 3 && f == 1 && wt == 2) {
          const uint8_t* lo; uint64_t len;
          ok = b.bytes(&lo, &len) && parse_command_id(Reader{lo, lo + len}, &cid);
          have |= 1;
        } else if (k == 4 && (f == 1 || f == 2) && wt == 0) {
          x[f - 1] = (int32_t)b.varint(); ok = b.ok; have |= 1u << (f - 1);
        } else {
          ok = b.skip(wt);
        }
      }
    }
    if (!ok || (k == 3 ? have != 1 || cid.have != 7 : have != 3)) { report(&st, &idx, kWireError, i); continue; }
    const int32_t g = r[0] >> 16, a = r[0] & 0xffff;
    if (r[0] < 0 || g >= groups || a >= per_group) { report(&st, &idx, kInvalidArg, i); continue; }
    Out body{nullptr};
    if (k == 3) {
      const int64_t cl = 1 + varint_size(cid.alen) + (int64_t)cid.alen + 2 + int32_size(cid.pseudo) + int32_size(cid.id);
      body.n = 1 + varint_size((uint64_t)cl) + cl + 3 + int32_size(g) + int32_size(a) + int32_size(r[1]);
      o.byte(0x22); o.varint((uint64_t)body.n);
      o.byte(0x0a); o.varint((uint64_t)cl);
      o.byte(0x0a); o.varint(cid.alen); o.raw(cid.addr, (int64_t)cid.alen);
      o.int32(2, cid.pseudo); o.int32(3, cid.id);
      o.int32(2, g); o.int32(3, a); o.int32(4, r[1]);
    } else {
      body.n = 4 + int32_size(x[0]) + int32_size(x[1]) + int32_size(a) + int32_size(r[1]);
      o.byte(0x22); o.varint((uint64_t)body.n);
      o.int32(1, x[0]); o.int32(2, x[1]); o.int32(3, a); o.int32(4, r[1]);
    }
  }
  offs[n] = (int32_t)o.n;
  if (st != kOk) { *err_index = idx; return st; }
  return o.n;
}

// fpx_reads_wire_encode_read_requests (out null: sizes only).  in[4i] = {key, id, slot, -}; batcher selects
// read_request_batch (5) over read_request (2).
int64_t fpo_reads_wire_encode_read_requests(const int32_t* in, int32_t n, int32_t batcher, const uint8_t* arena,
                                            const int32_t* value_offs, int32_t num_values, uint8_t* out, int32_t* offs,
                                            int64_t* err_index) {
  Out o{out};
  *err_index = -1;
  for (int32_t i = 0; i < n; ++i) {
    offs[i] = (int32_t)o.n;
    const int32_t key = in[4 * i], slot = in[4 * i + 2];
    if (key < 0 || key >= num_values || value_offs[key + 1] < value_offs[key]) { *err_index = i; return kInvalidArg; }
    const int64_t len = value_offs[key + 1] - value_offs[key];
    o.byte(batcher ? 0x2a : 0x12); o.varint((uint64_t)(1 + int32_size(slot) + len));
    o.int32(1, slot); o.raw(arena + value_offs[key], len);
  }
  offs[n] = (int32_t)o.n;
  return o.n;
}

}  // extern "C"
