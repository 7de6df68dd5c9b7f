// wire_ep_oracle.cc -- CPU oracle of the EPaxos wire codec (decode and pack).  TEST INFRASTRUCTURE.
//
// Restates the published proto2 wire format (protocol-buffers "Encoding": base-128 varints of at most 10 bytes,
// tag = field << 3 | wire type, int32 = the low 32 bits, unknown fields skipped by wire type, a known number with
// another wire type is unknown, repeated scalars packed or not, the last oneof member on the wire wins and a member
// or nested message given again merges into the earlier one, a missing `required` field fails the parse) for the
// shapes of S/epaxos/EPaxos.proto: Instance :35-41, Ballot :46-52, Command :61-78, CommandOrNoop :80-88,
// InstancePrefixSetProto :97-103, ClientRequest :106-111, PreAccept :113-123, PreAcceptOk :125-135, Accept
// :137-147, AcceptOk :149-156, Commit :158-166, Prepare :178-184, PrepareOk :186-209, Nack :211-217, ReplicaInbound
// :220-235, and IntPrefixSetProto (S/compact/IntPrefixSet.proto).  Written straight from the format, one message
// at a time, as a tree of parsed messages; the GPU codec (fpx_wire.cuh) is compared against it.  Pinned by
// tests/golden/wire_epaxos.json.
#include <stdint.h>
#include <string.h>

#include <vector>

namespace {
constexpr int kOk = 0, kInvalidArg = -1, kUnsupported = -11, kWireError = -15;
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
  // -> field number, 0 on a malformed tag
  int tag(int* wt) {
    uint64_t t = varint();
    if (!ok || (t >> 3) == 0 || (t >> 3) > 0x1fffffff) { ok = false; return 0; }
    *wt = (int)(t & 7);
    return (int)(t >> 3);
  }
  bool bytes(Reader* sub) {
    uint64_t n = varint();
    if (!ok || (uint64_t)(end - p) < n) return ok = false;
    *sub = Reader{p, p + n};
    p += n;
    return true;
  }
  bool skip(int wt) {
    Reader s{nullptr, nullptr};
    switch (wt) {
      case 0: varint(); return ok;
      case 1: if (end - p < 8) return ok = false; p += 8; return true;
      case 5: if (end - p < 4) return ok = false; p += 4; return true;
      case 2: return bytes(&s);
      default: return ok = false;                   // group wire types
    }
  }
};

// Instance / Ballot: two required int32
struct Pair { int32_t a = -1, b = -1; bool has_a = false, has_b = false; };
bool parse_pair(Reader r, Pair* m) {           // merges into *m
  while (!r.done()) {
    int wt, f = r.tag(&wt);
    if (!r.ok) return false;
    if (wt == 0 && (f == 1 || f == 2)) {
      int32_t v = (int32_t)r.varint();
      if (!r.ok) return false;
      if (f == 1) { m->a = v; m->has_a = true; } else { m->b = v; m->has_b = true; }
    } else if (!r.skip(wt)) {
      return false;
    }
  }
  return true;
}
// Command: client_address = 1 (bytes), client_pseudonym = 2, client_id = 3, command = 4 (bytes), all required
bool parse_command(Reader r, unsigned* have) {
  while (!r.done()) {
    int wt, f = r.tag(&wt);
    if (!r.ok) return false;
    if (((f == 1 || f == 4) && wt == 2) || ((f == 2 || f == 3) && wt == 0)) *have |= 1u << (f - 1);
    if (!r.skip(wt)) return false;
  }
  return true;
}
// CommandOrNoop -> 0 none, 1 command, 2 noop; false on malformed bytes or an incomplete Command
bool parse_value(Reader r, int* which) {
  *which = 0;
  unsigned cmd = 0;
  while (!r.done()) {
    int wt, f = r.tag(&wt);
    if (!r.ok) return false;
    if (wt == 2 && (f == 1 || f == 2)) {
      Reader s{nullptr, nullptr};
      if (!r.bytes(&s)) return false;
      if (f == 1) {
        if (*which != 1) cmd = 0;              // a new Command, or the one before merged
        if (!parse_command(s, &cmd)) return false;
      } else {
        while (!s.done()) { int w2; s.tag(&w2); if (!s.ok || !s.skip(w2)) return false; }   // Noop: all unknown
      }
      *which = f;
    } else if (!r.skip(wt)) {
      return false;
    }
  }
  return *which != 1 || cmd == 0xf;
}
struct Deps { int32_t num_replicas = 0; bool has_num = false; std::vector<int32_t> wm; int64_t values = 0; };
bool parse_prefix_set(Reader r, Deps* d) {
  bool has_wm = false; int32_t wm = 0;
  while (!r.done()) {
    int wt, f = r.tag(&wt);
    if (!r.ok) return false;
    if (f == 1 && wt == 0) { wm = (int32_t)r.varint(); has_wm = true; }
    else if (f == 2 && wt == 0) { r.varint(); ++d->values; }
    else if (f == 2 && wt == 2) {
      Reader s{nullptr, nullptr};
      if (!r.bytes(&s)) return false;
      while (!s.done()) { s.varint(); if (!s.ok) return false; ++d->values; }
    } else {
      r.skip(wt);
    }
    if (!r.ok) return false;
  }
  if (!has_wm) return false;
  d->wm.push_back(wm);
  return true;
}
bool parse_deps(Reader r, Deps* d) {            // merges: numReplicas overwritten, entries appended
  while (!r.done()) {
    int wt, f = r.tag(&wt);
    if (!r.ok) return false;
    if (f == 1 && wt == 0) { d->num_replicas = (int32_t)r.varint(); if (!r.ok) return false; d->has_num = true; }
    else if (f == 2 && wt == 2) { Reader s{nullptr, nullptr}; if (!r.bytes(&s) || !parse_prefix_set(s, d)) return false; }
    else if (!r.skip(wt)) return false;
  }
  return true;
}

// One member of ReplicaInbound, the fields of all members side by side
struct Member {
  Pair inst, ballot, vote;
  bool has_inst = false, has_ballot = false, has_vote = false;
  int32_t replica = 0, status = 0, seq = 0;
  bool has_replica = false, has_status = false, has_seq = false;
  bool has_value = false; int value_which = 0; int64_t voff = 0, vlen = 0;
  bool has_deps = false; Deps deps;
};
enum Role { NONE, INST, BALLOT, VOTE, VALUE, DEPS, REPLICA, STATUS, SEQ };
Role role(int which, int f) {
  static const Role t[10][9] = {
      {},
      {NONE, VALUE},                                                     // ClientRequest {command}
      {NONE, INST, BALLOT, VALUE, SEQ, DEPS},                            // PreAccept
      {NONE, INST, BALLOT, REPLICA, SEQ, DEPS},                          // PreAcceptOk
      {NONE, INST, BALLOT, VALUE, SEQ, DEPS},                            // Accept
      {NONE, NONE, INST, BALLOT, NONE, NONE, NONE, REPLICA},             // AcceptOk
      {NONE, INST, VALUE, SEQ, DEPS},                                    // Commit
      {NONE, INST, BALLOT},                                              // Prepare
      {NONE, BALLOT, INST, REPLICA, VOTE, STATUS, VALUE, SEQ, DEPS},     // PrepareOk
      {NONE, INST, BALLOT},                                              // Nack {instance, largest_ballot}
  };
  return f >= 1 && f <= 8 ? t[which][f] : NONE;
}
bool parse_member(const uint8_t* base, Reader r, int which, Member* m) {
  while (!r.done()) {
    const uint8_t* tpos = r.p;
    int wt, f = r.tag(&wt);
    if (!r.ok) return false;
    Role ro = role(which, f);
    bool scalar = ro == REPLICA || ro == STATUS || ro == SEQ;
    if (ro == NONE || wt != (scalar ? 0 : 2)) { if (!r.skip(wt)) return false; continue; }
    if (scalar) {
      int32_t v = (int32_t)r.varint();
      if (!r.ok) return false;
      if (ro == REPLICA) { m->replica = v; m->has_replica = true; }
      else if (ro == STATUS) { m->status = v; m->has_status = true; }
      else { m->seq = v; m->has_seq = true; }
      continue;
    }
    Reader s{nullptr, nullptr};
    if (!r.bytes(&s)) return false;
    switch (ro) {
      case INST: if (!parse_pair(s, &m->inst)) return false; m->has_inst = true; break;
      case BALLOT: if (!parse_pair(s, &m->ballot)) return false; m->has_ballot = true; break;
      case VOTE: if (!parse_pair(s, &m->vote)) return false; m->has_vote = true; break;
      case DEPS: if (!parse_deps(s, &m->deps)) return false; m->has_deps = true; break;
      default:                                                  // VALUE
        if (m->has_value) return false;                         // a second one would merge: not supported
        m->has_value = true;
        if (which == 1) {
          unsigned cmd = 0;
          if (!parse_command(s, &cmd) || cmd != 0xf) return false;
          m->value_which = 1; m->voff = tpos - base; m->vlen = s.end - tpos;
        } else {
          if (!parse_value(s, &m->value_which)) return false;
          m->voff = s.p - base; m->vlen = s.end - s.p;
        }
    }
  }
  return true;
}

// One ReplicaInbound -> kind, row (12 + n), value span; status kOk / kWireError / kUnsupported
int decode_one(const uint8_t* base, int64_t lo, int64_t hi, int n, int32_t vid, int32_t* kind, int32_t* row,
               int32_t* span) {
  Reader r{base + lo, base + hi};
  int which = 0;
  Member m;
  int status = kOk;
  while (!r.done()) {
    int wt, f = r.tag(&wt);
    if (!r.ok) { status = kWireError; break; }
    if (wt == 2) {
      Reader s{nullptr, nullptr};
      if (!r.bytes(&s)) { status = kWireError; break; }
      if (f <= 9) {
        if (f != which) { m = Member(); which = f; }
        if (!parse_member(base, s, which, &m)) { status = kWireError; break; }
      }
    } else if (!r.skip(wt)) {
      status = kWireError; break;
    }
  }
  if (status == kOk && which) {
    bool req = true;
    switch (which) {
      case 1: req = m.has_value; break;
      case 2: case 4: req = m.has_inst && m.has_ballot && m.has_value && m.has_seq && m.has_deps; break;
      case 3: req = m.has_inst && m.has_ballot && m.has_replica && m.has_seq && m.has_deps; break;
      case 5: req = m.has_inst && m.has_ballot && m.has_replica; break;
      case 6: req = m.has_inst && m.has_value && m.has_seq && m.has_deps; break;
      case 7: case 9: req = m.has_inst && m.has_ballot; break;
      case 8: req = m.has_ballot && m.has_inst && m.has_replica && m.has_vote && m.has_status; break;
    }
    auto full = [](const Pair& p) { return p.has_a && p.has_b; };
    if (!req || (m.has_inst && !full(m.inst)) || (m.has_ballot && !full(m.ballot)) || (m.has_vote && !full(m.vote)) ||
        (m.has_deps && !m.deps.has_num))
      status = kWireError;
    else if ((m.has_deps && (m.deps.num_replicas != n || (int)m.deps.wm.size() != n)) ||
             (which == 8 && (m.status < 0 || m.status > 2)))
      status = kUnsupported;
  }
  if (status != kOk) { which = 0; m = Member(); }
  *kind = which;
  row[0] = m.inst.a; row[1] = m.inst.b; row[2] = m.ballot.a; row[3] = m.ballot.b; row[4] = m.replica;
  row[5] = m.vote.a; row[6] = m.vote.b; row[7] = m.status;
  row[8] = !m.has_value ? -1 : m.value_which == 2 ? kNoop : vid;
  row[9] = m.seq;
  row[10] = which == 8 && m.has_value && m.has_seq && m.has_deps ? 1 : 0;
  row[11] = (int32_t)m.deps.values;
  for (int k = 0; k < n; ++k) row[12 + k] = m.has_deps ? m.deps.wm[k] : 0;
  span[0] = m.has_value ? (int32_t)m.voff : 0; span[1] = m.has_value ? (int32_t)m.vlen : 0;
  return status;
}
}  // namespace

extern "C" {
// status of the first failing message (err = its index), or 0
int fpo_wire_decode_ep(const uint8_t* bytes, const int32_t* offsets, int count, int n, int32_t value_id_base,
                       int32_t* kind, int32_t* rows, int32_t* values, int64_t* err) {
  *err = -1;
  int first = kOk;
  for (int i = 0; i < count; ++i) {
    int st = decode_one(bytes, offsets[i], offsets[i + 1], n, value_id_base + i, &kind[i], rows + (int64_t)i * (12 + n),
                        values + 2 * i);
    if (st != kOk && first == kOk) { first = st; *err = i; }
  }
  return first;
}
// decoded rows [first, first + count) -> one handler call's input rows (include/fpx.h fpx_epaxos_wire_pack)
int fpo_wire_pack_ep(int call, const int32_t* kind, const int32_t* rows, int first, int count, int n,
                     const int32_t* local_deps, int32_t* out, int64_t* err) {
  *err = -1;
  static const int want[11] = {0, 2, 4, 3, 5, 6, 9, 0, 7, 8, 0};
  if (call < 0 || call > 10 || !want[call]) return kInvalidArg;
  const int W = 12 + n;
  int WO = call == 1 ? 6 + 2 * n : call == 2 || call == 3 ? 6 + n : call == 4 ? 6 : call == 5 ? 4 + n : call == 9 ? 9 : 4;
  for (int j = 0; j < count; ++j) {
    const int i = first + j;
    const int32_t* r = rows + (int64_t)i * W;
    int32_t* o = out + (int64_t)j * WO;
    if (kind[i] != want[call]) { *err = i; return kInvalidArg; }
    if ((call == 1 || call == 2 || call == 3 || call == 5) && r[11] > 0) { *err = i; return kUnsupported; }
    const int32_t* deps = r + 12;
    switch (call) {
      case 1:
        o[0] = r[0]; o[1] = r[1]; o[2] = r[2]; o[3] = r[3]; o[4] = r[8]; o[5] = r[9];
        for (int k = 0; k < n; ++k) { o[6 + k] = local_deps ? local_deps[(int64_t)j * n + k] : 0; o[6 + n + k] = deps[k]; }
        break;
      case 2:
        o[0] = r[0]; o[1] = r[1]; o[2] = r[2]; o[3] = r[3]; o[4] = r[8]; o[5] = r[9];
        for (int k = 0; k < n; ++k) o[6 + k] = deps[k];
        break;
      case 3:
        o[0] = r[0]; o[1] = r[1]; o[2] = r[2]; o[3] = r[3]; o[4] = r[4]; o[5] = r[9];
        for (int k = 0; k < n; ++k) o[6 + k] = deps[k];
        break;
      case 4: o[0] = r[0]; o[1] = r[1]; o[2] = r[2]; o[3] = r[3]; o[4] = r[4]; o[5] = 0; break;
      case 5:
        o[0] = r[0]; o[1] = r[1]; o[2] = r[8]; o[3] = r[9];
        for (int k = 0; k < n; ++k) o[4 + k] = deps[k];
        break;
      case 6: case 8: o[0] = r[0]; o[1] = r[1]; o[2] = r[2]; o[3] = r[3]; break;
      case 9:
        o[0] = r[0]; o[1] = r[1]; o[2] = r[2]; o[3] = r[3]; o[4] = r[4]; o[5] = r[5]; o[6] = r[6]; o[7] = r[7];
        o[8] = (r[10] & 1) ? r[8] : 0;
        break;
    }
  }
  return kOk;
}
}
