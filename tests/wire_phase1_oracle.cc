// wire_phase1_oracle.cc -- CPU ORACLE of the new leader's Phase 1 from bytes (include/fpx.h fpx_leader_phase1b_wire)
// and of the Phase2a encoder (fpx_wire_encode_phase2a).  TEST INFRASTRUCTURE.
//
// One message at a time, the way the reference's leader sees them: LeaderInboundSerializer.fromBytes, then
// Leader.handlePhase1b (S/multipaxos/Leader.scala:504-577) with maxPhase1bSlot and safeValue (:304-329).  The
// config and the grid (Grid.isReadQuorum) are oracle/fpx_oracle.cc's MultiPaxos, compiled into this library
// unchanged.  The byte formats are restated from S/multipaxos/MultiPaxos.proto (Phase1bSlotInfo :254-261, Phase1b
// :263-271, Phase2a :273-280, LeaderInbound :525-539, ProxyLeaderInbound :541-549) and the published proto2 wire
// format.  tests/wire_phase1_oracle.py compiles it into a temporary directory and binds it with ctypes.

#include <unordered_map>

#include "../oracle/fpx_oracle.cc"

namespace fpo {
namespace p1 {

struct Reader {
  const uint8_t* b;
  size_t p, end;
  bool ok = true;
  uint64_t varint() {
    uint64_t v = 0;
    for (int i = 0; i < 10; ++i) {
      if (p >= end) { ok = false; return 0; }
      const uint8_t c = b[p++];
      v |= (uint64_t)(c & 0x7f) << (7 * i);
      if (!(c & 0x80)) return v;
    }
    ok = false;
    return 0;
  }
  // a tag (field number >= 1, fits 32 bits) or a length (< 2^31)
  uint32_t tag() {
    const uint64_t v = varint();
    if (!ok || (v >> 32) || (v >> 3) == 0) ok = false;
    return (uint32_t)v;
  }
  uint32_t length() {
    const uint64_t v = varint();
    if (!ok || (v >> 31) || v > end - p) { ok = false; return 0; }
    return (uint32_t)v;
  }
  bool skip(int wt) {
    if (wt == 0) { varint(); return ok; }
    if (wt == 2) { const uint32_t n = length(); if (ok) p += n; return ok; }
    if (wt == 1 || wt == 5) {
      const size_t k = wt == 1 ? 8 : 4;
      if (end - p < k) return ok = false;
      p += k;
      return true;
    }
    return ok = false;
  }
};

struct Info { int slot = 0, vote_round = 0; size_t voff = 0, vlen = 0; };
struct Phase1b {
  int group = 0, acceptor = 0, round = 0;
  unsigned have = 0;
  std::vector<std::pair<size_t, size_t>> info_spans;   // parsed once the message is whole
  std::vector<Info> info;
};

// Phase1bSlotInfo: false on malformed bytes, a missing required field or a second vote_value
bool parse_info(const uint8_t* b, size_t off, size_t len, Info* out) {
  Reader r{b, off, off + len};
  unsigned have = 0;
  while (r.p < r.end) {
    const uint32_t tag = r.tag();
    if (!r.ok) return false;
    const int f = (int)(tag >> 3), wt = (int)(tag & 7);
    if (wt == 0 && (f == 1 || f == 2)) {
      const int v = (int)(uint32_t)r.varint();
      if (!r.ok) return false;
      (f == 1 ? out->slot : out->vote_round) = v;
      have |= 1u << (f - 1);
    } else if (wt == 2 && f == 3) {
      const uint32_t n = r.length();
      if (!r.ok || (have & 4u)) return false;
      out->voff = r.p; out->vlen = n; have |= 4u;
      r.p += n;
    } else if (!r.skip(wt)) {
      return false;
    }
  }
  return have == 7u;
}

// LeaderInbound -> kind (the member's field number, 0 none); the Phase1b when kind == 1.  false: FPX_ERR_WIRE.
bool parse_leader_inbound(const uint8_t* b, size_t off, size_t len, int* kind, Phase1b* m) {
  Reader r{b, off, off + len};
  int which = 0;
  while (r.p < r.end) {
    const uint32_t tag = r.tag();
    if (!r.ok) return false;
    const int f = (int)(tag >> 3), wt = (int)(tag & 7);
    if (wt == 2 && f >= 1 && f <= 8) {
      const uint32_t n = r.length();
      if (!r.ok) return false;
      if (f == 1) {
        if (which != 1) *m = Phase1b();           // another member is replaced; the same one merges
        Reader s{b, r.p, r.p + n};
        while (s.p < s.end) {
          const uint32_t t = s.tag();
          if (!s.ok) return false;
          const int g = (int)(t >> 3), w = (int)(t & 7);
          if (w == 0 && g >= 1 && g <= 3) {
            const int v = (int)(uint32_t)s.varint();
            if (!s.ok) return false;
            (g == 1 ? m->group : g == 2 ? m->acceptor : m->round) = v;
            m->have |= 1u << (g - 1);
          } else if (w == 2 && g == 4) {
            const uint32_t k = s.length();
            if (!s.ok) return false;
            m->info_spans.push_back({s.p, k});
            s.p += k;
          } else if (!s.skip(w)) {
            return false;
          }
        }
      }
      which = f;
      r.p += n;
    } else if (!r.skip(wt)) {
      return false;
    }
  }
  *kind = which;
  if (which != 1) return true;
  if (m->have != 7u) return false;                // "Message missing required fields"
  for (auto& sp : m->info_spans) {
    Info in;
    if (!parse_info(b, sp.first, sp.second, &in)) return false;
    m->info.push_back(in);
  }
  return true;
}

// Leader.handlePhase1b over the batch; result = {complete, max_slot, n_out}
int leader_phase1b(const Config& cfg, int round, int chosen_watermark, const uint8_t* b, const int32_t* offs, int n,
                   int value_id_base, P2a* out, int32_t* spans, int cap, int32_t* result, int64_t* err) {
  *err = -1;
  result[0] = -1; result[1] = -1; result[2] = 0;
  if (chosen_watermark < 0 || cap < 0) return kInvalidArg;
  MultiPaxos mp(cfg);
  std::vector<std::map<int, Phase1b>> phase1bs(cfg.groups);   // Phase1.phase1bs
  NodeSet holders;                                              // Phase1.phase1bAcceptors, as grid node ids
  for (int i = 0; i < n; ++i) {
    int kind = 0;
    Phase1b m;
    if (offs[i] < 0 || offs[i + 1] < offs[i] || !parse_leader_inbound(b, offs[i], offs[i + 1] - offs[i], &kind, &m)) {
      *err = i;
      return -15;                                               // FPX_ERR_WIRE
    }
    if (kind != 1) continue;
    if (m.round != round) {
      if (m.round > round) { *err = i; return kCheckFailed; }   // logger.checkLt(phase1b.round, round)
      continue;
    }
    if (m.group < 0 || m.group >= cfg.groups || m.acceptor < 0 || m.acceptor >= cfg.per_group) {
      *err = i;
      return kBadAcceptor;
    }
    phase1bs[m.group][m.acceptor] = m;
    bool done;
    if (!cfg.flexible) {
      done = true;
      for (auto& g : phase1bs) done = done && (int)g.size() >= cfg.f + 1;
    } else {
      holders.insert(m.group * cfg.per_group + m.acceptor);
      done = mp.grid.is_read(holders) == kTrue;
    }
    if (!done) continue;
    int max_slot = INT32_MIN;                                   // maxPhase1bSlot over every held Phase1b
    for (auto& g : phase1bs)
      for (auto& kv : g) {
        int s = -1;
        if (!kv.second.info.empty()) {
          s = INT32_MIN;
          for (auto& in : kv.second.info) s = std::max(s, in.slot);
        }
        max_slot = std::max(max_slot, s);
      }
    const long long count = std::max(0ll, (long long)max_slot - chosen_watermark + 1);
    result[0] = i; result[1] = max_slot;
    if (count > cap) { *err = i; return kInvalidArg; }
    // info.find of every held Phase1b, by slot
    std::vector<std::vector<std::unordered_map<int, const Info*>>> find(cfg.groups);
    for (int g = 0; g < cfg.groups; ++g)
      for (auto& kv : phase1bs[g]) {
        find[g].emplace_back();
        for (auto& in : kv.second.info) find[g].back().emplace(in.slot, &in);   // emplace keeps the first
      }
    for (long long k = 0; k < count; ++k) {
      const int slot = (int)(chosen_watermark + k);
      // safeValue(phase1bs(slot % numAcceptorGroups).values, slot): maxBy voteRound, the first (lowest index) on ties
      const Info* best = nullptr;
      for (auto& f : find[slot % cfg.groups]) {
        auto it = f.find(slot);
        if (it != f.end() && (!best || it->second->vote_round > best->vote_round)) best = it->second;
      }
      out[k] = P2a{slot, round, best ? value_id_base + (int)k : kNoopValue, -1};
      spans[2 * k] = best ? (int32_t)best->voff : 0;
      spans[2 * k + 1] = best ? (int32_t)best->vlen : 0;
    }
    result[2] = (int32_t)count;
    return kOk;
  }
  return kOk;
}

void put_varint(std::vector<uint8_t>& o, uint64_t v) {
  while (v >= 0x80) { o.push_back((uint8_t)(v | 0x80)); v >>= 7; }
  o.push_back((uint8_t)v);
}
void put_int32(std::vector<uint8_t>& o, int field, int v) {
  o.push_back((uint8_t)(field << 3));
  put_varint(o, (uint64_t)(int64_t)v);
}
void put_bytes(std::vector<uint8_t>& o, int field, const uint8_t* p, size_t n) {
  o.push_back((uint8_t)(field << 3 | 2));
  put_varint(o, n);
  o.insert(o.end(), p, p + n);
}
const uint8_t kNoopBytes[2] = {0x12, 0x00};                      // CommandBatchOrNoop{noop {}}

}  // namespace p1
}  // namespace fpo

using namespace fpo;

extern "C" {

// fpx_leader_phase1b_wire's semantics; spans[2k..2k+1]
int fpo_leader_phase1b(int f, int groups, int per_group, int flexible, int round, int chosen_watermark,
                       const uint8_t* bytes, const int32_t* offsets, int n, int value_id_base, void* out, int32_t* spans,
                       int cap, int32_t* result, int64_t* err) {
  Config cfg{f, groups, per_group, flexible, f + 1, f + 1};
  return p1::leader_phase1b(cfg, round, chosen_watermark, bytes, offsets, n, value_id_base, (P2a*)out, spans, cap,
                            result, err);
}

// ProxyLeaderInbound{phase2a} per record: the total byte count (out = null: only counted), or a status < 0
int64_t fpo_wire_encode_phase2a(const void* in, int n, const uint8_t* bytes, int n_bytes, const int32_t* spans,
                                int num_spans, int value_id_base, uint8_t* out, int32_t* offsets, int64_t* err) {
  const P2a* r = (const P2a*)in;
  std::vector<uint8_t> all;
  *err = -1;
  offsets[0] = 0;
  for (int i = 0; i < n; ++i) {
    const uint8_t* v = p1::kNoopBytes;
    size_t vlen = 2;
    if (r[i].value_id != kNoopValue) {
      const long long k = (long long)r[i].value_id - value_id_base;
      if (k < 0 || k >= num_spans || spans[2 * k] < 0 || spans[2 * k + 1] < 0 ||
          (long long)spans[2 * k] + spans[2 * k + 1] > n_bytes) {
        *err = i;
        return kInvalidArg;
      }
      v = bytes + spans[2 * k]; vlen = (size_t)spans[2 * k + 1];
    }
    std::vector<uint8_t> body;
    p1::put_int32(body, 1, r[i].slot);
    p1::put_int32(body, 2, r[i].round);
    p1::put_bytes(body, 3, v, vlen);
    p1::put_bytes(all, 1, body.data(), body.size());
    offsets[i + 1] = (int32_t)all.size();
  }
  if (out) memcpy(out, all.data(), all.size());
  return (int64_t)all.size();
}

// LeaderInbound{phase1b{group, acceptor, round, info*}} canonically, info k = {slots[k], vote_rounds[k], value}: value
// value_ids[k] is arena[value_offsets[v] .. value_offsets[v+1]), FPX_VALUE_NOOP the Noop.  Returns the byte count
// (out = null: only counted).  Test input at the sizes the runtime's protobuf is too slow for.
int64_t fpo_encode_phase1b(int group, int acceptor, int round, const int32_t* slots, const int32_t* vote_rounds,
                           const int32_t* value_ids, int n_info, const uint8_t* arena, const int32_t* value_offsets,
                           uint8_t* out) {
  std::vector<uint8_t> body, info;
  p1::put_int32(body, 1, group);
  p1::put_int32(body, 2, acceptor);
  p1::put_int32(body, 3, round);
  for (int k = 0; k < n_info; ++k) {
    info.clear();
    p1::put_int32(info, 1, slots[k]);
    p1::put_int32(info, 2, vote_rounds[k]);
    const int v = value_ids[k];
    if (v == kNoopValue) p1::put_bytes(info, 3, p1::kNoopBytes, 2);
    else p1::put_bytes(info, 3, arena + value_offsets[v], (size_t)(value_offsets[v + 1] - value_offsets[v]));
    p1::put_bytes(body, 4, info.data(), info.size());
  }
  std::vector<uint8_t> msg;
  p1::put_bytes(msg, 1, body.data(), body.size());
  if (out) memcpy(out, msg.data(), msg.size());
  return (int64_t)msg.size();
}

}  // extern "C"

namespace fpo {
namespace p1 {
// Phase1a {round = 1, chosen_watermark = 2}, both required
bool parse_phase1a(const uint8_t* b, size_t off, size_t len, int* round, int* cw) {
  Reader r{b, off, off + len};
  unsigned have = 0;
  while (r.p < r.end) {
    const uint32_t tag = r.tag();
    if (!r.ok) return false;
    const int f = (int)(tag >> 3), wt = (int)(tag & 7);
    if (wt == 0 && (f == 1 || f == 2)) {
      const int v = (int)(uint32_t)r.varint();
      if (!r.ok) return false;
      (f == 1 ? *round : *cw) = v;
      have |= 1u << (f - 1);
    } else if (!r.skip(wt)) {
      return false;
    }
  }
  return have == 3u;
}
}  // namespace p1
}  // namespace fpo

extern "C" {

// Acceptor.handlePhase1a per record of a decoded AcceptorInbound batch (rec = {group << 16 | acceptor, -, body off,
// body len}) on the oracle's MultiPaxos `mp` (fpo_mp_new), whose votes below first_held are taken as retired.
// Returns the byte count of the replies (out = null: counted, nothing applied), or a status < 0 (nothing applied).
int64_t fpo_acceptor_phase1a_wire(void* mp, int first_held, const uint8_t* bytes, int n_bytes, const int32_t* kind,
                                  const int32_t* rec, int n, const uint8_t* arena, const int32_t* value_offsets,
                                  int num_values, uint8_t* out, int32_t* offsets, int64_t* err) {
  MultiPaxos& M = *(MultiPaxos*)mp;
  *err = -1;
  std::vector<int> rounds(n), cws(n);
  for (int i = 0; i < n; ++i) {                                   // every record is checked before any is applied
    if (kind[i] != 1) continue;
    const int32_t* r = rec + 4 * i;
    int code = kOk;
    if (r[2] < 0 || r[3] < 0 || (long long)r[2] + r[3] > n_bytes || !p1::parse_phase1a(bytes, r[2], r[3], &rounds[i], &cws[i]))
      code = -15;
    else if ((r[0] >> 16) >= M.cfg.groups || (r[0] & 0xffff) >= M.cfg.per_group)
      code = kInvalidArg;
    else if (cws[i] < first_held && first_held > 0)
      code = kSlotRange;
    if (code != kOk) { *err = i; return code; }
  }
  std::vector<std::vector<Acceptor>> saved;
  if (!out) saved = M.acceptors;
  std::vector<uint8_t> all;
  offsets[0] = 0;
  for (int i = 0; i < n; ++i) {
    if (kind[i] == 1) {
      const int g = rec[4 * i] >> 16, a = rec[4 * i] & 0xffff;
      Acceptor& acc = M.acceptors[g][a];
      std::vector<uint8_t> body, msg;
      if (rounds[i] < acc.round) {                                // Nack(round), Acceptor.scala:156-163
        p1::put_int32(body, 1, acc.round);
        p1::put_bytes(all, 6, body.data(), body.size());
      } else {
        acc.round = rounds[i];                                    // :166
        p1::put_int32(body, 1, g);
        p1::put_int32(body, 2, a);
        p1::put_int32(body, 3, acc.round);
        for (auto it = acc.states.lower_bound(std::max(cws[i], first_held)); it != acc.states.end(); ++it) {
          std::vector<uint8_t> info;
          p1::put_int32(info, 1, it->first);
          p1::put_int32(info, 2, it->second.first);
          const int v = it->second.second;
          if (v == kNoopValue) {
            p1::put_bytes(info, 3, p1::kNoopBytes, 2);
          } else {
            if (v < 0 || v >= num_values) { *err = i; if (!out) M.acceptors = saved; return kInvalidArg; }
            p1::put_bytes(info, 3, arena + value_offsets[v], (size_t)(value_offsets[v + 1] - value_offsets[v]));
          }
          p1::put_bytes(body, 4, info.data(), info.size());
        }
        p1::put_bytes(all, 1, body.data(), body.size());
      }
    }
    offsets[i + 1] = (int32_t)all.size();
  }
  if (out) memcpy(out, all.data(), all.size());
  else M.acceptors = saved;
  return (int64_t)all.size();
}

int fpo_p1_acceptor_round(void* mp, int g, int a) { return ((MultiPaxos*)mp)->acceptors[g][a].round; }

}  // extern "C"
