// wire_mencius_phase1_oracle.cc -- CPU ORACLE of compartmentalized Mencius' leader change from bytes (include/fpx.h
// fpx_mencius_acceptor_phase1a_wire, fpx_mencius_leader_phase1b_wire, fpx_wire_encode_mencius_phase2a).  TEST
// INFRASTRUCTURE.
//
// One message at a time, the way the reference's actors see them: Acceptor.handlePhase1a (S/mencius/Acceptor.scala:
// 166-200) on oracle/fpx_oracle.cc's mencius config (whose acceptors hold the Phase2aNoopRange votes too), and
// Leader.handlePhase1b (S/mencius/Leader.scala:582-659) with nextClassicRound (RoundSystem.scala:66-80).  The MultiPaxos
// oracle (tests/wire_phase1_oracle.cc) is compiled in unchanged for its reader, info parser and writers; the byte
// formats are restated from S/mencius/Mencius.proto (Phase1bSlotInfo :120-127, Phase1b :129-137, Phase2a :151-157,
// Nack :266-271, Recover :288-296, LeaderInbound :322-338, ProxyLeaderInbound :339-350).

#include "wire_phase1_oracle.cc"

namespace fpo {
namespace mp1 {
using p1::Reader;
using p1::Phase1b;

// LeaderInbound (nine members) -> kind (the member's field number, 0 none); the Phase1b when kind == 1.  false:
// FPX_ERR_WIRE.  Only the phase1b member is parsed; the others are skipped by length.
bool parse_mencius_leader_inbound(const uint8_t* b, size_t off, size_t len, int* kind, Phase1b* m) {
  Reader r{b, off, off + len};
  int which = 0;
  while (r.p < r.end) {
    const uint32_t tag = r.tag();
    if (!r.ok) return false;
    const int f = (int)(tag >> 3), wt = (int)(tag & 7);
    if (wt == 2 && f >= 1 && f <= 9) {
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
    p1::Info in;
    if (!p1::parse_info(b, sp.first, sp.second, &in)) return false;
    m->info.push_back(in);
  }
  return true;
}

// ClassicRoundRobin(n).nextClassicRound, in 64 bits
long long next_classic_round(long long n, long long leader, long long round) {
  if (round < 0) return leader;
  const long long smallest = n * (round / n), offset = leader % n;
  return smallest + offset > round ? smallest + offset : smallest + n + offset;
}

// result = {complete, max_slot, n_out, next_slot}
int leader_phase1b(int f, int lg_count, int agroups, int per_group, int leader_group, int round, int chosen_watermark,
                   int recover_slot, const uint8_t* b, const int32_t* offs, int n, int value_id_base, P2a* out,
                   int32_t* spans, int cap, int32_t* result, int64_t* err) {
  *err = -1;
  result[0] = -1; result[1] = -1; result[2] = 0; result[3] = -1;
  if (chosen_watermark < 0 || cap < 0 || leader_group < 0 || leader_group >= lg_count || recover_slot < -1)
    return kInvalidArg;
  std::vector<std::map<int, Phase1b>> phase1bs(agroups);        // Phase1.phase1bs, one map per acceptor group
  for (int i = 0; i < n; ++i) {
    int kind = 0;
    Phase1b m;
    if (offs[i] < 0 || offs[i + 1] < offs[i] || !parse_mencius_leader_inbound(b, offs[i], offs[i + 1] - offs[i], &kind, &m)) {
      *err = i;
      return -15;                                               // FPX_ERR_WIRE
    }
    if (kind != 1) continue;
    if (m.round != round) {
      if (m.round > round) { *err = i; return kCheckFailed; }   // logger.checkLt(phase1b.round, round)
      continue;
    }
    if (m.group < 0 || m.group >= agroups || m.acceptor < 0 || m.acceptor >= per_group) {
      *err = i;
      return kBadAcceptor;
    }
    phase1bs[m.group][m.acceptor] = m;
    bool wait = false;
    for (auto& g : phase1bs) wait |= (int)g.size() < f + 1;    // phase1bs.exists(_.size < quorumSize)
    if (wait) continue;
    long long max_slot = INT32_MIN;                             // maxPhase1bSlot over every held Phase1b
    for (auto& g : phase1bs)
      for (auto& kv : g) {
        int s = -1;
        if (!kv.second.info.empty()) {
          s = INT32_MIN;
          for (auto& in : kv.second.info) s = std::max(s, in.slot);
        }
        max_slot = std::max(max_slot, (long long)s);
      }
    max_slot = std::max(max_slot, (long long)recover_slot);     // max(..., phase1.recoverSlot)
    result[0] = i; result[1] = (int32_t)max_slot;
    // logger.check(maxSlot == -1 || slotSystem.leader(maxSlot) == groupIndex)
    if (max_slot != -1 && max_slot % lg_count != leader_group) { *err = i; return kCheckFailed; }
    const long long s0 = next_classic_round(lg_count, leader_group, (long long)chosen_watermark - 1);
    const long long next_slot = next_classic_round(lg_count, leader_group, max_slot);
    if (next_slot > INT32_MAX) { *err = i; return kSlotRange; } // the reference's Int would wrap
    const long long count = max_slot >= s0 ? (max_slot - s0) / lg_count + 1 : 0;
    if (count > cap) { *err = i; return kInvalidArg; }
    // info.find of every held Phase1b, by slot
    std::vector<std::vector<std::unordered_map<int, const p1::Info*>>> find(agroups);
    for (int g = 0; g < agroups; ++g)
      for (auto& kv : phase1bs[g]) {
        find[g].emplace_back();
        for (auto& in : kv.second.info) find[g].back().emplace(in.slot, &in);   // emplace keeps the first
      }
    for (long long k = 0; k < count; ++k) {
      const int slot = (int)(s0 + k * lg_count);
      // safeValue(phase1bs(acceptorGroupIndexBySlot(slot)).values, slot): the highest voteRound, lowest index on ties
      const p1::Info* best = nullptr;
      for (auto& fd : find[(slot / lg_count) % agroups]) {
        auto it = fd.find(slot);
        if (it != fd.end() && (!best || it->second->vote_round > best->vote_round)) best = it->second;
      }
      out[k] = P2a{slot, round, best ? value_id_base + (int)k : kNoopValue, -1};
      spans[2 * k] = best ? (int32_t)best->voff : 0;
      spans[2 * k + 1] = best ? (int32_t)best->vlen : 0;
    }
    result[2] = (int32_t)count;
    result[3] = (int32_t)next_slot;
    return kOk;
  }
  return kOk;
}

}  // namespace mp1
}  // namespace fpo

extern "C" {

// fpx_mencius_leader_phase1b_wire's semantics; spans[2k..2k+1], result[4]
int fpo_mencius_leader_phase1b(int f, int lgroups, int agroups, int per_group, int leader_group, int round,
                               int chosen_watermark, int recover_slot, const uint8_t* bytes, const int32_t* offsets,
                               int n, int value_id_base, void* out, int32_t* spans, int cap, int32_t* result,
                               int64_t* err) {
  return mp1::leader_phase1b(f, lgroups, agroups, per_group, leader_group, round, chosen_watermark, recover_slot, bytes,
                             offsets, n, value_id_base, (P2a*)out, spans, cap, result, err);
}

// Mencius' ProxyLeaderInbound{phase2a = 2}: MultiPaxos' phase2a = 1 with the outer tag of each message changed (the
// one-byte tag 0a becomes 12; nothing else differs)
int64_t fpo_wire_encode_mencius_phase2a(const void* in, int n, const uint8_t* bytes, int n_bytes, const int32_t* spans,
                                        int num_spans, int value_id_base, uint8_t* out, int32_t* offsets, int64_t* err) {
  const int64_t total = fpo_wire_encode_phase2a(in, n, bytes, n_bytes, spans, num_spans, value_id_base, out, offsets, err);
  if (total >= 0 && out)
    for (int i = 0; i < n; ++i) out[offsets[i]] = 0x12;
  return total;
}

// Acceptor.handlePhase1a (S/mencius/Acceptor.scala:166-200) per record of a decoded AcceptorInbound batch (rec =
// {engine_group << 16 | acceptor, -, body off, body len}) on the oracle's Mencius `mp` (fpo_mencius_new), whose votes
// below first_held are taken as retired.  The Phase1b's group_index is the acceptor group inside its leader group
// (engine_group % AG), the Nack is LeaderInbound member 7.  Returns the byte count (out = null: counted, nothing
// applied), or a status < 0 (nothing applied).
int64_t fpo_mencius_acceptor_phase1a_wire(void* mp, int first_held, const uint8_t* bytes, int n_bytes,
                                          const int32_t* kind, const int32_t* rec, int n, const uint8_t* arena,
                                          const int32_t* value_offsets, int num_values, uint8_t* out, int32_t* offsets,
                                          int64_t* err) {
  MultiPaxos& M = *(MultiPaxos*)mp;
  const int AG = M.agroups();
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
  std::vector<std::vector<Acceptor>> saved = M.acceptors;
  std::vector<uint8_t> all;
  offsets[0] = 0;
  for (int i = 0; i < n; ++i) {
    if (kind[i] == 1) {
      const int g = rec[4 * i] >> 16, a = rec[4 * i] & 0xffff;
      Acceptor& acc = M.acceptors[g][a];
      std::vector<uint8_t> body;
      if (rounds[i] < acc.round) {                                // leader.send(LeaderInbound().withNack(...)) :172-177
        p1::put_int32(body, 1, acc.round);
        p1::put_bytes(all, 7, body.data(), body.size());
      } else {
        acc.round = rounds[i];                                    // :181
        p1::put_int32(body, 1, g % AG);                           // acceptorGroupIndex
        p1::put_int32(body, 2, a);
        p1::put_int32(body, 3, acc.round);
        // states.iteratorFrom(chosenWatermark): Phase2a and Phase2aNoopRange votes alike
        for (auto it = acc.states.lower_bound(std::max(cws[i], first_held)); it != acc.states.end(); ++it) {
          std::vector<uint8_t> info;
          p1::put_int32(info, 1, it->first);
          p1::put_int32(info, 2, it->second.first);
          const int v = it->second.second;
          if (v == kNoopValue) {
            p1::put_bytes(info, 3, p1::kNoopBytes, 2);
          } else {
            if (v < 0 || v >= num_values) { *err = i; M.acceptors = saved; return kInvalidArg; }
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

}  // extern "C"
