// epaxos_recovery_oracle.cc -- CPU ORACLE of EPaxos recovery and the timer-driven transitions (include/fpx.h
// fpx_epaxos_commit / _nack / _prepare_phase / _prepare / _prepareok / _slow_path_timer).  TEST INFRASTRUCTURE.
//
// The replica of oracle/fpx_oracle.cc (struct fpo::EPaxos, its handlers on the path) extended by derivation, so one
// state serves traces that mix all eleven calls: that translation unit is compiled into this library unchanged and
// the recovery handlers are added next to it.  Nothing in the product links or calls this file;
// tests/epaxos_recovery_oracle.py compiles it into a temporary directory and binds it with ctypes.  The independent
// Python transcription it is checked against is tests/scala_transcription_recovery.py.
//
// Citations: lines of S/epaxos/Replica.scala, S/ = shared/src/main/scala/frankenpaxos/ in the reference tree.

#include "../oracle/fpx_oracle.cc"

namespace fpo {

struct EPaxosRecovery : EPaxos {
  EPaxosRecovery(int f_, int index_) : EPaxos(f_, index_) {}

  // ---- recovery and the timer-driven transitions (Replica.scala:969-1078, 1567-1869).  The leader kind
  // Preparing keeps its PrepareOks in prepare_responses; reads of largestBallot are floored at the reference's
  // initial value Ballot(0, index) (:458), the stored value keeps starting at (-1, -1).
  enum { kPreparing = 3 };
  enum { kEvRecoverTimer = 1, kEvRestart = 1 };                  // Nack / PrepareOk outcomes
  enum { kNotSeen = 0, kStPreAccepted = 1, kStAccepted = 2 };   // CommandStatus, EPaxos.proto:91-95
  struct PrepareOkMsg { Ballot vote_ballot; int status, value; };
  std::map<Instance, std::map<int, PrepareOkMsg>> prepare_responses;   // Preparing.responses
  Ballot floored_largest() const { return std::max(largest_ballot, Ballot(0, index)); }

  // handleCommit, :1567-1575
  void handle_commit(Instance I, int value, int seq, const InstancePrefixSet& deps) { commit(I, value, seq, deps); }

  // handleNack, :1577-1630: true = (re)arm the recoverInstance timer
  bool handle_nack(Instance I, Ballot lb) {
    largest_ballot = std::max(largest_ballot, lb);            // :1578
    auto it = leader_states.find(I);
    if (it == leader_states.end() || it->second.kind == kLNone) return false;   // :1581-1587
    return it->second.ballot < lb;                            // :1589-1617
  }

  // transitionToPreparePhase, :969-996; false = the ordering would pass FPX_MAX_ROUND
  bool prepare_phase(Instance I, Ballot* out) {
    Ballot L = floored_largest();
    if ((long long)L.first + 1 > 0x7ffffff0) return false;       // FPX_MAX_ROUND
    largest_ballot = Ballot(L.first + 1, index);              // :976
    Leader l;
    l.kind = (LKind)kPreparing; l.ballot = largest_ballot;
    leader_states[I] = l;                                     // :990-995
    prepare_responses[I].clear();
    *out = largest_ballot;
    return true;
  }

  struct PrepareReply { int kind; bool yielded; Ballot ballot, vote_ballot; int status, value, seq; InstancePrefixSet deps; };

  // handlePrepare, :1632-1757
  PrepareReply handle_prepare(Instance I, Ballot b) {
    PrepareReply r{kReplyNone, false, kNullBallot, kNullBallot, kNotSeen, 0, 0, InstancePrefixSet(n)};
    largest_ballot = std::max(largest_ballot, b);             // :1637
    auto ls = leader_states.find(I);                          // :1645-1649
    if (ls != leader_states.end() && ls->second.kind != kLNone && b > ls->second.ballot) {
      leader_states.erase(ls);
      r.yielded = true;
    }
    auto it = cmd_log.find(I);
    if (it != cmd_log.end() && it->second.kind == kCommitted) {   // :1746-1755
      r.kind = kReplyCommit; r.value = it->second.value; r.seq = it->second.seq; r.deps = it->second.deps;
      return r;
    }
    if (it != cmd_log.end() && b < it->second.ballot) {       // :1676-1679, :1700-1703, :1724-1727
      r.kind = kReplyNack; r.ballot = floored_largest();      // built after the update (:1652)
      return r;
    }
    r.kind = kReplyOk; r.ballot = b;
    if (it == cmd_log.end() || it->second.kind == kNoCommand) {   // :1654-1669, :1681-1696
      Entry e;
      e.kind = kNoCommand; e.ballot = b;
      cmd_log[I] = e;
      return r;
    }
    Entry& e = it->second;                                    // :1705-1720, :1729-1744
    r.vote_ballot = e.vote_ballot; r.status = e.kind == kPreAccepted ? kStPreAccepted : kStAccepted;
    r.value = e.value; r.seq = e.seq; r.deps = e.deps;
    e.ballot = b;
    return r;
  }

  struct PrepareOkEvent { int kind; Ballot ballot; int value; };

  // handlePrepareOk, :1759-1869; false = logger.checkLt failed (:1792).  Of the responses with the maximum vote
  // ballot, the PreAccepted one of the LOWEST replica index is taken (the reference iterates a hash map).  The
  // Accepted branch (:1813) and the fast-path candidates (:1836) are unreachable in the reference and here.
  bool handle_prepare_ok(Instance I, Ballot b, int from, Ballot vb, int status, int value, PrepareOkEvent* ev) {
    *ev = PrepareOkEvent{kEvNone, Ballot(0, 0), 0};            // an event row of zeros
    auto it = leader_states.find(I);
    if (it == leader_states.end() || it->second.kind != (LKind)kPreparing) return true;   // :1764-1780
    Leader& l = it->second;
    if (b != l.ballot) return b < l.ballot;                   // :1785-1794
    auto& resp = prepare_responses[I];
    resp[from] = PrepareOkMsg{vb, status, value};             // :1796
    if ((int)resp.size() < slow_quorum) return true;          // :1800-1802
    Ballot vmax = kNullBallot;
    for (auto& kv : resp) vmax = std::max(vmax, kv.second.vote_ballot);   // :1806-1808
    int chosen = kNoopValue;
    for (auto& kv : resp) {                                   // :1856-1866
      if (kv.second.vote_ballot == vmax && kv.second.status == kStPreAccepted) { chosen = kv.second.value; break; }
    }
    *ev = PrepareOkEvent{kEvRestart, l.ballot, chosen};
    leader_states.erase(it);                                  // transitionToPreAcceptPhase is the caller's lead
    prepare_responses.erase(I);
    return true;
  }

  // the defaultToSlowPath timer, :1015-1036: only while it has not been stopped (:618-630)
  Event slow_path_timer(Instance I, Ballot b) {
    auto it = leader_states.find(I);
    if (it == leader_states.end() || it->second.kind != kPreAccepting || it->second.ballot != b ||
        !it->second.timer_armed)
      return Event{kEvNone, 0, InstancePrefixSet(n)};
    return slow_path(I, it->second);
  }
};

}  // namespace fpo

static EPaxosRecovery* ep(void* p) { return (EPaxosRecovery*)p; }

extern "C" {

void* fpo_epr_new(int f, int index) { return new EPaxosRecovery(f, index); }
void fpo_epr_free(void* p) { delete ep(p); }
// the same object as the fpo::EPaxos the handlers on the path (fpo_ep_*) take
void* fpo_epr_base(void* p) { return static_cast<EPaxos*>(ep(p)); }
// the same rows as fpx_epaxos_commit / _nack / _prepare_phase / _prepare / _prepareok / _slow_path_timer
void fpo_epr_commit(void* p, int rep, int num, int value, int seq, const int* deps) {
  EPaxosRecovery* e = ep(p);
  e->handle_commit({rep, num}, value, seq, InstancePrefixSet::from_watermarks(deps, e->n));
}
int fpo_epr_nack(void* p, int rep, int num, int lb_ord, int lb_rep) {
  return (ep(p))->handle_nack({rep, num}, {lb_ord, lb_rep}) ? (int)EPaxosRecovery::kEvRecoverTimer : (int)EPaxosRecovery::kEvNone;
}
// out: {b_ord, b_rep}; returns 0 or kRoundRange
int fpo_epr_prepare_phase(void* p, int rep, int num, int* out) {
  Ballot b;
  if (!(ep(p))->prepare_phase({rep, num}, &b)) return kRoundRange;
  out[0] = b.first; out[1] = b.second;
  return 0;
}
// reply: {kind, yielded, b_ord, b_rep, vb_ord, vb_rep, status, value, seq, deps[n]}
void fpo_epr_prepare(void* p, int rep, int num, int b_ord, int b_rep, int* reply, int* sparse) {
  EPaxosRecovery* e = ep(p);
  auto r = e->handle_prepare({rep, num}, {b_ord, b_rep});
  reply[0] = r.kind; reply[1] = r.yielded; reply[2] = r.ballot.first; reply[3] = r.ballot.second;
  reply[4] = r.vote_ballot.first; reply[5] = r.vote_ballot.second; reply[6] = r.status; reply[7] = r.value;
  reply[8] = r.seq;
  *sparse = 0;
  put_deps(r.deps, e->n, reply + 9, sparse);
}
// event: {kind, b_ord, b_rep, value}; returns 0 or kCheckFailed
int fpo_epr_prepare_ok(void* p, int rep, int num, int b_ord, int b_rep, int from, int vb_ord, int vb_rep, int status,
                      int value, int* event) {
  EPaxosRecovery::PrepareOkEvent ev;
  bool ok = (ep(p))->handle_prepare_ok({rep, num}, {b_ord, b_rep}, from, {vb_ord, vb_rep}, status, value, &ev);
  event[0] = ev.kind; event[1] = ev.ballot.first; event[2] = ev.ballot.second; event[3] = ev.value;
  return ok ? 0 : kCheckFailed;
}
void fpo_epr_slow_path_timer(void* p, int rep, int num, int b_ord, int b_rep, int* event, int* sparse) {
  EPaxosRecovery* e = ep(p);
  auto ev = e->slow_path_timer({rep, num}, {b_ord, b_rep});
  event[0] = ev.kind; event[1] = ev.seq;
  *sparse = 0;
  put_deps(ev.deps, e->n, event + 2, sparse);
}

}  // extern "C"
