"""epaxos.Replica's recovery handlers and timer-driven transitions, transcribed line by line from the Scala
(S/epaxos/Replica.scala, S = shared/src/main/scala/frankenpaxos/), sharing no code with oracle/fpx_oracle.cc.
Extends the transcription of the handlers on the path (scala_transcription.EpaxosReplica) with the NoCommand
entry, the Preparing leader state, handleCommit, handleNack, transitionToPreparePhase, handlePrepare,
handlePrepareOk and the defaultToSlowPath timer.  `Rows` drives one replica with the row formats of
include/fpx.h, so traces can be compared with the oracle and the GPU handle.

Two points where the engine departs from a literal reading, as include/fpx.h documents:
  * reads of largestBallot by the new transitions are floored at Ballot(0, index), the reference's initial value
    (:458); the stored value starts at (-1, -1) like the existing transcription's;
  * handlePrepareOk picks among equal-ballot PreAccepted responses the lowest replica index (the reference
    iterates a hash map).
"""
from scala_transcription import NULL_BALLOT, EpaxosReplica, Fatal

NOT_SEEN, PRE_ACCEPTED, ACCEPTED = 0, 1, 2      # CommandStatus, EPaxos.proto:91-95
NOOP = -(1 << 31)
MAX_ORDERING = 0x7ffffff0


class RoundRange(Exception):
    """a prepare ballot whose ordering would pass the largest representable round"""


def popular_items(xs, threshold):  # S/Util.scala:19-21
    return {x for x in xs if xs.count(x) >= threshold}


class RecoveringReplica(EpaxosReplica):
    # cmd_log also holds ("nocommand", ballot, NULL_BALLOT, 0, 0, zeros): NoCommandEntry(ballot), :298-302

    def _zeros(self):
        return (0,) * self.n

    def _floored_largest(self):
        return max(self.largest_ballot, (0, self.index))

    # the existing transcription lets a NoCommand entry fall through; its stale check (:1181-1184, :1433-1438)
    def handle_pre_accept(self, instance, ballot, value, seq, local_deps, msg_deps):
        e = self.cmd_log.get(instance)
        if e is not None and e[0] == "nocommand" and ballot < e[1]:
            return ("nack", self.largest_ballot)
        return super().handle_pre_accept(instance, ballot, value, seq, local_deps, msg_deps)

    def handle_accept(self, instance, ballot, value, seq, deps):
        e = self.cmd_log.get(instance)
        if e is not None and e[0] == "nocommand" and ballot < e[1]:
            return ("nack", self.largest_ballot)
        return super().handle_accept(instance, ballot, value, seq, deps)

    def handle_commit(self, instance, value, seq, deps):  # :1567-1575
        self.commit(instance, value, seq, deps)

    def handle_nack(self, instance, largest_ballot):  # :1577-1630; True = (re)arm the recoverInstance timer
        self.largest_ballot = max(self.largest_ballot, largest_ballot)                        # :1578
        ls = self.leader_states.get(instance)
        if ls is None:                                                                        # :1581-1587
            return False
        if ls["ballot"] >= largest_ballot:                                                    # :1589-1617
            return False
        return True                                                                           # :1623-1629

    def transition_to_prepare_phase(self, instance):  # :969-996
        largest = self._floored_largest()
        if largest[0] + 1 > MAX_ORDERING:
            raise RoundRange()
        self.largest_ballot = (largest[0] + 1, self.index)                                    # :976
        ballot = self.largest_ballot
        self.leader_states[instance] = {"kind": "preparing", "ballot": ballot, "responses": {}}   # :990-995
        return ballot

    def handle_prepare(self, instance, ballot):  # :1632-1757
        self.largest_ballot = max(self.largest_ballot, ballot)                               # :1637
        yielded = False
        ls = self.leader_states.get(instance)
        if ls is not None and ballot > ls["ballot"]:                                          # :1645-1649
            del self.leader_states[instance]
            yielded = True
        nack = ("nack", yielded, self._floored_largest())                                     # :1652
        e = self.cmd_log.get(instance)
        if e is None:                                                                         # :1654-1669
            self.cmd_log[instance] = ("nocommand", ballot, NULL_BALLOT, 0, 0, self._zeros())
            return ("prepareok", yielded, ballot, NULL_BALLOT, NOT_SEEN, None)
        if e[0] == "nocommand":                                                               # :1671-1696
            if ballot < e[1]:
                return nack
            self.cmd_log[instance] = ("nocommand", ballot, NULL_BALLOT, 0, 0, self._zeros())
            return ("prepareok", yielded, ballot, NULL_BALLOT, NOT_SEEN, None)
        if e[0] in ("preaccepted", "accepted"):                                               # :1698-1744
            if ballot < e[1]:
                return nack
            status = PRE_ACCEPTED if e[0] == "preaccepted" else ACCEPTED
            self.cmd_log[instance] = (e[0], ballot) + e[2:]                                   # entry.copy(ballot = ...)
            return ("prepareok", yielded, ballot, e[2], status, (e[3], e[4], e[5]))
        return ("commit", yielded, (e[1], e[2], e[3]))                                        # :1746-1755

    def handle_prepare_ok(self, instance, ballot, replica_index, vote_ballot, status, value):  # :1759-1869
        ls = self.leader_states.get(instance)
        if ls is None or ls["kind"] != "preparing":                                           # :1764-1780
            return None
        if ballot != ls["ballot"]:                                                            # :1785-1794
            if not ballot < ls["ballot"]:
                raise Fatal("logger.checkLt")
            return None
        responses = ls["responses"]
        responses[replica_index] = {"ballot": ballot, "vote_ballot": vote_ballot, "status": status,
                                    "value": value, "replica_index": replica_index}           # :1796
        if len(responses) < self.slow_quorum:                                                 # :1800-1802
            return None
        max_ballot = max(p["vote_ballot"] for p in responses.values())                        # :1806-1807
        prepare_oks = [responses[k] for k in sorted(responses) if responses[k]["vote_ballot"] == max_ballot]
        # :1813 `_.status == Some(CommandStatus.Accepted)`: a proto enum against an Option, never equal
        accepted = [p for p in prepare_oks if p["status"] == ("Some", ACCEPTED)]
        assert not accepted
        # :1833-1851 the fast-path candidates: p.ballot is the Preparing ballot, never Ballot(0, _) here
        fast = [(p["value"],) for p in prepare_oks
                if p["status"] == PRE_ACCEPTED and p["ballot"] == (0, instance[0]) and p["replica_index"] != self.index]
        assert not popular_items(fast, self.f)
        pre = [p for p in prepare_oks if p["status"] == PRE_ACCEPTED]                         # :1856-1867
        value = pre[0]["value"] if pre else NOOP
        # transitionToPreAcceptPhase(instance, ballot, value, avoidFastPath = true): the caller's lead
        del self.leader_states[instance]
        return ("restart", ls["ballot"], value)

    def default_to_slow_path_timer(self, instance, ballot):  # :1015-1036, unless stopTimers stopped it (:618-630)
        ls = self.leader_states.get(instance)
        if ls is None or ls["kind"] != "preaccepting" or ls["ballot"] != ballot or not ls["timer"]:
            return None
        return self.pre_accepting_slow_path(instance, ls)


class Rows:
    """One RecoveringReplica behind the row formats of include/fpx.h (the eleven fpx_epaxos_* calls).  Calls that
    can fail return (status, err_index, out) like the oracle's."""

    def __init__(self, f, index):
        self.r = RecoveringReplica(f, index)
        self.n = self.r.n

    def _deps(self, xs):
        return tuple(int(x) for x in xs)

    def _event(self, ev):
        n = self.n
        if ev is None:
            return [0] * (2 + n)
        kind = {"fast": 1, "slow": 2, "timer": 3, "commit": 4}[ev[0]]
        if ev[0] == "timer":
            return [3, 0] + [0] * n
        return [kind, ev[1]] + list(ev[2])

    def lead(self, rows):
        n = self.n
        for i, r in enumerate(rows):
            try:
                self.r.transition_to_pre_accept_phase((int(r[0]), int(r[1])), (int(r[2]), int(r[3])), int(r[4]),
                                                      int(r[5]), self._deps(r[8:8 + n]), bool(r[6]))
            except Fatal:
                return -13, i
        return 0, -1

    def _reply(self, rep):
        n = self.n
        if rep[0] == "ok":
            seq, deps = (rep[2], rep[3]) if rep[3] is not None else (0, (0,) * n)
            return [1, rep[1][0], rep[1][1], seq] + list(deps)
        if rep[0] == "nack":
            return [2, rep[1][0], rep[1][1], 0] + [0] * n
        if rep[0] == "none":
            return [0, rep[1][0], rep[1][1], 0] + [0] * n
        return [3, -1, -1, rep[1]] + list(rep[2])

    def preaccept(self, rows):
        n = self.n
        return [self._reply(self.r.handle_pre_accept((int(r[0]), int(r[1])), (int(r[2]), int(r[3])), int(r[4]),
                                                     int(r[5]), self._deps(r[6:6 + n]), self._deps(r[6 + n:6 + 2 * n])))
                for r in rows]

    def accept(self, rows):
        n = self.n
        return [self._reply(self.r.handle_accept((int(r[0]), int(r[1])), (int(r[2]), int(r[3])), int(r[4]), int(r[5]),
                                                 self._deps(r[6:6 + n])))
                for r in rows]

    def preacceptok(self, rows):
        n = self.n
        return [self._event(self.r.handle_pre_accept_ok((int(r[0]), int(r[1])), (int(r[2]), int(r[3])), int(r[4]),
                                                        int(r[5]), self._deps(r[6:6 + n])))
                for r in rows]

    def acceptok(self, rows):
        return [self._event(self.r.handle_accept_ok((int(r[0]), int(r[1])), (int(r[2]), int(r[3])), int(r[4])))
                for r in rows]

    def commit(self, rows):
        n = self.n
        for r in rows:
            self.r.handle_commit((int(r[0]), int(r[1])), int(r[2]), int(r[3]), self._deps(r[4:4 + n]))

    def nack(self, rows):
        return [[1 if self.r.handle_nack((int(r[0]), int(r[1])), (int(r[2]), int(r[3]))) else 0] for r in rows]

    def prepare_phase(self, rows):
        out = []
        for i, r in enumerate(rows):
            try:
                out.append(list(self.r.transition_to_prepare_phase((int(r[0]), int(r[1])))))
            except RoundRange:
                return -7, i, out
        return 0, -1, out

    def prepare(self, rows):
        n = self.n
        out = []
        for r in rows:
            rep = self.r.handle_prepare((int(r[0]), int(r[1])), (int(r[2]), int(r[3])))
            if rep[0] == "prepareok":
                _, y, b, vb, status, triple = rep
                value, seq, deps = triple if triple is not None else (0, 0, (0,) * n)
                out.append([1, int(y), b[0], b[1], vb[0], vb[1], status, value, seq] + list(deps))
            elif rep[0] == "nack":
                out.append([2, int(rep[1]), rep[2][0], rep[2][1], -1, -1, NOT_SEEN, 0, 0] + [0] * n)
            else:
                value, seq, deps = rep[2]
                out.append([3, int(rep[1]), -1, -1, -1, -1, NOT_SEEN, value, seq] + list(deps))
        return out

    def prepareok(self, rows):
        out = []
        for i, r in enumerate(rows):
            try:
                ev = self.r.handle_prepare_ok((int(r[0]), int(r[1])), (int(r[2]), int(r[3])), int(r[4]),
                                              (int(r[5]), int(r[6])), int(r[7]), int(r[8]))
            except Fatal:
                return -14, i, out
            out.append([0, 0, 0, 0] if ev is None else [1, ev[1][0], ev[1][1], ev[2]])
        return 0, -1, out

    def slow_path_timer(self, rows):
        return [self._event(self.r.default_to_slow_path_timer((int(r[0]), int(r[1])), (int(r[2]), int(r[3]))))
                for r in rows]

    def entry(self, rep, num):
        """{kind, b_ord, b_rep, vb_ord, vb_rep, value, seq, deps[n]}, leader kind, largestBallot as stored"""
        n = self.n
        e = self.r.cmd_log.get((rep, num))
        if e is None:
            row = [0, -1, -1, -1, -1, 0, 0] + [0] * n
        elif e[0] == "committed":
            row = [4, -1, -1, -1, -1, e[1], e[2]] + list(e[3])
        else:
            kind = {"nocommand": 1, "preaccepted": 2, "accepted": 3}[e[0]]
            row = [kind, e[1][0], e[1][1], e[2][0], e[2][1], e[3], e[4]] + list(e[5])
        ls = self.r.leader_states.get((rep, num))
        lk = 0 if ls is None else {"preaccepting": 1, "accepting": 2, "preparing": 3}[ls["kind"]]
        return row, lk, list(self.r.largest_ballot)
