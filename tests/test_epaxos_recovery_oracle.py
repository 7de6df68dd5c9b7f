"""Known answers for EPaxos recovery and the timer-driven transitions, checked on the CPU oracle
(tests/epaxos_recovery_oracle.cc) and on the
independent transcription of the Scala; then both on seeded traces that mix all eleven fpx_epaxos_* calls.
S/ = shared/src/main/scala/frankenpaxos/, every line cited is S/epaxos/Replica.scala."""
import numpy as np
import pytest

import epaxos_recovery_oracle as R
import scala_transcription_recovery as T
from epaxos_recovery_traces import Trace

NOOP = -(1 << 31)


def L(x):
    return np.asarray(x).tolist()


def backends(f, index):
    return [R.EPaxos(f, index), T.Rows(f, index)]


def entry(b, rep, num):
    row, lk, lb = b.entry(rep, num)
    return L(row), int(lk), L(lb)


@pytest.mark.parametrize("k", [0, 1])
def test_commit_overwrites_and_drops_any_leader_state(k):
    b = backends(2, 1)[k]
    d = [1, 2, 3, 4, 5]
    b.lead([[1, 0, 0, 1, 7, 0, 0, 0] + d])
    b.commit([[1, 0, 9, 4, 1, 1, 1, 1, 1]])                              # CommittedEntry(triple) (:826-827)
    assert entry(b, 1, 0)[:2] == ([4, -1, -1, -1, -1, 9, 4, 1, 1, 1, 1, 1], 0)   # leaderStates -= instance (:831)
    b.commit([[1, 0, 10, 5, 2, 2, 2, 2, 2]])                             # no check: a Committed entry is replaced
    assert entry(b, 1, 0)[0] == [4, -1, -1, -1, -1, 10, 5, 2, 2, 2, 2, 2]
    b.prepare_phase([[2, 0]])
    assert entry(b, 2, 0)[1] == 3
    b.commit([[2, 0, 3, 0, 0, 0, 0, 0, 0]])                              # Preparing is dropped too
    assert entry(b, 2, 0)[1] == 0


@pytest.mark.parametrize("k", [0, 1])
def test_nack_raises_largest_ballot_and_arms_recovery_below_the_nack(k):
    b = backends(2, 1)[k]
    b.lead([[1, 0, 0, 1, 7, 0, 0, 0] + [0] * 5])
    ev = b.nack([[1, 0, 0, 1], [1, 0, 0, 2], [1, 1, 5, 0]])
    # (0,1) >= (0,1): no (:1589-1597); (0,1) < (0,2): recover (:1623-1629); not leading (1,1) (:1581-1587)
    assert L(ev) == [[0], [1], [0]]
    assert entry(b, 0, 0)[2] == [5, 0]                                   # largestBallot = max (:1578), every Nack
    st, _, out = b.prepare_phase([[2, 0]])
    assert L(out) == [[6, 1]]
    assert L(b.nack([[2, 0, 6, 1], [2, 0, 6, 2]])) == [[0], [1]]         # Preparing is a leader kind (:1609-1617)


@pytest.mark.parametrize("k", [0, 1])
def test_prepare_decision_table_and_inclusive_nack(k):
    b = backends(2, 1)[k]
    z = [0] * 5
    # lead does not touch largestBallot: entries at (5,1), largestBallot still (-1,-1)
    b.lead([[1, 0, 5, 1, 7, 2, 0, 0] + [1, 1, 1, 1, 1], [1, 1, 5, 1, 8, 0, 0, 0] + z])
    # a Nacked Prepare carries largestBallot AFTER its own ballot is folded in (:1637 before :1652): (4,3), not (0,1)
    r = b.prepare([[1, 0, 4, 3]])
    assert L(r) == [[2, 0, 4, 3, -1, -1, 0, 0, 0] + z]
    assert entry(b, 1, 0)[0][:3] == [2, 5, 1]                            # a Nack changes nothing
    # row 0 of the batch raises largestBallot to (6,0) before row 1's Nack is built; None -> NoCommand (:1654-1669)
    r = b.prepare([[2, 0, 6, 0], [1, 1, 4, 4]])
    assert L(r) == [[1, 0, 6, 0, -1, -1, 0, 0, 0] + z, [2, 0, 6, 0, -1, -1, 0, 0, 0] + z]
    assert entry(b, 2, 0)[0] == [1, 6, 0, -1, -1, 0, 0] + z
    # PreAccepted, ballot >= entry ballot: PrepareOk with the vote ballot, status and triple; ballot := prepare's
    r = b.prepare([[1, 0, 7, 0]])
    assert L(r) == [[1, 1, 7, 0, 5, 1, 1, 7, 2, 1, 1, 1, 1, 1]]          # yielded: (7,0) > leader ballot (5,1)
    assert entry(b, 1, 0)[:2] == ([2, 7, 0, 5, 1, 7, 2, 1, 1, 1, 1, 1], 0)
    # Accepted -> status Accepted; NoCommand with an equal ballot -> PrepareOk NotSeen again (`<`, :1676)
    b.accept([[3, 0, 2, 2, 9, 4] + [3, 3, 3, 3, 3]])
    r = b.prepare([[3, 0, 8, 2], [2, 0, 6, 0]])
    assert L(r) == [[1, 0, 8, 2, 2, 2, 2, 9, 4, 3, 3, 3, 3, 3], [1, 0, 6, 0, -1, -1, 0, 0, 0] + z]
    # Committed -> Commit(triple), no state change (:1746-1755)
    b.commit([[4, 0, 5, 6, 1, 0, 1, 0, 1]])
    assert L(b.prepare([[4, 0, 0, 0]])) == [[3, 0, -1, -1, -1, -1, 0, 5, 6, 1, 0, 1, 0, 1]]
    # yielded although Nacked: leader Preparing at (9,1) (the floored largestBallot (8,2) + 1), entry at (12,1)
    b.lead([[0, 1, 12, 1, 4, 0, 0, 0] + z])
    st, _, out = b.prepare_phase([[0, 1]])
    assert L(out) == [[9, 1]]
    r = b.prepare([[0, 1, 10, 3]])
    assert L(r) == [[2, 1, 10, 3, -1, -1, 0, 0, 0] + z]                  # yield (:1645-1649) precedes the Nack
    assert entry(b, 0, 1)[1] == 0


@pytest.mark.parametrize("k", [0, 1])
def test_prepare_nack_is_floored_at_ballot_zero_index(k):
    b = backends(2, 3)[k]
    b.lead([[3, 0, 0, 4, 1, 0, 0, 0] + [0] * 5])
    # largestBallot (-1,-1) -> with (0,2) folded in (0,2); the reference starts it at (0,3) (:458)
    assert L(b.prepare([[3, 0, 0, 2]]))[0][:4] == [2, 0, 0, 3]
    assert entry(b, 3, 0)[2] == [0, 2]                                   # the stored value is not floored


@pytest.mark.parametrize("k", [0, 1])
def test_prepare_phase_ballots(k):
    b = backends(2, 3)[k]
    st, _, out = b.prepare_phase([[0, 0], [1, 0], [2, 0]])
    # Ballot(largestBallot.ordering + 1, index) (:976) with largestBallot floored at (0,3), raised per row
    assert st == 0 and L(out) == [[1, 3], [2, 3], [3, 3]]
    assert entry(b, 1, 0) == ([0, -1, -1, -1, -1, 0, 0, 0, 0, 0, 0, 0], 3, [3, 3])   # cmdLog untouched
    b.preaccept([[4, 0, 7, 2, 1, 0] + [0] * 10])
    assert L(b.prepare_phase([[4, 0]])[2]) == [[8, 3]]
    b.preaccept([[4, 1, 0x7ffffff0, 0, 1, 0] + [0] * 10])
    st, i, _ = b.prepare_phase([[0, 1]])
    assert (st, i) == (-7, 0)                                            # an ordering past FPX_MAX_ROUND


@pytest.mark.parametrize("k", [0, 1])
def test_prepareok_decision(k):
    b = backends(2, 0)[k]
    st, _, out = b.prepare_phase([[0, 0], [0, 1], [0, 2], [0, 3]])
    assert L(out) == [[1, 0], [2, 0], [3, 0], [4, 0]]
    # (0,0): max vote ballot (0,1) held by an Accepted (11) and a PreAccepted (22) response; the Accepted branch
    # (:1813) never matches, the fast path (:1836) needs ballot (0,0): restart with the PreAccepted command
    st, _, ev = b.prepareok([[0, 0, 1, 0, 1, 0, 1, 2, 11], [0, 0, 1, 0, 3, -1, -1, 0, 0], [0, 0, 1, 0, 2, 0, 1, 1, 22]])
    assert st == 0 and L(ev) == [[0, 0, 0, 0], [0, 0, 0, 0], [1, 1, 0, 22]]
    assert entry(b, 0, 0)[1] == 0                                        # leads nothing until the caller's lead
    # (0,1): two PreAccepted at the max vote ballot: the lowest replica index; a quorum split over two calls
    assert L(b.prepareok([[0, 1, 2, 0, 4, 1, 1, 1, 44], [0, 1, 2, 0, 0, 0, 0, 1, 0]])[2]) == [[0] * 4, [0] * 4]
    assert L(b.prepareok([[0, 1, 2, 0, 3, 1, 1, 1, 33]])[2]) == [[1, 2, 0, 33]]
    # (0,2): only Accepted and NotSeen -> Noop
    st, _, ev = b.prepareok([[0, 2, 3, 0, 1, 0, 0, 2, 5], [0, 2, 3, 0, 2, -1, -1, 0, 0], [0, 2, 3, 0, 3, -1, -1, 0, 0]])
    assert L(ev)[2] == [1, 3, 0, NOOP]
    # (0,3): an older ballot is ignored, a newer one fails logger.checkLt (:1792) at its index
    st, i, ev = b.prepareok([[0, 3, 3, 0, 1, -1, -1, 0, 0], [0, 3, 5, 0, 2, -1, -1, 0, 0]])
    assert (st, i) == (-14, 1) and L(ev)[0] == [0, 0, 0, 0]


@pytest.mark.parametrize("k", [0, 1])
def test_slow_path_timer(k):
    b = backends(2, 0)[k]
    d = [1, 2, 3, 4, 5]
    b.lead([[0, 0, 0, 0, 7, 1, 0, 0] + d, [0, 1, 0, 0, 8, 1, 0, 0] + d])
    assert L(b.slow_path_timer([[0, 0, 0, 0]])) == [[0, 0] + [0] * 5]    # no timer armed yet
    ev = b.preacceptok([[0, 0, 0, 0, 1, 2] + [9, 0, 0, 0, 0], [0, 0, 0, 0, 2, 0] + [0, 9, 0, 0, 0]])
    assert L(ev)[1][0] == 3                                              # TIMER (:1353-1364)
    assert L(b.slow_path_timer([[0, 0, 1, 0]])) == [[0, 0] + [0] * 5]    # another ballot: that timer was stopped
    ev = b.slow_path_timer([[0, 0, 0, 0]])                               # preAcceptingSlowPath (:796-813)
    assert L(ev) == [[2, 2, 9, 9, 3, 4, 5]]
    assert entry(b, 0, 0)[:2] == ([3, 0, 0, 0, 0, 7, 2, 9, 9, 3, 4, 5], 2)
    assert L(b.slow_path_timer([[0, 0, 0, 0]])) == [[0, 0] + [0] * 5]    # Accepting now


def _run_trace(f, seed, steps):
    index = seed % (2 * f + 1)
    ora, tr = R.EPaxos(f, index), T.Rows(f, index)
    trace = Trace(f, index, 4, seed, ora)
    for _ in range(steps):
        call, rows = trace.step()
        rows = np.asarray(rows, dtype=np.int32)
        a, c = getattr(ora, call)(rows), getattr(tr, call)(rows)
        if call in ("prepare_phase", "prepareok"):
            assert a[0] == c[0] == 0, (call, a, c)
            a, c = a[2], c[2]
        if a is not None and not isinstance(a, tuple):
            assert L(a) == L(c), (call, rows.tolist())
        elif call == "lead":
            assert a == c == (0, -1)
        trace.observe(call, rows, a)
        for r in rows:
            assert entry(ora, int(r[0]), int(r[1])) == entry(tr, int(r[0]), int(r[1])), (call, r.tolist())
    return trace


@pytest.mark.parametrize("f", [1, 2, 3])
def test_oracle_matches_transcription_on_mixed_traces(f):
    for seed in range(6):
        _run_trace(f, 100 * f + seed, 300)
