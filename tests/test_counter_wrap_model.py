"""The renormalization of 32-bit delivery numbers, checked on the CPU against the oracle (no GPU).  The engines
number deliveries with a 32-bit counter; before a call of n deliveries could come within 16 of the wrap, every
recorded first-delivery stamp collapses to 0 and the numbering restarts at 1 (fpx_replica_misc.cuh,
renormalize_stamps_kernel).  The claim that makes this sound: a key still pending holds fewer stamps than a
quorum, so the order among its old stamps never decides a completing vote again, and every old stamp stays
below every new one.  Here each decision rule the kernels evaluate is run with such a counter started just
below the wrap, so that the collapse lands at a random call boundary of the trace, and its decisions must equal
the sequential handlers':

  tally         (f+1)-th smallest stamp of a key, or the grid's max over rows of the row minimum (fpx_tally.cuh)
  ranges        every acceptor group of the NoopRange reaches its quorum (fpx_ranges.cuh, range_tally_kernel)
  EPaxos        a response decides when before < q <= after (fpx_epaxos.cuh, ep_response_decide_kernel)"""
import numpy as np
import pytest

import epaxos_recovery_oracle as R
import harness as H
from frankenpaxos_b200 import traces as T
from frankenpaxos_b200.engine import P2A_RANGE
from oracle import fpx_oracle_py as O

EMPTY = np.uint32(0xFFFFFFFF)


class Counter32:
    """The host side of one 32-bit numbering and the stamp tables it collapses."""

    def __init__(self, start, tables):
        self.seq = start
        self.tables = tables            # uint32 arrays whose non-EMPTY entries are stamps of this numbering
        self.collapses = []             # call indices at which the numbering restarted
        self.calls = 0

    def take(self, n):
        """first number of a call of n deliveries"""
        if self.seq > 0xFFFFFFFF - n - 16:
            for t in self.tables:
                t[t != EMPTY] = 0
            self.seq = 1
            self.collapses.append(self.calls)
        first = self.seq
        self.seq += n
        self.calls += 1
        return first


def start_at(sizes, j):
    """the start from which calls of these sizes restart the numbering at call j and at no other call"""
    return 0xFFFFFFFF - 16 - sum(sizes[:j]) - (sizes[j] + 1) // 2


def stamp_first(table, index, first, n):
    """stamps first + i of deliveries i at `index` (a tuple of arrays), keeping the smallest per cell"""
    np.minimum.at(table, index, (np.uint64(first) + np.arange(n, dtype=np.uint64)).astype(np.uint32))


def closed_form(stamps, value, f, flexible, groups, per_group, lo, hi):
    if not flexible:
        c = np.sort(stamps, axis=1)[:, f]
    else:
        c = stamps.reshape(len(stamps), groups, per_group).min(axis=2).max(axis=1)
    hit = np.nonzero((c >= lo) & (c < hi))[0]
    order = hit[np.argsort(c[hit], kind="stable")]
    return [(int(s), int(value[s])) for s in order]


@pytest.mark.parametrize("name", ["cfg1", "cfg2", "cfg3"] + list(H.WIDE_SHAPES))
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_tally_rule_across_the_collapse(name, seed):
    cfg = H.WIDE_SHAPES[name] if name in H.WIDE_SHAPES else T.config_by_name(name)[0]
    f, G, A, flexible = cfg["f"], cfg["num_acceptor_groups"], cfg["acceptors_per_group"], cfg["flexible"]
    n_slots = 2000
    g = T.rng(300 + seed)
    a, _, b = T.workload(seed, cfg, n_slots)
    votes = np.concatenate([b, b[g.integers(0, len(b), len(b) // 3)]])
    votes = votes[g.permutation(len(votes))]
    ora = O.MultiPaxos(f, G, A, flexible, cfg["num_leaders"], cfg["num_replicas"])
    assert ora.arm(a) == (0, -1)
    stamps = np.full((n_slots, G * A if flexible else A), EMPTY, dtype=np.uint32)
    value = np.zeros(n_slots, dtype=np.int64)
    value[a["slot"]] = a["value_id"]
    chunks = np.split(votes, np.sort(g.choice(np.arange(1, len(votes)), size=9, replace=False)))
    at = int(g.integers(1, len(chunks)))
    ctr = Counter32(start_at([len(c) for c in chunks], at), [stamps])
    for chunk in chunks:
        st, _, oc = ora.proxyleader_phase2b(chunk)
        assert st == 0
        first = ctr.take(len(chunk))
        v = chunk["group"] * A + chunk["acceptor"] if flexible else chunk["acceptor"]
        stamp_first(stamps, (chunk["slot"], v), first, len(chunk))
        assert oc.tolist() == closed_form(stamps, value, f, flexible, G, A, first, first + len(chunk))
    assert ctr.collapses == [at]


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_range_rule_across_the_collapse(seed):
    """A NoopRange is chosen by the first delivery after which every acceptor group of its leader group holds
    f+1 votes: its completing number is the max over groups of the group's (f+1)-th smallest stamp."""
    f, LG, AG, per, cap = 1, 2, 3, 3, 1 << 14
    g = T.rng(400 + seed)
    ora = O.MultiPaxos(f, AG, per, False, 2, 2, mencius_leader_groups=LG)
    ranges = [(lg + LG * 30 * k, lg + LG * 30 * (k + 1)) for lg in range(LG) for k in range(60)]
    arm = np.array([(s, e, 0, -1) for s, e in ranges], dtype=P2A_RANGE)
    assert ora.arm_range(arm, cap) == (0, -1)
    recs = np.array([(s, e, 0, ((s % LG * AG + ag) << 16) | k) for s, e in ranges for ag in range(AG)
                     for k in range(per)], dtype=P2A_RANGE)
    st, _, votes, _ = ora.acceptor_noop_range(recs[g.permutation(len(recs))], cap)
    assert st == 0
    votes = np.concatenate([votes, votes[g.integers(0, len(votes), len(votes) // 3)]])
    votes = votes[g.permutation(len(votes))]
    row = {s: i for i, (s, _) in enumerate(ranges)}
    stamps = np.full((len(ranges), AG * per), EMPTY, dtype=np.uint32)
    chunks = np.split(votes, np.sort(g.choice(np.arange(1, len(votes)), size=7, replace=False)))
    at = int(g.integers(1, len(chunks)))
    ctr = Counter32(start_at([len(c) for c in chunks], at), [stamps])
    n_chosen = 0
    for chunk in chunks:
        st, _, oc = ora.range_phase2b(chunk)
        assert st == 0
        first = ctr.take(len(chunk))
        r = np.array([row[s] for s in chunk["slot_start"]])
        stamp_first(stamps, (r, ((chunk["dst"] >> 16) % AG) * per + (chunk["dst"] & 0xFFFF)), first, len(chunk))
        c = np.sort(stamps.reshape(len(ranges), AG, per), axis=2)[:, :, f].max(axis=1)
        hit = np.nonzero((c >= first) & (c < first + len(chunk)))[0]
        want = [ranges[i] for i in hit[np.argsort(c[hit], kind="stable")]]
        assert [tuple(x) for x in oc.tolist()] == want
        n_chosen += len(oc)
    assert n_chosen == len(ranges)
    assert ctr.collapses == [at]


@pytest.mark.parametrize("kind", ["acceptok", "prepareok"])
@pytest.mark.parametrize("f", [1, 2, 3])
def test_epaxos_threshold_rule_across_the_collapse(f, kind):
    """Per instance, one first-delivery stamp per replica (AcceptOk: the leader's own is 0 from the start); a
    response decides (commit, or the PrepareOk restart) iff before < f+1 <= before + 1, before counting the
    stamps below its own.  Rounds of responses with re-deliveries, one round per call."""
    n, idx, K = 2 * f + 1, 0, 60
    g = T.rng(500 + 10 * f + (kind == "prepareok"))
    ora = R.EPaxos(f, idx)
    z = [0] * n
    stamps = np.full((K, n), EMPTY, dtype=np.uint32)
    if kind == "acceptok":
        ora.lead(np.array([[idx, k, 1, idx, k, 0, 1, 0] + z for k in range(K)], dtype=np.int32))
        others = [r for r in range(n) if r != idx]
        ev = ora.preacceptok(np.array([[idx, k, 1, idx, r, 0] + z for k in range(K) for r in others[:f]], dtype=np.int32))
        assert (ev[:, 0] == 2).sum() == K                       # the slow path: every instance is Accepting
        stamps[:, idx] = 0
        senders, ballot = others, {k: (1, idx) for k in range(K)}
        row = lambda k, s: [idx, k, 1, idx, s, 0]
        decided = 4
    else:
        st, _, b = ora.prepare_phase(np.array([[1, k] for k in range(K)], dtype=np.int32))
        assert st == 0
        senders, ballot = list(range(n)), {k: (int(b[k][0]), int(b[k][1])) for k in range(K)}
        row = lambda k, s: [1, k, ballot[k][0], ballot[k][1], s, -1, -1, 0, 0]
        decided = 1
    calls = []
    for _ in range(6):
        rows = [(k, s) for k in range(K) for s in senders if g.random() < 0.3]
        calls.append([rows[i] for i in g.permutation(len(rows))])
    at = int(g.integers(1, len(calls)))
    ctr = Counter32(start_at([len(c) for c in calls], at), [stamps])
    for rows in calls:
        arr = np.array([row(k, s) for k, s in rows], dtype=np.int32)
        if kind == "acceptok":
            ev = ora.acceptok(arr)
        else:
            st, _, ev = ora.prepareok(arr)
            assert st == 0
        first = ctr.take(len(rows))
        inst = np.array([k for k, _ in rows])
        snd = np.array([s for _, s in rows])
        fresh = stamps[inst, snd] == EMPTY
        stamp_first(stamps, (inst, snd), first, len(rows))
        seq = (np.uint64(first) + np.arange(len(rows), dtype=np.uint64)).astype(np.uint32)
        before = (stamps[inst] < seq[:, None]).sum(axis=1)
        want = fresh & (before < f + 1) & (before + 1 >= f + 1)
        assert (ev[:, 0] == decided).tolist() == want.tolist()
    assert ctr.collapses == [at]
