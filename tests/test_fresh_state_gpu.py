"""The arm's fast path: a batch certified as fresh keys in strict slot order is armed with plain row stores,
anything else takes the per-record CAS.  Every case asserts which path the arm took (Engine.last_arm_path) and
that every reply, Chosen stream, error and the replica log equal the oracle's, on both tally paths.  Marked gpu."""
import numpy as np
import pytest

import harness as H
from frankenpaxos_b200 import MENCIUS, P2B, Engine, FpxError
from frankenpaxos_b200 import traces as T
from oracle import fpx_oracle_py as O

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True, params=["auto", "exact"])
def tally_path(request, monkeypatch):
    monkeypatch.setenv("FPX_TALLY_PATH", request.param)
    return request.param


SHAPES = {"cfg2": T.config_by_name("cfg2")[0], "cfg3": T.config_by_name("cfg3")[0],
          "maj15": H.WIDE_SHAPES["maj15"], "groups2x15": H.WIDE_SHAPES["groups2x15"]}


def grid(cfg):
    return cfg["f"], cfg["num_acceptor_groups"], cfg["acceptors_per_group"], cfg["flexible"]


def arm(eng, ora, recs, path):
    H.arm(eng, ora, recs)
    assert eng.last_arm_path == path


def vote(eng, ora, cfg, g, slots, rnd, values, extra_votes=None):
    """Phase2as to the acceptors, their votes shuffled (plus extra_votes) to the tally, Chosen to the replica."""
    p = T.phase2as(g, slots, *grid(cfg), rnd, values)
    ob, on = H.phase2a(eng, ora, T.shuffled(g, p))
    votes = ob if extra_votes is None else np.concatenate([ob, extra_votes])
    st, c = H.phase2b(eng, ora, T.shuffled(g, votes))
    H.replica(eng, ora, c)
    return st, c


@pytest.mark.parametrize("shape", list(SHAPES))
def test_fresh_windows_through_the_ring(shape):
    """Ten windows of 3000 slots through a 4096-slot ring, each retired behind the watermark: every window's
    arm batch is in slot order over never-touched or recycled rows, so every one takes the fast path -- also
    when it wraps the ring -- and the state it leaves is the CAS path's."""
    cfg = SHAPES[shape]
    eng = Engine(slot_capacity=4096, max_batch=1 << 15, overflow_capacity=1 << 8, **cfg)
    ora = O.MultiPaxos(*grid(cfg), cfg["num_leaders"], cfg["num_replicas"])
    g = T.rng(77 + len(shape))
    step = 3000
    for w in range(10):
        slots = np.arange(w * step, (w + 1) * step, dtype=np.int32)
        values = slots * 3 + w
        arm(eng, ora, T.arms(slots, w, values), "fresh")
        st, c = vote(eng, ora, cfg, g, slots, w, values)
        assert st == 0 and len(c) == step
        H.compare_acceptors(eng, ora, cfg, w * step, step)
        H.compare_log(eng, ora, w * step, step)
        eng.retire_below((w + 1) * step)
    eng.close()


def test_mencius_fresh_batch():
    """Compartmentalized Mencius (two leader groups): an ordered arm batch takes the fast path; f + 1 votes per
    slot complete every key."""
    f, LG, AG, per = 1, 2, 1, 3
    eng = Engine(f, AG, per, num_leaders=2, num_replicas=2, slot_capacity=8192, max_batch=1 << 15, protocol=MENCIUS,
                 num_leader_groups=LG)
    ora = O.MultiPaxos(f, AG, per, False, 2, 2, mencius_leader_groups=LG)
    g = T.rng(5)
    slots = np.arange(0, 5000, dtype=np.int32)
    arm(eng, ora, T.arms(slots, 0, slots + 11), "fresh")
    voters = np.array([g.permutation(per)[: f + 1] for _ in slots])
    b = np.zeros(len(slots) * (f + 1), dtype=P2B)
    b["group"] = (np.repeat(slots, f + 1) % LG) * AG
    b["acceptor"] = voters.reshape(-1)
    b["slot"] = np.repeat(slots, f + 1)
    b["round"] = 0
    st, c = H.phase2b(eng, ora, T.shuffled(g, b))
    assert st == 0 and len(c) == len(slots)
    H.replica(eng, ora, c)
    H.compare_log(eng, ora, 0, len(slots))
    eng.close()


def test_batches_the_fast_path_refuses():
    """Each batch breaks one condition of the certificate and is armed by the CAS path, with the oracle's
    result: a repeated slot, a second round of a fresh slot, slots out of order, a re-arm below the fresh
    frontier, an out-of-range slot at the end (error index), and an ordered batch right after them."""
    cfg = T.config_by_name("cfg2")[0]
    eng = Engine(slot_capacity=1 << 14, max_batch=1 << 14, overflow_capacity=1 << 8, **cfg)
    ora = O.MultiPaxos(*grid(cfg), cfg["num_leaders"], cfg["num_replicas"])
    g = T.rng(11)
    # a repeated slot (same value: the second arm is ignored)
    s = np.arange(0, 1000, dtype=np.int32)
    a = T.arms(s, 0, s + 1)
    arm(eng, ora, np.concatenate([a[:500], a[499:]]), "cas")
    assert vote(eng, ora, cfg, g, s, 0, s + 1)[0] == 0
    # a second round of a fresh slot, right behind its first round
    s = np.arange(1000, 2000, dtype=np.int32)
    a = T.arms(s, 0, s + 1)
    a2 = T.arms(s[300:301], 1, s[300:301] + 7)
    arm(eng, ora, np.concatenate([a[:301], a2, a[301:]]), "cas")
    st, _ = vote(eng, ora, cfg, g, s, 0, s + 1, extra_votes=T.votes_of(T.phase2as(g, s[300:301], *grid(cfg), 1,
                                                                                      s[300:301] + 7)))
    assert st == 0
    # out of order
    s = np.arange(2000, 3000, dtype=np.int32)
    arm(eng, ora, T.arms(s, 0, s + 1)[g.permutation(len(s))], "cas")
    assert vote(eng, ora, cfg, g, s, 0, s + 1)[0] == 0
    # ordered, but it re-arms keys below the frontier (2500 .. 2999 exist) before new ones
    s = np.arange(2500, 4000, dtype=np.int32)
    arm(eng, ora, T.arms(s, 0, s + 1), "cas")
    assert vote(eng, ora, cfg, g, s[500:], 0, s[500:] + 1)[0] == 0
    # ordered, and its last slot lies outside the engine (the oracle has no capacity): FPX_ERR_SLOT_RANGE at that
    # index, the rest armed
    s = np.append(np.arange(4000, 4100, dtype=np.int32), 1 << 20)
    with pytest.raises(FpxError) as ei:
        eng.proxyleader_arm(T.arms(s, 0, s + 1))
    assert (ei.value.status, ei.value.index) == (-6, 100) and eng.last_arm_path == "cas"
    assert ora.arm(T.arms(s[:-1], 0, s[:-1] + 1))[0] == 0
    assert vote(eng, ora, cfg, g, s[:-1], 0, s[:-1] + 1)[0] == 0
    # after all of them an ordered batch of new keys is fresh again
    s = np.arange(4100, 6000, dtype=np.int32)
    arm(eng, ora, T.arms(s, 0, s + 1), "fresh")
    assert vote(eng, ora, cfg, g, s, 0, s + 1)[0] == 0
    H.compare_acceptors(eng, ora, cfg, 0, 6000)
    H.compare_log(eng, ora, 0, 6000)
    eng.close()


def test_stray_vote_makes_its_row_stale_until_reset():
    """A vote for a slot nobody armed is fatal (the oracle's logger.fatal), but the tally has stamped it into
    the unarmed row: the frontier moves past it, so an ordered arm over that slot takes the CAS path.  After
    fpx_reset the rows are fresh again and the same ordered batch takes the fast path, bit-exact."""
    cfg = T.config_by_name("cfg2")[0]
    eng = Engine(slot_capacity=1 << 13, max_batch=1 << 13, overflow_capacity=1 << 8, **cfg)
    ora = O.MultiPaxos(*grid(cfg), cfg["num_leaders"], cfg["num_replicas"])
    g = T.rng(3)
    stray = np.zeros(1, dtype=P2B)
    stray[0] = (0, 1, 700, 0)
    st, _ = H.phase2b(eng, ora, stray)
    assert st != 0
    s = np.arange(0, 2000, dtype=np.int32)
    H.arm(eng, O.MultiPaxos(*grid(cfg), cfg["num_leaders"], cfg["num_replicas"]), T.arms(s, 0, s + 1))
    assert eng.last_arm_path == "cas"
    eng.reset()
    ora = O.MultiPaxos(*grid(cfg), cfg["num_leaders"], cfg["num_replicas"])
    arm(eng, ora, T.arms(s, 0, s + 1), "fresh")
    st, c = vote(eng, ora, cfg, g, s, 0, s + 1)
    assert st == 0 and len(c) == len(s)
    H.compare_acceptors(eng, ora, cfg, 0, len(s))
    H.compare_log(eng, ora, 0, len(s))
    eng.close()


def test_phase1_snapshot_after_fast_path_votes():
    """Acceptor snapshots (what Phase1b reports) after fast-path arms and votes, then a leader change: the new
    round's arm of those slots is a second round of existing keys and goes through the CAS path."""
    cfg = T.config_by_name("cfg2")[0]
    eng = Engine(slot_capacity=1 << 13, max_batch=1 << 14, overflow_capacity=1 << 10, **cfg)
    ora = O.MultiPaxos(*grid(cfg), cfg["num_leaders"], cfg["num_replicas"])
    g = T.rng(9)
    s = np.arange(0, 3000, dtype=np.int32)
    arm(eng, ora, T.arms(s, 0, s + 1), "fresh")
    p = T.phase2as(g, s, *grid(cfg), 0, s + 1)
    H.phase2a(eng, ora, T.shuffled(g, p))
    H.compare_acceptors(eng, ora, cfg, 0, len(s))
    s1 = s[:200]
    arm(eng, ora, T.arms(s1, 1, s1 + 5), "cas")
    st, c = vote(eng, ora, cfg, g, s1, 1, s1 + 5)
    assert st == 0 and len(c) == len(s1)
    H.compare_acceptors(eng, ora, cfg, 0, len(s))
    H.compare_log(eng, ora, 0, len(s))
    eng.close()
