"""Parity of the CUDA path (through the C ABI) against the CPU oracle, bit-exact:
Phase2b / Nack / Chosen streams INCLUDING ORDER, error status + first offending
index, final acceptor state (round, maxVotedSlot, voteRound[], voteValue[]) and
replica log / watermark.  Marked gpu: needs an H100."""
import json
import os

import numpy as np
import pytest

import harness as H
from frankenpaxos_b200 import CHOSEN, NACK, P2A, P2B, Engine, FpxError, dst
from frankenpaxos_b200 import traces as T
from oracle import fpx_oracle_py as O

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True, params=["auto", "exact"])
def tally_path(request, monkeypatch):
    """Every test of this module runs twice: with the tally free to take its row sweep
    (steady-state batches) and forced onto the exact per-vote path (FPX_TALLY_PATH)."""
    monkeypatch.setenv("FPX_TALLY_PATH", request.param)
    return request.param


def D(g, a):
    return (g << 16) | a


def recs(dtype, *rows):
    return np.array(list(rows), dtype=dtype)


# --------------------------------------------------------------------------- golden vectors on the GPU
@pytest.mark.parametrize("kind", ["grid", "simple_majority"])
def test_quorum_predicates_golden(golden_dir, kind):
    """GridTest.scala:11-102 / SimpleMajorityTest.scala:11-63 replayed on the CUDA
    predicate kernel (fpx_quorum_eval)."""
    g = json.load(open(os.path.join(golden_dir, "quorums.json")))[kind]
    if kind == "grid":
        members = [x for row in g["members"] for x in row]
        eng = Engine(1, 2, 3, flexible=True, slot_capacity=8, max_batch=1024)
    else:
        members = g["members"]
        eng = Engine(2, 1, 5, slot_capacity=8, max_batch=1024)
    index = {m: i for i, m in enumerate(members)}
    for which, pred in enumerate(["isReadQuorum", "isWriteQuorum", "isSuperSetOfReadQuorum",
                                  "isSuperSetOfWriteQuorum"]):
        cases = [c for c in g["cases"] if c["pred"] == pred]
        masks = []
        for c in cases:
            m = 0
            for x in c["set"]:
                m |= (1 << index[x]) if x in index else (1 << 31)
            masks.append(m)
        got = eng.quorum_eval(which, np.array(masks, dtype=np.uint32))
        for c, r in zip(cases, got):
            assert int(r) == int(c["expect"]), (g["source"], c["line"], c)
    # `require` on non-members (Grid.scala:36-39)
    assert eng.quorum_eval(1, np.array([(1 << 31) | 0b001001], dtype=np.uint32))[0] == 2
    eng.close()


# --------------------------------------------------------------------------- hand-derived micro traces
def test_micro_trace_survey_8g():
    cfg = dict(f=1, num_acceptor_groups=1, acceptors_per_group=3, flexible=False, num_leaders=2, num_replicas=2)
    eng, ora = H.make_pair(cfg, 64)
    H.arm(eng, ora, recs(P2A, (0, 0, 100, -1)))
    b, _ = H.phase2a(eng, ora, recs(P2A, (0, 0, 100, D(0, 0))))
    H.phase2b(eng, ora, b)
    H.phase2b(eng, ora, b)                      # duplicate vote
    b2, _ = H.phase2a(eng, ora, recs(P2A, (0, 0, 100, D(0, 2))))
    st, c = H.phase2b(eng, ora, b2)
    assert c.tolist() == [(0, 100)]
    H.phase2b(eng, ora, recs(P2B, (0, 1, 0, 0)))  # late vote, Done
    H.phase2a(eng, ora, recs(P2A, (1, 3, 101, D(0, 0))))
    b, n = H.phase2a(eng, ora, recs(P2A, (2, 0, 102, D(0, 0))))
    assert n.tolist() == [(0, 3)]
    H.phase2a(eng, ora, recs(P2A, (0, 3, 109, D(0, 0))))
    H.compare_acceptors(eng, ora, cfg, 0, 8)
    st, _ = H.phase2b(eng, ora, recs(P2B, (0, 1, 0, 0), (0, 0, 5, 0)))
    assert st == -4
    eng.close()


def test_whole_micro_trace_in_single_batches():
    """Same deliveries as above but batched: order semantics inside one launch."""
    cfg = dict(f=1, num_acceptor_groups=1, acceptors_per_group=3, flexible=False, num_leaders=2, num_replicas=2)
    eng, ora = H.make_pair(cfg, 64)
    H.arm(eng, ora, recs(P2A, (0, 0, 100, -1), (1, 3, 101, -1), (0, 3, 109, -1), (0, 0, 555, -1)))
    b, n = H.phase2a(eng, ora, recs(P2A, (0, 0, 100, D(0, 0)), (0, 0, 100, D(0, 2)), (1, 3, 101, D(0, 0)),
                                    (2, 0, 102, D(0, 0)), (0, 3, 109, D(0, 0)), (0, 3, 777, D(0, 0)),
                                    (0, 3, 3, D(0, 0))))
    H.compare_acceptors(eng, ora, cfg, 0, 8)
    votes = recs(P2B, (0, 0, 0, 0), (0, 0, 0, 0), (0, 2, 0, 0), (0, 1, 0, 0), (0, 0, 1, 3), (0, 0, 0, 3),
                 (0, 1, 0, 3), (0, 1, 1, 3))
    st, c = H.phase2b(eng, ora, votes)
    assert c.tolist() == [(0, 100), (0, 109), (1, 101)]
    H.replica(eng, ora, c)
    H.compare_log(eng, ora, 0, 8)
    eng.close()


def test_grid_and_bad_acceptor():
    cfg = dict(f=1, num_acceptor_groups=2, acceptors_per_group=3, flexible=True, num_leaders=2, num_replicas=2)
    eng, ora = H.make_pair(cfg, 64)
    H.arm(eng, ora, recs(P2A, (0, 0, 7, -1), (1, 0, 8, -1), (2, 0, 9, -1)))
    st, c = H.phase2b(eng, ora, recs(P2B, (0, 1, 0, 0), (0, 2, 0, 0), (1, 0, 0, 0), (1, 1, 0, 0)))
    assert c.tolist() == [(0, 7)]
    # foreign acceptor on a Done key is ignored; on a Pending key it is `require`
    st, c = H.phase2b(eng, ora, recs(P2B, (5, 0, 0, 0), (0, 0, 1, 0)))
    assert st == 0
    st, c = H.phase2b(eng, ora, recs(P2B, (1, 1, 1, 0), (0, 0, 2, 0), (5, 0, 2, 0), (9, 9, 2, 0)))
    assert st == -5
    eng.close()


def test_bad_acceptor_after_completion_in_same_batch_is_ignored():
    cfg = dict(f=1, num_acceptor_groups=2, acceptors_per_group=3, flexible=True, num_leaders=2, num_replicas=2)
    eng, ora = H.make_pair(cfg, 64)
    H.arm(eng, ora, recs(P2A, (3, 0, 7, -1)))
    st, c = H.phase2b(eng, ora, recs(P2B, (0, 1, 3, 0), (1, 1, 3, 0), (7, 7, 3, 0)))
    assert st == 0 and c.tolist() == [(3, 7)]
    eng.close()


def test_two_live_rounds_and_overflow_table():
    cfg = dict(f=1, num_acceptor_groups=1, acceptors_per_group=3, flexible=False, num_leaders=2, num_replicas=2)
    eng, ora = H.make_pair(cfg, 64)
    H.arm(eng, ora, recs(P2A, (4, 0, 40, -1), (4, 1, 41, -1), (4, 2, 42, -1), (5, 7, 50, -1)))
    st, c = H.phase2b(eng, ora, recs(P2B, (0, 0, 4, 1), (0, 0, 4, 0), (0, 1, 4, 1), (0, 2, 4, 0), (0, 2, 4, 2)))
    assert c.tolist() == [(4, 41), (4, 40)]
    H.replica(eng, ora, c)
    st, c = H.phase2b(eng, ora, recs(P2B, (0, 1, 4, 2), (0, 1, 5, 7), (0, 0, 5, 7)))
    assert c.tolist() == [(4, 42), (5, 50)]
    H.replica(eng, ora, c)
    H.compare_log(eng, ora, 0, 8)
    # unknown round of a known slot is fatal too
    st, _ = H.phase2b(eng, ora, recs(P2B, (0, 1, 4, 9)))
    assert st == -4
    eng.close()


def test_duplicate_arm_different_value_keeps_first_in_order():
    cfg = dict(f=1, num_acceptor_groups=1, acceptors_per_group=3, flexible=False, num_leaders=2, num_replicas=2)
    eng, ora = H.make_pair(cfg, 4096)
    n = 900                             # <= kMaxConflicts (1024) detections per batch
    a = np.zeros(2 * n, dtype=P2A)
    a["slot"] = np.concatenate([np.arange(n), np.arange(n)[::-1]])
    a["value_id"] = np.arange(2 * n) + 10
    a["dst"] = -1
    H.arm(eng, ora, a[:50])             # some keys exist before the conflicting batch
    H.arm(eng, ora, a)                  # every key armed twice with different values
    votes = T.votes_of(T.phase2as(T.rng(0), np.arange(n), 1, 1, 3, False))
    st, c = H.phase2b(eng, ora, votes)
    assert len(c) == n
    eng.close()


def test_same_cell_same_round_different_value_last_wins():
    cfg = dict(f=1, num_acceptor_groups=1, acceptors_per_group=3, flexible=False, num_leaders=2, num_replicas=2)
    eng, ora = H.make_pair(cfg, 4096)
    n = 300                             # <= kMaxConflicts (1024) detections per batch
    p = np.zeros(3 * n, dtype=P2A)
    p["slot"] = np.tile(np.arange(n), 3)
    p["round"] = 2
    p["value_id"] = T.rng(1).integers(0, 1 << 30, size=3 * n)
    p["dst"] = D(0, 1)
    H.phase2a(eng, ora, p[:100])
    H.phase2a(eng, ora, p)
    H.compare_acceptors(eng, ora, cfg, 0, n)
    eng.close()


def test_conflict_cap_is_reported_not_silently_wrong():
    """More than 1024 same-key/different-value collisions in ONE batch (only a
    faulty leader produces even one) exceed the in-kernel resolver: the engine
    must say FPX_ERR_CONFLICT, never return a wrong value (documented limit)."""
    eng = Engine(1, 1, 3, num_leaders=2, num_replicas=2, slot_capacity=8192, max_batch=1 << 16)
    n = 4000
    a = np.zeros(2 * n, dtype=P2A)
    a["slot"] = np.tile(np.arange(n), 2)
    a["value_id"] = np.arange(2 * n)
    with pytest.raises(FpxError) as ei:
        eng.proxyleader_arm(a)
    assert ei.value.status == -9
    eng.close()


# --------------------------------------------------------------------------- the tally's two paths
def test_tally_takes_the_sweep_in_steady_state_and_falls_back_otherwise(tally_path):
    """fpx_tally.cuh: a one-round batch over armed rows of that round is evaluated by the row
    sweep; a batch that mixes rounds, touches an unarmed row, hides a vote of another round
    behind an older stamp, or carries a foreign voter is evaluated per vote.  Same outputs."""
    cfg, _ = T.config_by_name("cfg2")
    n_slots = 6000
    eng, ora = H.make_pair(cfg, 3 * n_slots, max_batch=1 << 16, overflow_capacity=1 << 10)
    want = "sweep" if tally_path == "auto" else "exact"
    a, p, b = T.workload(5, cfg, n_slots)
    H.arm(eng, ora, a)
    ob, _ = H.phase2a(eng, ora, p)
    # votes of one key spread over several batches: completion decided by stamps of earlier batches
    for chunk in np.array_split(b, 7):
        st, c = H.phase2b(eng, ora, chunk)
        assert st == 0 and eng.last_tally_path == want
        H.replica(eng, ora, c)
    # duplicates of old votes only: nothing new is chosen, still a sweep
    st, c = H.phase2b(eng, ora, b[:500])
    assert st == 0 and len(c) == 0 and eng.last_tally_path == want
    # a second window in round 1; one batch mixes it with late round-0 votes -> exact
    a1, p1, b1 = T.workload(6, cfg, n_slots, slot0=n_slots, round_=1)
    H.arm(eng, ora, a1)
    mix = np.concatenate([b1[:3000], b[:10]])
    st, c = H.phase2b(eng, ora, mix)
    assert st == 0 and eng.last_tally_path == "exact"
    H.replica(eng, ora, c)
    st, c = H.phase2b(eng, ora, b1[3000:])
    assert st == 0 and eng.last_tally_path == want
    H.replica(eng, ora, c)
    H.compare_log(eng, ora, 0, 2 * n_slots)
    # a vote of round 1 for a round-0 key whose voter already voted: hidden behind the older stamp
    hidden = b[:1].copy()
    hidden["round"] = 1
    st, _ = H.phase2b(eng, ora, hidden)
    assert st == -4 and eng.last_tally_path == "exact"
    eng.close()


@pytest.mark.parametrize("order", ["by_slot", "reversed", "by_acceptor"])
def test_skewed_delivery_orders(tally_path, order):
    """Votes delivered in slot order, reversed, or one acceptor after the other (the last acceptor's votes
    complete every key: all completing votes in the last third of the batch) give the oracle's stream."""
    cfg, _ = T.config_by_name("cfg2")
    n_slots = 150000
    eng, ora = H.make_pair(cfg, n_slots, max_batch=3 * n_slots, overflow_capacity=1 << 10)
    a, p, b = T.workload(17, cfg, n_slots)
    H.arm(eng, ora, a)
    if order == "by_slot":
        b = b[np.argsort(b["slot"], kind="stable")]
    elif order == "reversed":
        b = b[np.argsort(b["slot"], kind="stable")][::-1].copy()
    else:
        b = b[np.lexsort((b["slot"], b["acceptor"]))]
    st, c = H.phase2b(eng, ora, b)
    assert st == 0 and len(c) == n_slots
    eng.close()


def test_sweep_error_paths_report_the_reference_index(tally_path):
    cfg, _ = T.config_by_name("cfg2")
    n_slots = 4000
    # an unarmed slot in the middle of the window: every one of its votes is fatal, the first is reported
    eng, ora = H.make_pair(cfg, n_slots)
    a, p, b = T.workload(8, cfg, n_slots)
    H.arm(eng, ora, a[a["slot"] != 1234])
    st, _ = H.phase2b(eng, ora, b)
    assert st == -4
    eng.close()


def test_sweep_window_far_larger_than_the_batch_uses_the_exact_path(tally_path):
    cfg, _ = T.config_by_name("cfg2")
    n_slots = 1 << 20
    eng, ora = H.make_pair(cfg, n_slots, max_batch=1 << 12)
    slots = np.array([3, n_slots - 5, 77777, 500000], dtype=np.int32)
    H.arm(eng, ora, T.arms(slots, 0, slots + 1))
    v = T.votes_of(T.phase2as(T.rng(1), slots, cfg["f"], 1, 5, False, 0, slots + 1))
    st, c = H.phase2b(eng, ora, v)
    assert st == 0 and len(c) == 4 and eng.last_tally_path == "exact"
    eng.close()


# --------------------------------------------------------------------------- BASELINE configs, seeded
@pytest.mark.parametrize("name,n_slots", [("cfg1", 128), ("cfg2", 20000), ("cfg3", 30000)])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_baseline_configs(name, n_slots, seed):
    cfg, _ = T.config_by_name(name)
    eng, ora = H.make_pair(cfg, n_slots, max_batch=1 << 17)
    a, p, b = T.workload(seed, cfg, n_slots, partitions=10 if name == "cfg3" else None)
    H.arm(eng, ora, a)
    ob, on = H.phase2a(eng, ora, p)
    assert len(on) == 0
    H.compare_acceptors(eng, ora, cfg, 0, n_slots)
    total = 0
    for chunk in np.array_split(b, 5):
        st, c = H.phase2b(eng, ora, chunk)
        total += len(c)
        H.replica(eng, ora, c)
    assert total == n_slots
    assert eng.chosen_watermark() == n_slots
    H.compare_log(eng, ora, 0, n_slots)
    eng.close()


def test_cfg1_round_bump_nacks():
    """cfg1 variant: a mid-trace round bump (leader 1, round 1) makes later round-0
    Phase2as stale at the acceptors that saw it (BASELINE.md section 4)."""
    cfg, n_slots = T.config_by_name("cfg1")
    for seed in range(3):
        g = T.rng(100 + seed)
        eng, ora = H.make_pair(cfg, n_slots)
        slots = np.arange(n_slots)
        p0 = T.phase2as(g, slots, 1, 1, 3, False, 0)
        p1 = T.phase2as(g, slots[: n_slots // 2], 1, 1, 3, False, 1, values=slots[: n_slots // 2] + 1000)
        mix = np.concatenate([p0, p1])[g.permutation(len(p0) + len(p1))]
        H.arm(eng, ora, np.concatenate([T.arms(slots, 0), T.arms(slots[: n_slots // 2], 1,
                                                                 slots[: n_slots // 2] + 1000)]))
        ob, on = H.phase2a(eng, ora, mix)
        assert len(on) > 0
        H.compare_acceptors(eng, ora, cfg, 0, n_slots)
        st, c = H.phase2b(eng, ora, ob[g.permutation(len(ob))])
        H.replica(eng, ora, c)
        H.compare_log(eng, ora, 0, n_slots)
        eng.close()


# --------------------------------------------------------------------------- adversarial differential
@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("shape", ["majority5", "grid2x3", "groups3x3"])
def test_adversarial_random_traces(seed, shape):
    """Random rounds (stale and fresh), duplicate deliveries, late votes, several
    live rounds per slot, non-thrifty fan-out, many small and large batches."""
    if shape == "majority5":
        cfg = dict(f=2, num_acceptor_groups=1, acceptors_per_group=5, flexible=False, num_leaders=3,
                   num_replicas=3)
    elif shape == "grid2x3":
        cfg = dict(f=1, num_acceptor_groups=2, acceptors_per_group=3, flexible=True, num_leaders=2,
                   num_replicas=2)
    else:
        cfg = dict(f=1, num_acceptor_groups=3, acceptors_per_group=3, flexible=False, num_leaders=2,
                   num_replicas=2)
    _adversarial(cfg, 1000 * seed + len(shape), 3000, 2500)


def _adversarial(cfg, seed, n_slots, kmax, coop_ctas_per_sm=0, max_batch=1 << 16):
    g = T.rng(seed)
    eng, ora = H.make_pair(cfg, n_slots, max_batch=max_batch, overflow_capacity=1 << 13 if n_slots <= 3000 else 1 << 20)
    eng.set_coop_ctas_per_sm(coop_ctas_per_sm)
    for phase in range(4):
        k = int(g.integers(1, kmax))
        slots = g.integers(0, n_slots, size=k).astype(np.int32)
        rounds = g.integers(0, 4, size=k).astype(np.int32) if phase else np.zeros(k, dtype=np.int32)
        values = (slots * 8 + rounds).astype(np.int32)   # one value per (slot, round)
        a = T.arms(slots, 0, values)
        a["round"] = rounds
        H.arm(eng, ora, a)
        p = T.phase2as(g, slots, cfg["f"], cfg["num_acceptor_groups"], cfg["acceptors_per_group"],
                       cfg["flexible"], rounds, values, thrifty=bool(g.integers(0, 2)))
        p = p[g.permutation(len(p))]
        dup = p[g.integers(0, len(p), size=len(p) // 10)]
        p = np.concatenate([p, dup])[g.permutation(len(p) + len(dup))]
        votes = []
        for chunk in np.array_split(p, int(g.integers(1, 4))):
            ob, on = H.phase2a(eng, ora, chunk)
            votes.append(ob)
        H.compare_acceptors(eng, ora, cfg, 0, n_slots)
        v = np.concatenate(votes)
        v = np.concatenate([v, v[g.integers(0, max(len(v), 1), size=len(v) // 5)]]) if len(v) else v
        v = v[g.permutation(len(v))]
        for chunk in np.array_split(v, int(g.integers(1, 6))):
            st, c = H.phase2b(eng, ora, chunk)
            assert st == 0
            H.replica(eng, ora, c)
    H.compare_log(eng, ora, 0, n_slots)
    eng.close()


@pytest.mark.parametrize("ctas_per_sm", [1, 0])
def test_results_do_not_depend_on_the_grid_size(ctas_per_sm):
    """The persistent kernels split the delivery stream into per-warp ranges; the outputs must be
    the same for any grid (fpx_set_coop_ctas_per_sm: engines sharing a GPU run smaller grids).
    Batches of up to 2 * 10^5 records, i.e. more CTAs than one wave at 1 CTA/SM."""
    cfg = dict(f=2, num_acceptor_groups=1, acceptors_per_group=5, flexible=False, num_leaders=3, num_replicas=3)
    _adversarial(cfg, 4242, 50000, 40000, coop_ctas_per_sm=ctas_per_sm, max_batch=1 << 18)


def test_unknown_key_error_index_is_first_in_order():
    cfg, _ = T.config_by_name("cfg2")
    eng, ora = H.make_pair(cfg, 5000)
    a, p, b = T.workload(3, cfg, 4000)
    H.arm(eng, ora, a[:3990])              # slots 3990.. never armed
    st, _ = H.phase2b(eng, ora, b)
    assert st == -4
    eng.close()


def test_empty_and_ragged_batches():
    cfg, _ = T.config_by_name("cfg2")
    eng, ora = H.make_pair(cfg, 5000)
    z2a, z2b = np.zeros(0, dtype=P2A), np.zeros(0, dtype=P2B)
    H.arm(eng, ora, z2a)
    H.phase2a(eng, ora, z2a)
    H.phase2b(eng, ora, z2b)
    for n in (1, 31, 32, 33, 255, 1023, 1024, 1025, 2049):
        eng.reset()
        ora = O.MultiPaxos(2, 1, 5, False, 3, 3)
        a, p, b = T.workload(n, cfg, n)
        H.arm(eng, ora, a)
        H.phase2a(eng, ora, p)
        st, c = H.phase2b(eng, ora, b)
        assert len(c) == n
    eng.close()


def test_sharded_engines_cover_the_log():
    """Slot-residue sharding (SURVEY 8(e)): P engines, slot % P == g; the union of
    their Chosen streams is the unsharded one and the global watermark is
    min_g(local frontier)."""
    cfg, _ = T.config_by_name("cfg2")
    n_slots, P = 6000, 4
    ora = O.MultiPaxos(2, 1, 5, False, 3, 3)
    a, p, b = T.workload(11, cfg, n_slots)
    ora.arm(a)
    ora.acceptor_phase2a(p)
    _, _, oc = ora.proxyleader_phase2b(b)
    ora.replica_chosen(oc)
    got = []
    wms = []
    for gi in range(P):
        eng = Engine(slot_capacity=n_slots, max_batch=1 << 16, shard_index=gi, shard_count=P, **cfg)
        eng.proxyleader_arm(a[a["slot"] % P == gi])
        pb, nk = eng.acceptor_phase2a(p[p["slot"] % P == gi])
        assert len(nk) == 0
        c = eng.proxyleader_phase2b(b[b["slot"] % P == gi])
        eng.replica_chosen(c)
        wms.append(eng.chosen_watermark())
        got.append(c)
        with pytest.raises(FpxError) as ei:
            eng.proxyleader_arm(a[a["slot"] % P == (gi + 1) % P][:5])
        assert ei.value.status == -6
        eng.close()
    allc = np.concatenate(got)
    assert sorted(allc.tolist()) == sorted(oc.tolist())
    assert min(wms) >= n_slots and ora.executed_watermark() == n_slots


def test_full_size_properties_cfg2():
    """BASELINE cfg2 at full size (2^20 slots, 3*2^20 votes): size-independent
    properties instead of the (slow) oracle: every slot chosen exactly once with
    value == slot, Chosen order == order of completing votes, watermark == n."""
    cfg, n_slots = T.config_by_name("cfg2")
    eng = Engine(slot_capacity=n_slots, max_batch=3 << 20, **cfg)
    a, p, b = T.workload(0, cfg, n_slots)
    eng.proxyleader_arm(a)
    pb, nk = eng.acceptor_phase2a(p)
    assert len(nk) == 0 and len(pb) == len(p)
    assert np.array_equal(pb, T.votes_of(p))
    c = eng.proxyleader_phase2b(b)
    assert len(c) == n_slots
    assert np.array_equal(np.sort(c["slot"]), np.arange(n_slots))
    assert np.array_equal(c["slot"], c["value_id"])
    # completing vote of a slot = the LAST of its 3 votes in delivery order
    last = np.zeros(n_slots, dtype=np.int64)
    np.maximum.at(last, b["slot"], np.arange(len(b)))
    assert np.array_equal(c["slot"], b["slot"][np.sort(last)])
    eng.replica_chosen(c)
    assert eng.chosen_watermark() == n_slots
    for g_, a_ in [(0, 0), (0, 4)]:
        r, m, vr, vv = eng.snapshot_acceptor(g_, a_, 0, n_slots)
        mine = p[(p["dst"] & 0xffff) == a_]
        assert r == 0 and m == mine["slot"].max()
        exp = np.full(n_slots, -1, dtype=np.int32)
        exp[mine["slot"]] = 0
        assert np.array_equal(vr, exp)
    eng.close()


# --------------------------------------------------------------------------- compartmentalized Mencius (a9)
@pytest.mark.parametrize("seed", [0, 1])
def test_mencius_index_math_and_tally(seed):
    """S/mencius: slot s -> leader group s % LG, acceptor group (s / LG) % AG
    (mencius/ProxyLeader.scala:169-176,231-234), quorum f+1 keyed by acceptor index
    (:334-336), Nack to leaders(s % LG)(round % leadersPerGroup) (mencius/Acceptor.scala:215-219)."""
    from frankenpaxos_b200 import MENCIUS
    f, LG, AG, per = 1, 3, 2, 3
    n_slots = 5000
    g = T.rng(70 + seed)
    eng = Engine(f, AG, per, num_leaders=2, num_replicas=2, slot_capacity=n_slots, max_batch=1 << 16,
                 protocol=MENCIUS, num_leader_groups=LG)
    ora = O.MultiPaxos(f, AG, per, False, 2, 2, mencius_leader_groups=LG)
    slots = np.arange(n_slots, dtype=np.int32)
    grp = (slots % LG) * AG + (slots // LG) % AG
    def p2as(sl, rnd, thrifty=True):
        q = f + 1 if thrifty else per
        keys = g.random((len(sl), per))
        acc = np.argsort(keys, axis=1)[:, :q].astype(np.int32)
        out = np.zeros(len(sl) * q, dtype=P2A)
        out["slot"] = np.repeat(sl, q); out["round"] = rnd; out["value_id"] = np.repeat(sl, q) * 4 + rnd
        out["dst"] = (np.repeat(grp[sl], q) << 16) | acc.reshape(-1)
        return out
    a0 = T.arms(slots, 0, slots * 4)
    H.arm(eng, ora, a0)
    bump = slots[::7]
    a1 = T.arms(bump, 1, bump * 4 + 1)
    H.arm(eng, ora, a1)
    mix = np.concatenate([p2as(slots, 0), p2as(bump, 1, thrifty=False)])
    mix = mix[g.permutation(len(mix))]
    votes = []
    for chunk in np.array_split(mix, 3):
        ob, on = H.phase2a(eng, ora, chunk)
        votes.append(ob)
    assert sum(len(v) for v in votes) < len(mix)          # some Nacks happened
    cfg = dict(num_acceptor_groups=LG * AG, acceptors_per_group=per)
    H.compare_acceptors(eng, ora, cfg, 0, n_slots)
    v = np.concatenate(votes)
    v = v[g.permutation(len(v))]
    for chunk in np.array_split(v, 4):
        st, c = H.phase2b(eng, ora, chunk)
        assert st == 0
        H.replica(eng, ora, c)
    H.compare_log(eng, ora, 0, n_slots)
    # a Phase2a delivered to the wrong acceptor group is a precondition violation
    bad = np.array([(0, 0, 0, (1 << 16) | 0)], dtype=P2A)
    with pytest.raises(FpxError) as ei:
        eng.acceptor_phase2a(bad)
    assert ei.value.status == -5
    eng.close()


# --------------------------------------------------------------------------- vanilla Mencius (a9, BASELINE cfg5 shape)
@pytest.mark.parametrize("f", [1, 3])
def test_vanilla_mencius_matches_oracle(f):
    """cfg5: n = 2f+1 servers, owner = slot % n, the coordinator's own vote is
    pre-seeded, up to n-1 Phase2bs per slot, quorum f+1 (Server.scala:767-829,
    1001-1142).  Also: per-slot round compare (Phase2Nack), Phase2a for an entry that
    is already chosen, stale / unknown Phase2bs, learn-chosen at other servers."""
    from frankenpaxos_b200 import VANILLA_MENCIUS
    n = 2 * f + 1
    n_slots = 4000
    g = T.rng(90 + f)
    eng = Engine(f, 1, n, num_leaders=f + 1, num_replicas=f + 1, slot_capacity=n_slots, max_batch=1 << 16,
                 protocol=VANILLA_MENCIUS)
    ora = O.VanillaMencius(f)
    slots = np.arange(n_slots, dtype=np.int32)
    req = np.zeros(n_slots, dtype=P2A)
    req["slot"] = slots; req["round"] = 0; req["value_id"] = slots * 3 + 1; req["dst"] = slots % n
    eng.vm_client_request(req)
    assert ora.client_request(req) == (0, -1)
    # Phase2a from each coordinator to all other servers (:806-815), shuffled delivery
    others = np.array([[s for s in range(n) if s != o] for o in range(n)], dtype=np.int32)
    p = np.zeros(n_slots * (n - 1), dtype=P2A)
    p["slot"] = np.repeat(slots, n - 1); p["round"] = 0; p["value_id"] = np.repeat(req["value_id"], n - 1)
    p["dst"] = others[slots % n].reshape(-1)
    p = p[g.permutation(len(p))]
    votes = []
    for chunk in np.array_split(p, 3):
        st, _, orep = ora.phase2a(chunk)
        erep = eng.vm_phase2a(chunk)
        H.same(erep, orep, "vanilla Phase2a replies")
        votes.append(erep[erep["group"] == 0])
    v = np.concatenate(votes)
    v["group"] = 0
    v = v[g.permutation(len(v))]
    # a stale-round vote and a vote for a slot without Phase 2 are ignored
    junk = np.array([(0, 1, n_slots - 1, 0)], dtype=P2B)
    total = 0
    for chunk in np.array_split(v, 5):
        st, c = H.phase2b(eng, ora, chunk)
        assert st == 0
        total += len(c)
        H.replica(eng, ora, c) if False else None
    assert total == n_slots
    st, c = H.phase2b(eng, ora, junk)
    assert st == 0 and len(c) == 0
    # higher-round Phase2a at a non-coordinator: accepted; lower round afterwards: Phase2Nack
    hi = np.array([(10, 5, 777, 1 if 10 % n != 1 else 2), (11, 5, 778, 0 if 11 % n != 0 else 2)], dtype=P2A)
    H.same(eng.vm_phase2a(hi), ora.phase2a(hi)[2], "higher round")
    lo = np.array([(10, 2, 779, hi[0]["dst"]), (11, 5, 780, hi[1]["dst"])], dtype=P2A)
    er = eng.vm_phase2a(lo)
    H.same(er, ora.phase2a(lo)[2], "lower/equal round")
    assert er["group"].tolist() == [1, 0] and er["round"][0] == 5
    # Phase2a for a slot the coordinator already chose: reply Chosen(value) (:1017-1027)
    ch = np.array([(20, 0, 1, 20 % n)], dtype=P2A)
    er = eng.vm_phase2a(ch)
    H.same(er, ora.phase2a(ch)[2], "Phase2a on a chosen entry")
    assert er["group"][0] == 2 and er["round"][0] == 20 * 3 + 1
    # learn-chosen at another server, then a Phase2a there
    lc = np.array([(0, (30 % n + 1) % n, 30, 91)], dtype=P2B)
    eng.vm_learn_chosen(lc); ora.learn_chosen(lc)
    q = np.array([(30, 9, 5, lc[0]["acceptor"])], dtype=P2A)
    H.same(eng.vm_phase2a(q), ora.phase2a(q)[2], "Phase2a after learn-chosen")
    # batch contract: two Phase2as for one (slot, server) in one call
    with pytest.raises(FpxError) as ei:
        eng.vm_phase2a(np.array([(40, 1, 1, (40 % n + 1) % n), (41, 1, 1, (41 % n + 1) % n), (40, 2, 2, (40 % n + 1) % n)], dtype=P2A))
    assert (ei.value.status, ei.value.index) == (-12, 2)
    # a Phase2b in a LARGER round than the one proposed fails checkEq (:1116)
    eng2 = Engine(f, 1, n, num_leaders=f + 1, num_replicas=f + 1, slot_capacity=64, max_batch=1024, protocol=VANILLA_MENCIUS)
    ora2 = O.VanillaMencius(f)
    r2 = np.array([(0, 0, 5, 0)], dtype=P2A)
    eng2.vm_client_request(r2); ora2.client_request(r2)
    st, c = H.phase2b(eng2, ora2, np.array([(0, 1, 0, 3)], dtype=P2B))
    assert st == -4
    eng.close(); eng2.close()


# --------------------------------------------------------------------------- Phase 1 reads (SURVEY 8(f) rank 2)
@pytest.mark.parametrize("shape", ["majority5", "grid2x3", "groups3x3"])
def test_phase1a_and_safe_values(shape):
    """Acceptor.handlePhase1a (Acceptor.scala:148-182) and Leader.safeValue
    (Leader.scala:318-329) over the same vote cells, after traffic in several rounds."""
    if shape == "majority5":
        cfg = dict(f=2, num_acceptor_groups=1, acceptors_per_group=5, flexible=False, num_leaders=3, num_replicas=3)
    elif shape == "grid2x3":
        cfg = dict(f=1, num_acceptor_groups=2, acceptors_per_group=3, flexible=True, num_leaders=2, num_replicas=2)
    else:
        cfg = dict(f=1, num_acceptor_groups=3, acceptors_per_group=3, flexible=False, num_leaders=2, num_replicas=2)
    g = T.rng(len(shape))
    n_slots = 3000
    eng, ora = H.make_pair(cfg, n_slots, overflow_capacity=1 << 13)
    for rnd in (0, 1, 3):
        slots = np.sort(g.choice(n_slots, size=1200, replace=False)).astype(np.int32)
        p = T.phase2as(g, slots, cfg["f"], cfg["num_acceptor_groups"], cfg["acceptors_per_group"], cfg["flexible"],
                       rnd, slots * 4 + rnd)
        H.phase2a(eng, ora, p[g.permutation(len(p))])
    G, A = cfg["num_acceptor_groups"], cfg["acceptors_per_group"]
    # a stale Phase1a is nacked with the acceptor's round; a fresh one raises it and reads the votes
    kind, val = eng.acceptor_phase1a(0, 0, 1)
    assert (kind, val) == ("nack", 3) and ora.phase1a(0, 0, 1) == 3
    for gi in range(G):
        for a in range(A):
            assert ora.phase1a(gi, a, 7) == -1
            kind, info = eng.acceptor_phase1a(gi, a, 7, chosen_watermark=100)
            assert kind == "phase1b"
            r, m, vr, vv = ora.snapshot_acceptor(gi, a, 100, max(0, m_ := ora.snapshot_acceptor(gi, a, 0, 0)[1]) + 1 - 100)
            exp = [(100 + i, int(vr[i]), int(vv[i])) for i in range(len(vr)) if vr[i] >= 0]
            assert info == exp and r == 7
    H.compare_acceptors(eng, ora, cfg, 0, n_slots)
    for responders in (0b1, (1 << (G * A)) - 1, 0b101011 & ((1 << (G * A)) - 1), 0):
        ev, evv, em = eng.leader_safe_values(responders, 50, 2500)
        ov, ovv, om = ora.safe_values(responders, 50, 2500)
        H.same(ev, ov, "safeValue voteRound"); H.same(evv, ovv, "safeValue value"); assert em == om
    eng.close()


def test_full_size_properties_cfg3():
    """BASELINE cfg3 at full size: 2x3 grid, 2^22 slots, thrifty write quorum = one grid
    column (2 votes per slot), 10 proxy-leader partitions (slot % 10) shuffled within a
    partition; 8.4M-record batches (two tally launches).  Size-independent properties."""
    cfg, n_slots = T.config_by_name("cfg3")
    eng = Engine(slot_capacity=n_slots, max_batch=2 * n_slots, **cfg)
    a, p, b = T.workload(1, cfg, n_slots, partitions=10)
    eng.proxyleader_arm(a)
    pb, nk = eng.acceptor_phase2a(p)
    assert len(nk) == 0 and np.array_equal(pb, T.votes_of(p))
    c = eng.proxyleader_phase2b(b)
    assert len(c) == n_slots
    assert np.array_equal(np.sort(c["slot"]), np.arange(n_slots)) and np.array_equal(c["slot"], c["value_id"])
    last = np.zeros(n_slots, dtype=np.int64)
    np.maximum.at(last, b["slot"], np.arange(len(b)))
    assert np.array_equal(c["slot"], b["slot"][np.sort(last)])   # Chosen order == order of the completing votes
    eng.replica_chosen(c)
    assert eng.chosen_watermark() == n_slots
    # votes of one grid row only are never a write quorum (Grid.scala:49): re-run with row-0 votes only
    eng.reset()
    eng.proxyleader_arm(a[:100000])
    row0 = b[(b["group"] == 0) & (b["slot"] < 100000)]
    assert len(eng.proxyleader_phase2b(row0)) == 0
    eng.close()


def test_full_size_properties_cfg4_epaxos():
    """BASELINE cfg4 shape at 2^18 instances per replica view (the generator is O(N) host
    work): every led instance produces exactly one decision event; fast commits carry the
    leader's deps when all answers agree; entries end Committed or Accepted."""
    from frankenpaxos_b200.epaxos import EpaxosReplica
    f, n, N = 2, 5, 1 << 15
    lead, pa, ok = T.epaxos_cfg4(3, f=f, n_instances=N, me=0)
    eng = EpaxosReplica(f, 0, N // n + 2, max_batch=1 << 17)
    eng.lead(lead)
    rep = eng.preaccept(pa)
    assert (rep[:, 0] == 1).all()
    # reply deps = elementwise max(local, msg)
    assert np.array_equal(rep[:, 4:], np.maximum(pa[:, 6:6 + n], pa[:, 6 + n:]))
    ev = eng.preacceptok(ok)
    decided = ev[(ev[:, 0] == 1) | (ev[:, 0] == 2)]
    assert len(decided) == len(lead)
    assert (ev[:, 0] == 3).sum() == len(lead)          # one timer event per instance (f+1 < n-1)
    eng.close()


def test_full_size_properties_cfg5_vanilla_mencius():
    """BASELINE cfg5 at full size: n=7, f=3, 2^20 slots, owner = slot % 7, 6 Phase2as and up
    to 6 Phase2bs per slot.  Every Phase2a in a fresh log is answered Phase2b(round 0); a slot
    is chosen by the 3rd remote vote in delivery order (own vote pre-seeded, quorum f+1 = 4,
    Server.scala:818-825,1122-1125); later votes hit a ChosenEntry and are dropped (:1090-1093)."""
    from frankenpaxos_b200 import VANILLA_MENCIUS
    cfg, n_slots = T.config_by_name("cfg5")
    f, n = cfg["f"], cfg["acceptors_per_group"]
    eng = Engine(slot_capacity=n_slots, max_batch=(n - 1) * n_slots, protocol=VANILLA_MENCIUS, **cfg)
    req, p, b = T.vanilla_cfg5(2, f, n_slots)
    eng.vm_client_request(req)
    rep = eng.vm_phase2a(p)
    assert (rep["group"] == 0).all()                       # kind 0 = Phase2b
    assert np.array_equal(rep["acceptor"], p["dst"]) and np.array_equal(rep["slot"], p["slot"])
    assert (rep["round"] == 0).all()
    c = eng.proxyleader_phase2b(b)
    assert len(c) == n_slots
    assert np.array_equal(np.sort(c["slot"]), np.arange(n_slots))
    assert np.array_equal(c["value_id"], c["slot"] * 3 + 1)
    # completing vote of a slot = its f-th (3rd) remote vote in delivery order
    order = np.lexsort((np.arange(len(b)), b["slot"]))
    third = order.reshape(n_slots, n - 1)[:, f - 1]
    assert np.array_equal(c["slot"], b["slot"][np.sort(third)])
    # replaying every vote afterwards changes nothing (ChosenEntry is absorbing)
    assert len(eng.proxyleader_phase2b(b[: 1 << 18])) == 0
    eng.close()


def test_vanilla_mencius_sharded_by_slot_residue():
    """cfg5's multi-GPU layout: shard slot % 8 (SURVEY 8(d)); the shards' Chosen streams
    partition the unsharded stream."""
    from frankenpaxos_b200 import VANILLA_MENCIUS
    cfg, _ = T.config_by_name("cfg5")
    f, n, P, per = cfg["f"], cfg["acceptors_per_group"], 8, 1500
    whole = []
    for gi in range(P):
        eng = Engine(slot_capacity=per * P, max_batch=1 << 16, protocol=VANILLA_MENCIUS, shard_index=gi,
                     shard_count=P, **cfg)
        req, p, b = T.vanilla_cfg5(10 + gi, f, per, slot_stride=P, slot_offset=gi)
        eng.vm_client_request(req)
        assert (eng.vm_phase2a(p)["group"] == 0).all()
        c = eng.proxyleader_phase2b(b)
        assert len(c) == per and (c["slot"] % P == gi).all()
        whole.append(c)
        # a slot of another shard is a range error
        with pytest.raises(FpxError):
            eng.vm_phase2a(np.array([((gi + 1) % P, 0, 1, ((gi + 1) % P % n + 1) % n)], dtype=P2A))
        eng.close()
    allc = np.concatenate(whole)
    assert np.array_equal(np.sort(allc["slot"]), np.arange(per * P))


@pytest.mark.parametrize("one_call", [False, True])
def test_device_pointer_path_matches_oracle(one_call):
    """(one_call: the same five launches issued by fpx_step_dev, with its event ring.)
    The *_dev entry points bench.py times (inputs and outputs resident in HBM, one fpx_sync at the
    end): arm -> acceptor -> tally -> replica (count taken from the device) -> watermark, with a round
    bump in the middle so that the Nack stream and the exact compaction are exercised too."""
    import torch
    cfg, _ = T.config_by_name("cfg2")
    n_slots = 20000
    eng, ora = H.make_pair(cfg, n_slots, max_batch=1 << 17, overflow_capacity=1 << 12)
    g = T.rng(77)
    dev = torch.device("cuda", 0)
    slots = np.arange(n_slots, dtype=np.int32)
    a = T.arms(slots, 0, slots * 2 + 1)
    p = T.phase2as(g, slots, cfg["f"], 1, 5, False, 0, slots * 2 + 1)
    hi = T.phase2as(g, slots[::50], cfg["f"], 1, 5, False, 2, slots[::50] * 2)      # a newer leader's messages
    p = np.concatenate([p[: len(p) // 2], hi, p[len(p) // 2:]])                       # later round-0 messages get Nacks
    st, idx = ora.arm(np.concatenate([a, T.arms(slots[::50], 2, slots[::50] * 2)]))
    _, _, ob, on = ora.acceptor_phase2a(p)
    votes = ob[g.permutation(len(ob))]
    _, _, oc = ora.proxyleader_phase2b(votes)
    ora.replica_chosen(oc)

    def td(x):
        return torch.from_numpy(x.view(np.int32).reshape(len(x), -1).copy()).to(dev)
    d_a = td(np.concatenate([a, T.arms(slots[::50], 2, slots[::50] * 2)])); d_p = td(p); d_v = td(votes)
    d_p2b = torch.zeros((len(p), 4), dtype=torch.int32, device=dev); d_nack = torch.zeros((len(p), 2), dtype=torch.int32, device=dev)
    d_ch = torch.zeros((len(votes), 2), dtype=torch.int32, device=dev); d_wm = torch.zeros(1, dtype=torch.int32, device=dev)
    if one_call:
        eng.step_dev(d_a.data_ptr(), len(d_a), d_p.data_ptr(), len(p), d_p2b.data_ptr(), d_nack.data_ptr(),
                     d_v.data_ptr(), len(votes), d_ch.data_ptr(), d_wm.data_ptr(), ring_slot=3)
    else:
        eng.proxyleader_arm_dev(d_a.data_ptr(), len(d_a))
        eng.acceptor_phase2a_dev(d_p.data_ptr(), len(p), d_p2b.data_ptr(), d_nack.data_ptr())
        eng.proxyleader_phase2b_dev(d_v.data_ptr(), len(votes), d_ch.data_ptr())
        eng.replica_chosen_last_dev(d_ch.data_ptr())
        eng.chosen_watermark_dev(d_wm.data_ptr())
    r = eng.sync()
    if one_call:
        acc_ms, tally_ms = eng.step_kernel_ms(3)
        assert 0 < acc_ms < 50 and 0 < tally_ms < 50
    assert (r.status, r.n_p2b, r.n_nack, r.n_chosen) == (0, len(ob), len(on), len(oc)) and len(on) > 0
    assert r.watermark == ora.executed_watermark() == int(d_wm.item())
    H.same(d_p2b[: r.n_p2b].cpu().numpy().view(P2B).reshape(-1), ob, "Phase2b stream (device)")
    H.same(d_nack[: r.n_nack].cpu().numpy().view(NACK).reshape(-1), on, "Nack stream (device)")
    H.same(d_ch[: r.n_chosen].cpu().numpy().view(CHOSEN).reshape(-1), oc, "Chosen stream (device)")
    H.compare_acceptors(eng, ora, cfg, 0, n_slots)
    H.compare_log(eng, ora, 0, n_slots)
    eng.close()


# --------------------------------------------------------------------------- full size, bit-exact vs the oracle
def _full_size(name, seed, partitions=None):
    cfg, n_slots = T.config_by_name(name)
    a, p, b = T.workload(seed, cfg, n_slots, partitions=partitions)
    eng, ora = H.make_pair(cfg, n_slots, max_batch=len(p), overflow_capacity=1 << 10)
    H.arm(eng, ora, a)
    ob, on = H.phase2a(eng, ora, p)                  # Phase2b / Nack streams, bit-exact incl. order
    assert len(on) == 0
    H.compare_acceptors(eng, ora, cfg, 0, n_slots)   # every acceptor: round, maxVotedSlot, voteRound[], voteValue[]
    st, c = H.phase2b(eng, ora, b)                   # Chosen stream, bit-exact incl. order
    assert st == 0 and len(c) == n_slots
    H.replica(eng, ora, c)
    H.compare_log(eng, ora, 0, n_slots)
    eng.close()


def test_full_size_bit_exact_cfg2(tally_path):
    """BASELINE cfg2 at its full size (2^20 slots, 3*2^20 Phase2a / Phase2b) against the oracle:
    every stream, every acceptor's state, the replica log."""
    _full_size("cfg2", 0)


def test_full_size_bit_exact_cfg3(tally_path):
    """BASELINE cfg3 at its full size (2x3 grid, 2^22 slots, 10 proxy-leader partitions)."""
    if tally_path == "exact":
        pytest.skip("full-size cfg3 runs once (oracle time); the exact path is covered at 30000 slots")
    _full_size("cfg3", 1, partitions=10)


def test_full_size_bit_exact_cfg5_vanilla_mencius(tally_path):
    """BASELINE cfg5 at its full size (n=7, 2^20 slots, 6 Phase2a + 6 Phase2b per slot) against the oracle."""
    if tally_path == "exact":
        pytest.skip("one full-size pass against the oracle is enough (the exact path is covered at 4000 slots)")
    from frankenpaxos_b200 import VANILLA_MENCIUS
    cfg, n_slots = T.config_by_name("cfg5")
    f, n = cfg["f"], cfg["acceptors_per_group"]
    eng = Engine(slot_capacity=n_slots, max_batch=(n - 1) * n_slots, protocol=VANILLA_MENCIUS, **cfg)
    ora = O.VanillaMencius(f)
    req, p, b = T.vanilla_cfg5(2, f, n_slots)
    eng.vm_client_request(req)
    assert ora.client_request(req) == (0, -1)
    st, _, orep = ora.phase2a(p)
    H.same(eng.vm_phase2a(p), orep, "vanilla Phase2a replies")
    st, c = H.phase2b(eng, ora, b)
    assert st == 0 and len(c) == n_slots
    eng.close()


def test_vanilla_step_in_one_call_matches_the_separate_calls_and_the_oracle(tally_path):
    """fpx_vm_step_dev (client requests, Phase2a batch, tally with the log put and the watermark riding in it:
    three launches) against the five separate device calls on a second engine and against the oracle, over
    several windows of one log; the second window carries a stale duplicate of every earlier vote."""
    import torch
    from frankenpaxos_b200 import VANILLA_MENCIUS
    cfg, _ = T.config_by_name("cfg5")
    f, n, W, wins = cfg["f"], cfg["acceptors_per_group"], 1 << 15, 3
    mk = lambda: Engine(slot_capacity=wins * W, max_batch=2 * (n - 1) * W, protocol=VANILLA_MENCIUS, **cfg)
    one, sep, ora = mk(), mk(), O.VanillaMencius(f)
    dev = torch.device("cuda", 0)
    td = lambda x: torch.from_numpy(x.view(np.int32).reshape(len(x), -1).copy()).to(dev)
    outs = [[torch.zeros((2 * (n - 1) * W, k), dtype=torch.int32, device=dev) for k in (4, 2)] + [torch.zeros(1, dtype=torch.int32, device=dev)]
            for _ in range(2)]
    prev_b = None
    for w in range(wins):
        req, p, b = T.vanilla_cfg5(70 + w, f, W, slot_offset=w * W)
        if prev_b is not None:
            b = np.concatenate([prev_b[: len(prev_b) // 2], b])     # votes for chosen entries: ignored (:1090-1093)
        prev_b = b
        assert ora.client_request(req) == (0, -1)
        _, _, orep = ora.phase2a(p)
        st, _, oc = ora.proxyleader_phase2b(b)
        assert st == 0
        d_req, d_p, d_b = td(req), td(p), td(b)
        (r1, c1, w1), (r2, c2, w2) = outs
        one.vm_step_dev(d_req.data_ptr(), len(req), d_p.data_ptr(), len(p), r1.data_ptr(), d_b.data_ptr(), len(b), c1.data_ptr(), w1.data_ptr())
        sep.vm_client_request_dev(d_req.data_ptr(), len(req))
        sep.vm_phase2a_dev(d_p.data_ptr(), len(p), r2.data_ptr())
        sep.proxyleader_phase2b_dev(d_b.data_ptr(), len(b), c2.data_ptr())
        sep.replica_chosen_last_dev(c2.data_ptr())
        sep.chosen_watermark_dev(w2.data_ptr())
        ra, rb = one.sync(), sep.sync()
        assert (ra.status, ra.n_chosen, ra.watermark) == (rb.status, rb.n_chosen, rb.watermark) == (0, len(oc), (w + 1) * W)
        assert int(w1.item()) == int(w2.item()) == (w + 1) * W
        H.same(r1[: len(p)].cpu().numpy().view(P2B).reshape(-1), orep, f"Phase2a replies, window {w}")
        H.same(c1[: ra.n_chosen].cpu().numpy().view(CHOSEN).reshape(-1), oc, f"Chosen stream, window {w}")
        H.same(c2[: rb.n_chosen].cpu().numpy().view(CHOSEN).reshape(-1), oc, f"Chosen stream (separate calls), window {w}")
    H.same(one.snapshot_log(0, wins * W), sep.snapshot_log(0, wins * W), "log")
    for a in range(n):
        x, y = one.snapshot_acceptor(0, a, 0, wins * W), sep.snapshot_acceptor(0, a, 0, wins * W)
        assert x[:2] == y[:2]
        H.same(x[2], y[2], f"server {a} voteRound"); H.same(x[3], y[3], f"server {a} voteValue")
    one.close(); sep.close()


def test_bench_shaped_step_on_a_rebased_window_matches_the_oracle(tally_path):
    """What bench.py times: the device-pointer path on window w != 0 of a long log (slots
    w*2^20 .. (w+1)*2^20, earlier windows already committed), compared with the oracle."""
    import torch
    cfg, _ = T.config_by_name("cfg2")
    W, win = 1 << 20, 2
    eng, ora = H.make_pair(cfg, 3 * W, max_batch=3 * W, overflow_capacity=1 << 10)
    dev = torch.device("cuda", 0)

    def td(x):
        return torch.from_numpy(x.view(np.int32).reshape(len(x), -1).copy()).to(dev)
    d_p2b = torch.zeros((3 * W, 4), dtype=torch.int32, device=dev)
    d_nack = torch.zeros((3 * W, 2), dtype=torch.int32, device=dev)
    d_ch = torch.zeros((3 * W, 2), dtype=torch.int32, device=dev)
    d_wm = torch.zeros(1, dtype=torch.int32, device=dev)
    for w in range(win + 1):
        a, p, b = T.workload(40 + w, cfg, W, slot0=w * W)
        ora.arm(a)
        _, _, ob, on = ora.acceptor_phase2a(p)
        _, _, oc = ora.proxyleader_phase2b(b)
        ora.replica_chosen(oc)
        d_a, d_p, d_b = td(a), td(p), td(b)
        eng.proxyleader_arm_dev(d_a.data_ptr(), len(a))
        eng.acceptor_phase2a_dev(d_p.data_ptr(), len(p), d_p2b.data_ptr(), d_nack.data_ptr())
        eng.proxyleader_phase2b_dev(d_b.data_ptr(), len(b), d_ch.data_ptr())
        eng.replica_chosen_last_dev(d_ch.data_ptr())
        eng.chosen_watermark_dev(d_wm.data_ptr())
        r = eng.sync()
        assert (r.status, r.n_p2b, r.n_nack, r.n_chosen) == (0, len(ob), 0, len(oc))
        assert r.watermark == ora.executed_watermark() == (w + 1) * W
        H.same(d_p2b[: r.n_p2b].cpu().numpy().view(P2B).reshape(-1), ob, f"Phase2b stream, window {w}")
        H.same(d_ch[: r.n_chosen].cpu().numpy().view(CHOSEN).reshape(-1), oc, f"Chosen stream, window {w}")
    H.compare_acceptors(eng, ora, cfg, win * W, W)
    H.compare_log(eng, ora, win * W, W)
    eng.close()


def test_async_host_step_matches_oracle(tally_path):
    """fpx_step_submit / fpx_step_wait: double-buffered host-pointer steps (what bench.py's e2e times),
    arming from the Phase2a batch itself (arm = NULL) and from an explicit arm batch; a round bump in the
    middle exercises the Nack re-copy.  Streams, counts, watermark and final state vs the oracle."""
    import torch
    cfg, _ = T.config_by_name("cfg2")
    W_, n_steps = 5000, 4
    eng, ora = H.make_pair(cfg, n_steps * W_, max_batch=1 << 16, overflow_capacity=1 << 12)
    g = T.rng(123)
    steps = []
    for w in range(n_steps):
        a, p, b = T.workload(60 + w, cfg, W_, slot0=w * W_, round_=3 if w == 3 else 0)   # the new leader's round after the bump
        if w == 2:   # a newer leader's Phase2as for some slots of this window, delivered in the middle
            sl = np.arange(w * W_, w * W_ + W_, 40, dtype=np.int32)
            hi = T.phase2as(g, sl, cfg["f"], 1, 5, False, 3, sl * 2)
            p = np.concatenate([p[: len(p) // 2], hi, p[len(p) // 2:]])
            a = np.concatenate([a, T.arms(sl, 3, sl * 2)])
        steps.append((a, p))
    pin = lambda x: torch.from_numpy(x.view(np.int32).reshape(len(x), x.dtype.itemsize // 4).copy()).pin_memory()
    outs = []
    expect = []
    # the votes of step w are the oracle's replies of step w, shuffled: compute the oracle first
    for w, (a, p) in enumerate(steps):
        ora.arm(a)
        _, _, ob, on = ora.acceptor_phase2a(p)
        votes = ob[g.permutation(len(ob))]
        _, _, oc = ora.proxyleader_phase2b(votes)
        ora.replica_chosen(oc)
        expect.append((ob, on, oc, ora.executed_watermark(), votes))
    bufs = []
    for w, (a, p) in enumerate(steps):
        votes = expect[w][4]
        hp, hv = pin(p), pin(votes)
        ha = pin(a) if w % 2 else None          # odd steps: explicit arm batch; even steps: arm from the Phase2as
        o1 = torch.zeros((len(p), 4), dtype=torch.int32).pin_memory()
        o2 = torch.zeros((len(p), 2), dtype=torch.int32).pin_memory()
        o3 = torch.zeros((len(votes), 2), dtype=torch.int32).pin_memory()
        bufs.append((hp, hv, ha, o1, o2, o3))
        if w == 2 and ha is None:
            # arming from the Phase2a stream covers the bumped keys too (they are in the stream)
            pass
        eng.step_submit(ha.data_ptr() if ha is not None else None, len(a) if ha is not None else 0, hp.data_ptr(), len(p),
                        hv.data_ptr(), len(votes), o1.data_ptr(), o2.data_ptr(), o3.data_ptr())
        if w >= 1:
            outs.append(eng.step_wait())
    outs.append(eng.step_wait())
    for w in range(n_steps):
        ob, on, oc, wm, _ = expect[w]
        n1, n2, n3, gw = outs[w]
        assert (n1, n2, n3, gw) == (len(ob), len(on), len(oc), wm), (w, outs[w], (len(ob), len(on), len(oc), wm))
        _, _, _, o1, o2, o3 = bufs[w]
        H.same(o1[:n1].numpy().view(P2B).reshape(-1), ob, f"Phase2b stream, step {w}")
        H.same(o2[:n2].numpy().view(NACK).reshape(-1), on, f"Nack stream, step {w}")
        H.same(o3[:n3].numpy().view(CHOSEN).reshape(-1), oc, f"Chosen stream, step {w}")
    assert len(expect[2][1]) > 0
    H.compare_acceptors(eng, ora, cfg, 0, n_steps * W_)
    H.compare_log(eng, ora, 0, n_steps * W_)
    eng.close()


@pytest.mark.parametrize("shards", [1, 3])
def test_ring_window_slides_past_slot_capacity(tally_path, shards):
    """fpx_retire_below: a log ten times longer than slot_capacity runs through one engine (per shard), the
    executed prefix retired as it goes; every stream equals the oracle's, which keeps everything.  Late
    messages for retired slots meet Done / an existing entry: duplicate arms, votes and Chosen are ignored, a
    Phase2a is still answered.  A slot beyond the live window is FPX_ERR_SLOT_RANGE."""
    cfg, _ = T.config_by_name("cfg2")
    cap, step, total = 4096, 1000, 40000
    g = T.rng(2024)
    engs = [Engine(slot_capacity=cap, max_batch=1 << 14, overflow_capacity=1 << 8, shard_index=s, shard_count=shards, **cfg)
            for s in range(shards)]
    ora = O.MultiPaxos(2, 1, 5, False, 3, 3)
    mine = lambda recs, s: recs[recs["slot"] % shards == s]
    old_votes = None
    for w in range(total // step):
        a, p, b = T.workload(300 + w, cfg, step, slot0=w * step)
        extra_a, extra_p, extra_b = a[:0], p[:0], b[:0]
        if old_votes is not None and w % 3 == 0:        # stragglers of a window that is retired by now
            oa, op, ob_ = old_votes
            extra_a, extra_p, extra_b = oa[:20], op[:30], ob_[:40]
        A, Pm, B = np.concatenate([extra_a, a]), np.concatenate([extra_p, p]), np.concatenate([b[:500], extra_b, b[500:]])
        ora.arm(A)
        _, _, ob, on = ora.acceptor_phase2a(Pm)
        _, _, oc = ora.proxyleader_phase2b(B)
        ora.replica_chosen(oc)
        got_b, got_c = [], []
        for s, e in enumerate(engs):
            e.proxyleader_arm(mine(A, s))
            eb, en = e.acceptor_phase2a(mine(Pm, s))
            assert len(en) == 0
            got_b.append(eb)
            ec = e.proxyleader_phase2b(mine(B, s))
            e.replica_chosen(ec)
            got_c.append(ec)
            wm = e.chosen_watermark()
            assert wm >= (w + 1) * step
        for s in range(shards):
            H.same(got_b[s], mine(ob, s), f"Phase2b stream, window {w}, shard {s}")
            H.same(got_c[s], mine(oc, s), f"Chosen stream, window {w}, shard {s}")
        if w >= 2:
            for e in engs:
                e.retire_below((w - 1) * step)          # keep the last two windows
            old_votes = T.workload(300 + w - 2, cfg, step, slot0=(w - 2) * step)
    assert ora.executed_watermark() == total
    # live part of the acceptors' state and of the log
    lo = total - step
    if shards == 1:
        H.compare_acceptors(engs[0], ora, cfg, lo, step)
        H.compare_log(engs[0], ora, lo, step)
    with pytest.raises(FpxError) as ei:                  # beyond the window: base + capacity
        engs[0].proxyleader_arm(T.arms(np.array([total + 2 * cap * shards], dtype=np.int32), 0))
    assert ei.value.status == -6
    with pytest.raises(FpxError):                        # only the executed prefix may be retired
        engs[0].retire_below(total + 10)
    [e.close() for e in engs]
