"""GPU parity of the range-fill variants of the vote path (SURVEY 8(f) rank 3) against the
oracle: S/mencius Phase2aNoopRange / Phase2bNoopRange / ChosenNoopRange and
S/vanillamencius Skip, through the C ABI (fpx_mencius_*, fpx_vm_skip)."""
import numpy as np
import pytest

import harness as H
from frankenpaxos_b200 import (CHOSEN, CHOSEN_RANGE, MENCIUS, P2A, P2A_RANGE, P2B, P2B_RANGE, VALUE_NOOP,
                               VANILLA_MENCIUS, VM_SKIP, Engine, FpxError)
from frankenpaxos_b200 import traces as T
from oracle import fpx_oracle_py as O

pytestmark = pytest.mark.gpu


def dst(lg, ag, a, AG):
    return ((lg * AG + ag) << 16) | a


def both(eng_call, ora_result):
    """Run the engine call; statuses must agree with the oracle's (status, index, ...)."""
    try:
        out = eng_call()
        est, eidx = 0, -1
    except FpxError as e:
        out, est, eidx = None, e.status, e.index
    assert (est, eidx) == (ora_result[0], ora_result[1]), f"engine {(est, eidx)} oracle {ora_result[:2]}"
    return out


def make(f, LG, AG, per, cap, **kw):
    eng = Engine(f, AG, per, num_leaders=2, num_replicas=2, slot_capacity=cap, max_batch=1 << 16, protocol=MENCIUS,
                 num_leader_groups=LG, **kw)
    ora = O.MultiPaxos(f, AG, per, False, 2, 2, mencius_leader_groups=LG)
    return eng, ora


def range_round_trip(eng, ora, g, ranges, cap, LG, AG, per, voters_per_group=None, dup=True):
    """arm -> acceptors -> votes (shuffled, with duplicates) -> replica, engine vs oracle."""
    arm = np.array([(s, e, r, -1) for (s, e, r) in ranges], dtype=P2A_RANGE)
    both(lambda: eng.mencius_arm_range(arm), ora.arm_range(arm, cap))
    recs = []
    for (s, e, r) in ranges:
        lg = s % LG
        for ag in range(AG):
            k = per if voters_per_group is None else voters_per_group
            for a in g.permutation(per)[:k]:
                recs.append((s, e, r, dst(lg, ag, int(a), AG)))
    recs = np.array([recs[i] for i in g.permutation(len(recs))], dtype=P2A_RANGE)
    st, err, ob, on = ora.acceptor_noop_range(recs, cap)
    out = both(lambda: eng.mencius_acceptor_noop_range(recs), (st, err))
    H.same(out[0], ob, "Phase2bNoopRange stream")
    H.same(out[1], on, "range Nack stream")
    votes = ob
    if dup and len(ob):
        votes = np.concatenate([ob, ob[g.integers(0, len(ob), size=max(1, len(ob) // 3))]])
    votes = votes[g.permutation(len(votes))]
    chosen = []
    for chunk in np.array_split(votes, 3):
        st, err, oc = ora.range_phase2b(chunk)
        ec = both(lambda: eng.mencius_range_phase2b(chunk), (st, err))
        H.same(ec, oc, "ChosenNoopRange stream")
        chosen.append(oc)
    chosen = np.concatenate(chosen)
    return chosen, on


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_mencius_noop_ranges_match_oracle(seed):
    g = T.rng(800 + seed)
    f, LG, AG, per = 1, 2 + seed % 2, 1 + seed % 2, 3
    cap = 30000
    eng, ora = make(f, LG, AG, per, cap)
    cfg = dict(num_acceptor_groups=LG * AG, acceptors_per_group=per)
    slots = np.arange(cap, dtype=np.int32)
    grp = (slots % LG) * AG + (slots // LG) % AG
    n_nack = n_chosen = 0
    # each leader group alternates single-slot windows and NoopRanges over its own slots
    pos = {lg: lg for lg in range(LG)}
    for step in range(8):
        # single-slot traffic of one leader group, round = step // 3
        lg = int(g.integers(0, LG))
        rnd = step // 3
        sl = pos[lg] + LG * np.arange(int(g.integers(50, 400)), dtype=np.int32)
        sl = sl[sl < cap]
        if len(sl) == 0:
            continue
        pos[lg] = int(sl[-1]) + LG
        H.arm(eng, ora, T.arms(sl, rnd, sl * 4 + rnd))
        q = np.zeros(len(sl) * (f + 1), dtype=P2A)
        acc = np.argsort(g.random((len(sl), per)), axis=1)[:, : f + 1].astype(np.int32)
        q["slot"] = np.repeat(sl, f + 1); q["round"] = rnd; q["value_id"] = np.repeat(sl * 4 + rnd, f + 1)
        q["dst"] = (np.repeat(grp[sl], f + 1) << 16) | acc.reshape(-1)
        ob, on = H.phase2a(eng, ora, q[g.permutation(len(q))])
        stt, oc = H.phase2b(eng, ora, ob[g.permutation(len(ob))])
        assert stt == 0
        H.replica(eng, ora, oc)
        # two or three ranges, possibly of different leader groups, one of them in a stale round
        ranges = []
        for _ in range(int(g.integers(2, 4))):
            lg2 = int(g.integers(0, LG))
            start = pos[lg2]
            end = min(cap, start + LG * int(g.integers(1, 600)) + int(g.integers(0, LG)))
            if start >= end:
                continue
            pos[lg2] = start + LG * ((end - start + LG - 1) // LG)
            ranges.append((start, end, rnd if g.random() < 0.7 else max(0, rnd - 1)))
        if not ranges:
            continue
        chosen, on = range_round_trip(eng, ora, g, ranges, cap, LG, AG, per)
        n_nack += len(on); n_chosen += len(chosen)
        both(lambda: eng.mencius_replica_chosen_range(chosen), ora.replica_chosen_range(chosen, cap))
        assert eng.chosen_watermark() == ora.first_hole()
    assert n_chosen > 0
    H.compare_acceptors(eng, ora, cfg, 0, cap)
    H.compare_log(eng, ora, 0, cap)
    eng.close()


def test_range_error_paths_and_key_sharing():
    f, LG, AG, per, cap = 1, 2, 2, 3, 4096
    eng, ora = make(f, LG, AG, per, cap)
    RA, RB, RC = P2A_RANGE, P2B_RANGE, CHOSEN_RANGE
    for bad in ([(5, 4, 0, -1)], [(0, cap + 1, 0, -1)], [(0, 8, -1, -1)], [(0, 8, 0, -1), (9, 3, 0, -1)]):
        b = np.array(bad, dtype=RA)
        both(lambda: eng.mencius_arm_range(b), ora.arm_range(b, cap))
    # acceptor of the wrong leader group / unknown acceptor
    for d in (dst(0, 0, 0, AG), dst(1, 0, 5, AG), (99 << 16)):
        b = np.array([(1, 41, 0, dst(1, 0, 0, AG)), (1, 41, 0, d)], dtype=RA)
        st, err, _, _ = ora.acceptor_noop_range(b, cap)
        assert (st, err) == (-5, 1)
        both(lambda: eng.mencius_acceptor_noop_range(b), (st, err))
    eng.reset(); ora = O.MultiPaxos(f, AG, per, False, 2, 2, mencius_leader_groups=LG)
    # a Phase2bNoopRange for a key that was never armed: logger.fatal at its index
    a = np.array([(1, 41, 0, -1)], dtype=RA)
    both(lambda: eng.mencius_arm_range(a), ora.arm_range(a, cap))
    v = np.array([(dst(1, 0, 0, AG), 1, 41, 0), (dst(1, 0, 1, AG), 1, 43, 0), (dst(1, 1, 1, AG), 1, 41, 0)], dtype=RB)
    st, err, _ = ora.range_phase2b(v)
    assert (st, err) == (-4, 1)
    both(lambda: eng.mencius_range_phase2b(v), (st, err))
    # a vote from an acceptor group index out of bounds
    v = np.array([(dst(0, 1, 1, AG), 1, 41, 0)], dtype=RB)
    st, err, _ = ora.range_phase2b(v)
    assert st == -5
    both(lambda: eng.mencius_range_phase2b(v), (st, err))
    eng.close()
    # one-slot ranges share the key space with Phase2a (first one wins, both directions)
    eng, ora = make(1, 1, 1, 3, 64)
    H.arm(eng, ora, np.array([(4, 0, 44, -1)], dtype=P2A))
    r = np.array([(4, 5, 0, -1), (6, 7, 0, -1)], dtype=RA)
    both(lambda: eng.mencius_arm_range(r), ora.arm_range(r, 64))
    H.arm(eng, ora, np.array([(6, 0, 66, -1), (8, 0, 88, -1)], dtype=P2A))
    v = np.array([(0, 4, 5, 0), (1, 4, 5, 0), (0, 6, 7, 0), (2, 6, 7, 0)], dtype=RB)
    st, err, oc = ora.range_phase2b(v)
    H.same(both(lambda: eng.mencius_range_phase2b(v), (st, err)), oc, "ChosenNoopRange")
    assert oc.tolist() == [(6, 7)]
    st, oc = H.phase2b(eng, ora, np.array([(0, 0, 4, 0), (0, 1, 4, 0), (0, 0, 8, 0), (0, 2, 8, 0)], dtype=P2B))
    assert st == 0 and oc.tolist() == [(4, 44), (8, 88)]
    with pytest.raises(FpxError) as ei:     # slot 6's key is the range's: the Phase2a was never forwarded
        eng.proxyleader_phase2b(np.array([(0, 0, 6, 0)], dtype=P2B))
    assert ei.value.status == -4
    eng.close()


def test_replica_range_stops_at_first_present_slot_and_batch_contract():
    f, LG, AG, per, cap = 1, 3, 1, 3, 1 << 16
    eng, ora = make(f, LG, AG, per, cap)
    RC = CHOSEN_RANGE
    ch = np.array([(0, 5), (3000, 1), (9001, 2)], dtype=CHOSEN)
    ora.replica_chosen(ch); eng.replica_chosen(ch)
    r = np.array([(0, 6000), (1, 9000), (2, 30002)], dtype=RC)       # three leader groups, disjoint slots
    both(lambda: eng.mencius_replica_chosen_range(r), ora.replica_chosen_range(r, cap))
    H.compare_log(eng, ora, 0, cap)
    assert eng.chosen_watermark() == ora.first_hole()
    log = eng.snapshot_log(0, cap)
    assert log[0] == 5 and log[3] == -1          # slot 0 was present: the whole range (0, 6000) was dropped
    assert log[4] == VALUE_NOOP and log[8998] == VALUE_NOOP and log[9001] == 2
    r = np.array([(3, 6000), (9004, 20000)], dtype=RC)
    both(lambda: eng.mencius_replica_chosen_range(r), ora.replica_chosen_range(r, cap))
    H.compare_log(eng, ora, 0, cap)
    # residues 1 and 2 were filled by the first call; residue 0 stopped at slot 3000
    assert eng.snapshot_log(2997, 7).tolist() == [VALUE_NOOP, VALUE_NOOP, VALUE_NOOP, 1, VALUE_NOOP, VALUE_NOOP, -1]
    assert eng.chosen_watermark() == ora.first_hole()
    # two records of one call covering a common slot: contract violation at the later one
    with pytest.raises(FpxError) as ei:
        eng.mencius_replica_chosen_range(np.array([(40000, 40100), (50000, 50010), (40030, 40200)], dtype=RC))
    assert (ei.value.status, ei.value.index) == (-12, 2)
    eng.close()


def test_one_range_of_a_million_slots():
    """Size-independent properties of the fills at BASELINE scale: one NoopRange over 2^20 slots of
    leader group 1 of 2, two acceptor groups."""
    f, LG, AG, per, cap = 1, 2, 2, 3, 1 << 21
    eng, _ = make(f, LG, AG, per, cap)
    start, end = 1, cap - 5
    eng.mencius_arm_range(np.array([(start, end, 2, -1)], dtype=P2A_RANGE))
    recs = np.array([(start, end, 2, dst(1, ag, a, AG)) for ag in range(AG) for a in range(per)], dtype=P2A_RANGE)
    ob, on = eng.mencius_acceptor_noop_range(recs)
    assert len(ob) == AG * per and len(on) == 0
    own = np.arange(start, end, LG)
    for ag in range(AG):
        r, _, vr, vv = eng.snapshot_acceptor(1 * AG + ag, 1, 0, cap)
        mine = own[(own // LG) % AG == ag]
        exp = np.full(cap, -1, dtype=np.int32); exp[mine] = 2
        assert r == 2 and np.array_equal(vr, exp) and (vv[mine] == VALUE_NOOP).all()
    oc = eng.mencius_range_phase2b(ob)
    assert oc.tolist() == [(start, end)]
    eng.replica_chosen(np.array([(0, 9)], dtype=CHOSEN))
    eng.mencius_replica_chosen_range(oc)
    log = eng.snapshot_log(0, cap)
    assert (log[own] == VALUE_NOOP).all() and (log[2::2] == -1).all()
    assert eng.chosen_watermark() == 2
    eng.close()


def test_ranges_on_slot_residue_shards():
    """Every shard sees every range message and fills its own residue class; the union of the
    shards' logs is the unsharded log."""
    f, LG, AG, per, cap, P = 1, 2, 1, 3, 6000, 3
    g = T.rng(5)
    _, ora = make(f, LG, AG, per, cap)
    engs = [Engine(f, AG, per, num_leaders=2, num_replicas=2, slot_capacity=cap, max_batch=1 << 12, protocol=MENCIUS,
                   num_leader_groups=LG, shard_index=i, shard_count=P) for i in range(P)]
    ranges = [(0, 2000, 0), (1, 4001, 0), (2000, 5000, 1)]
    arm = np.array([(s, e, r, -1) for s, e, r in ranges], dtype=P2A_RANGE)
    recs = np.array([(s, e, r, dst(s % LG, 0, a, AG)) for s, e, r in ranges for a in range(per)], dtype=P2A_RANGE)
    ora.arm_range(arm, cap)
    st, err, ob, on = ora.acceptor_noop_range(recs, cap)
    st, err, oc = ora.range_phase2b(ob)
    ora.replica_chosen_range(oc, cap)
    logs = []
    for e in engs:
        e.mencius_arm_range(arm)
        eb, en = e.mencius_acceptor_noop_range(recs)
        H.same(eb, ob, "sharded Phase2bNoopRange"); H.same(en, on, "sharded Nack")
        H.same(e.mencius_range_phase2b(eb), oc, "sharded ChosenNoopRange")
        e.mencius_replica_chosen_range(oc)
        logs.append(e.snapshot_log(0, cap))
    merged = np.full(cap, -1, dtype=np.int32)
    for i, lg_ in enumerate(logs):
        merged[i::P] = lg_[i::P]
    H.same(merged, ora.snapshot_log(0, cap), "union of the shards' logs")
    for i, e in enumerate(engs):
        for a in range(per):
            for lg in range(LG):
                _, _, vr, vv = e.snapshot_acceptor(lg * AG, a, 0, cap)
                _, _, ovr, ovv = ora.snapshot_acceptor(lg * AG, a, 0, cap)
                assert np.array_equal(vr[i::P], ovr[i::P]) and np.array_equal(vv[i::P], ovv[i::P])
        e.close()


def test_sharded_range_stops_at_a_slot_held_by_another_shard():
    """handleChosenNoopRange returns at the first slot already in the log (mencius/Replica.scala:476-480); on a
    log sharded by slot residue that slot may belong to another shard.  _first / min over shards / _fill gives
    the reference's log; each shard on its own would fill past the hit."""
    f, LG, AG, per, cap, P = 1, 2, 1, 3, 6000, 3
    _, ora = make(f, LG, AG, per, cap)
    engs = [Engine(f, AG, per, num_leaders=2, num_replicas=2, slot_capacity=cap, max_batch=1 << 12, protocol=MENCIUS,
                   num_leader_groups=LG, shard_index=i, shard_count=P) for i in range(P)]
    # slots 1000 (shard 1), 2501 (shard 2) and 4000 (shard 1) are chosen before the ranges arrive
    pre = np.array([(1000, 7), (2501, 8), (4000, 9)], dtype=CHOSEN)
    ora.replica_chosen(pre)
    for i, e in enumerate(engs):
        mine = pre[pre["slot"] % P == i]
        if len(mine):
            e.replica_chosen(mine)
    RC = CHOSEN_RANGE
    ranges = np.array([(0, 2000), (2001, 3001), (3000, 3800), (3800, 5000)], dtype=RC)
    ora.replica_chosen_range(ranges, cap)
    firsts = np.stack([e.mencius_replica_range_first(ranges) for e in engs])
    assert firsts[1, 0] == 1000 and firsts[0, 0] == Engine.RANGE_NO_HIT and firsts[2, 1] == 2501
    assert (firsts[:, 2] == Engine.RANGE_NO_HIT).all() and firsts[:, 3].min() == 4000
    bound = firsts.min(axis=0)
    for e in engs:
        e.mencius_replica_range_fill(ranges, bound)
    merged = np.full(cap, -1, dtype=np.int32)
    for i, e in enumerate(engs):
        merged[i::P] = e.snapshot_log(0, cap)[i::P]
    want = ora.snapshot_log(0, cap)
    H.same(merged, want, "union of the shards' logs")
    assert want[998] == VALUE_NOOP and want[1002] == -1 and want[3002] == VALUE_NOOP and want[4002] == -1
    for e in engs:
        e.close()


# --------------------------------------------------------------------------- vanilla Mencius skips
def vm_logs(eng, ora, n, cap):
    for s in range(n):
        k, r, v = ora.snapshot(s, 0, cap)
        _, _, vr, vv = eng.snapshot_acceptor(0, s, 0, cap)
        chosen = vr == 0x7fffffff
        assert np.array_equal(chosen, k == 3), f"server {s}: ChosenEntry positions"
        assert np.array_equal(vv[chosen], v[chosen])
        pend = k == 2
        assert np.array_equal(vr[pend], r[pend]) and (vr[k == 0] == -1).all()


@pytest.mark.parametrize("f", [1, 3, 7])
def test_vanilla_skips_match_oracle(f):
    """S/vanillamencius Skip: advanceWithSkips at the skipping server and handleSkip elsewhere, against the
    oracle's logs.  f = 1, 3, 7: 3, 7 and 15 servers, i.e. 8-, 16- and 32-word rows."""
    n = 2 * f + 1
    cap = 40000
    g = T.rng(60 + f)
    eng = Engine(f, 1, n, num_leaders=f + 1, num_replicas=f + 1, slot_capacity=cap, max_batch=1 << 16,
                 protocol=VANILLA_MENCIUS)
    ora = O.VanillaMencius(f)
    # every server proposes a few of its own slots, then falls behind and skips ahead
    next_slot = list(range(n))
    for step in range(6):
        reqs = []
        for s in range(n):
            k = int(g.integers(0, 40))
            sl = next_slot[s] + n * np.arange(k)
            next_slot[s] += n * k
            reqs += [(int(x), 0, int(x) * 3 + 1, s) for x in sl]
        req = np.array(reqs, dtype=P2A).reshape(-1)
        if len(req):
            eng.vm_client_request(req)
            assert ora.client_request(req) == (0, -1)
        hi = max(next_slot)
        skips = []
        for s in range(n):
            if g.random() < 0.7 and next_slot[s] < hi:
                stop = hi + int(g.integers(0, n))
                skips.append((s, next_slot[s], stop, 1))                       # advanceWithSkips at s
                skips += [(o, next_slot[s], stop, 0) for o in range(n) if o != s and g.random() < 0.8]  # handleSkip elsewhere
                next_slot[s] += n * ((stop - next_slot[s] + n - 1) // n)
        sk = np.array(skips, dtype=VM_SKIP).reshape(-1)
        sk = sk[g.permutation(len(sk))]
        both(lambda: eng.vm_skip(sk), ora.skip(sk, cap))
        vm_logs(eng, ora, n, max(next_slot) + n)
    # a Phase2a for a skipped slot is answered Chosen(Noop) (:1017-1027)
    own = np.array([(s, n + s, 2 * n + s, 1) for s in range(n)], dtype=VM_SKIP)
    eng2 = Engine(f, 1, n, num_leaders=f + 1, num_replicas=f + 1, slot_capacity=64, max_batch=64, protocol=VANILLA_MENCIUS)
    ora2 = O.VanillaMencius(f)
    both(lambda: eng2.vm_skip(own), ora2.skip(own, 64))
    q = np.array([(n + 1, 0, 5, 1)], dtype=P2A)
    rep = eng2.vm_phase2a(q)
    H.same(rep, ora2.phase2a(q)[2], "Phase2a on a skipped slot")
    assert rep["group"][0] == 2 and rep["round"][0] == VALUE_NOOP
    # logger.check failures and preconditions
    req = np.array([(1, 0, 4, 1)], dtype=P2A)
    eng2.vm_client_request(req); ora2.client_request(req)
    for bad in ([(1, 1, 1 + n, 1)], [(1, n + 1, 2 * n + 1, 1)], [(1, 2, 9, 1)], [(n, 0, 4, 0)], [(0, 5, 4, 0)], [(0, 0, 65, 0)]):
        b = np.array(bad, dtype=VM_SKIP)
        r = ora2.skip(b, 64)
        assert r[0] != 0
        both(lambda: eng2.vm_skip(b), r)
    eng.close(); eng2.close()
