"""Every engine across the wrap of its 32-bit delivery numbers and batch tags, against the CPU oracle (which has
no counters).  The host counters are started just below their wrap through Engine.set_counters /
EpaxosReplica.set_counters, so that real calls lay down stamps, log numbers and claims near the top; the
renormalization or the tag wrap then fires in the middle of the trace while that state is still live.  Every
test also reads the counters back and asserts that they restarted where the trace expects, so a change of a
threshold cannot make a test pass without running the path.

  tally seq_base         renormalize_stamps_kernel on the primary and the overflow-table rows
  replica rseq_base      renormalize_rlog_kernel (replica_chosen, replica_chosen_last_dev, the fused step's 2n bound,
                         the asynchronous host step, the Mencius range fill)
  Mencius rng_seq_base   renormalize_range_stamps_kernel
  EPaxos seq_base        ep_renormalize_kernel (PreAcceptOk, AcceptOk and PrepareOk stamps)
  EPaxos tag             claims and counts of the previous cycle are forgotten at the wrap
  vanilla Mencius tag    claims of the previous cycle are forgotten at the wrap"""
import random

import numpy as np
import pytest

import epaxos_recovery_oracle as R
import harness as H
from epaxos_recovery_traces import Trace
from frankenpaxos_b200 import (CHOSEN, CHOSEN_RANGE, MENCIUS, P2A, P2A_RANGE, P2B, VALUE_NOOP, VANILLA_MENCIUS,
                               Engine, FpxError)
from frankenpaxos_b200 import traces as T
from frankenpaxos_b200.epaxos import EpaxosReplica
from oracle import fpx_oracle_py as O

pytestmark = pytest.mark.gpu

TOP = 0xFFFFFFFF
LAST_TAG = 0xFFFFFFFE          # the last batch tag of a cycle; the call after it uses tag 1
CFG1, _ = T.config_by_name("cfg1")
CFG2, _ = T.config_by_name("cfg2")
CFG3, _ = T.config_by_name("cfg3")
TALLY_SHAPES = {"cfg2": CFG2, "cfg3": CFG3, "maj15": H.WIDE_SHAPES["maj15"]}


def start_for(bounds, at):
    """The counter value from which calls with these bounds renormalize at call `at` and at no call before it
    (a call of bound b renormalizes when counter > 2^32 - 1 - b - 16)."""
    return TOP - 16 - sum(bounds[:at]) - (bounds[at] + 1) // 2


def _td(x, cols=None):
    import torch
    a = x.view(np.int32).reshape(len(x), -1) if cols is None else np.asarray(x, dtype=np.int32).reshape(len(x), cols)
    return torch.from_numpy(a.copy()).to(torch.device("cuda", 0))


def block_votes(cfg, g, slots, round_=0, values=None, thrifty=True):
    return T.votes_of(T.phase2as(g, slots, cfg["f"], cfg["num_acceptor_groups"], cfg["acceptors_per_group"],
                                 cfg["flexible"], round_, values, thrifty=thrifty))


# --------------------------------------------------------------------------- tally seq_base
@pytest.mark.parametrize("max_sub", [0, 700])
@pytest.mark.parametrize("path", ["auto", "exact"])
@pytest.mark.parametrize("shape", list(TALLY_SHAPES))
def test_tally_stamps_renormalize_in_the_middle_of_a_trace(shape, path, max_sub):
    """Every slot armed in round 0, a third also in round 1 (a second live round: its key lives in the
    overflow table), every acceptor sent a copy (round 0's copies first), the Phase2b stream with 20 %
    duplicates and late votes to Done keys in eight calls.  seq_base starts so that the fourth call
    renormalizes; keys that got votes before it complete in it or after it.  max_sub = 700 cuts the
    renormalizing call into several launches.  Chosen streams, every acceptor and the log."""
    cfg = TALLY_SHAPES[shape]
    n_slots = 1500
    g = T.rng(len(shape) + 10 * (path == "exact") + max_sub)
    eng, ora = H.make_pair(cfg, n_slots, max_batch=1 << 17, overflow_capacity=1 << 12, tally_max_sub=max_sub)
    eng.set_tally_path(path == "exact")
    slots = np.arange(n_slots, dtype=np.int32)
    dual = slots[::3]
    H.arm(eng, ora, np.concatenate([T.arms(slots, 0, slots * 8), T.arms(dual, 1, dual * 8 + 1)]))
    mk = lambda s, r, v: T.phase2as(g, s, cfg["f"], cfg["num_acceptor_groups"], cfg["acceptors_per_group"],
                                    cfg["flexible"], r, v, thrifty=False)
    p0, p1 = mk(slots, 0, slots * 8), mk(dual, 1, dual * 8 + 1)
    ob, _ = H.phase2a(eng, ora, np.concatenate([p0[g.permutation(len(p0))], p1[g.permutation(len(p1))]]))
    H.compare_acceptors(eng, ora, cfg, 0, n_slots)
    votes = np.concatenate([ob, ob[g.integers(0, len(ob), size=len(ob) // 5)]])
    chunks = np.array_split(votes[g.permutation(len(votes))], 8)
    at = 3
    start = start_for([len(c) for c in chunks], at)
    eng.set_counters(seq_base=start)
    voted_before = set()
    completed_after = set()
    for k, chunk in enumerate(chunks):
        st, c = H.phase2b(eng, ora, chunk)
        assert st == 0
        H.replica(eng, ora, c)
        seq = eng.counters()["seq_base"]
        if k < at:
            assert seq == start + sum(len(x) for x in chunks[:k + 1]), (k, seq)
            voted_before |= set(chunk["slot"].tolist())
        else:
            assert seq == 1 + sum(len(x) for x in chunks[at:k + 1]), (k, seq)
            completed_after |= set(c["slot"].tolist())
    assert len(voted_before & completed_after) > 100
    H.compare_acceptors(eng, ora, cfg, 0, n_slots)
    H.compare_log(eng, ora, 0, n_slots)
    eng.close()


@pytest.mark.parametrize("path", ["auto", "exact"])
@pytest.mark.parametrize("shape", list(TALLY_SHAPES))
def test_tally_renormalizes_exactly_when_a_call_would_come_within_16_of_the_wrap(shape, path):
    """A call of n votes that starts at seq_base = 2^32 - 1 - n - 16 does not renormalize; the next call does.
    The first call carries all but one of the quorum's votes of every key, in round 0 and in round 1 (primary
    rows and overflow-table rows hold stamps at the very top); the second carries the completing votes."""
    cfg = TALLY_SHAPES[shape]
    g = T.rng(5 + len(shape))
    n_slots = 1200
    eng, ora = H.make_pair(cfg, n_slots, max_batch=1 << 17, overflow_capacity=1 << 12)
    eng.set_tally_path(path == "exact")
    slots = np.arange(n_slots, dtype=np.int32)
    dual = slots[1::2]
    H.arm(eng, ora, np.concatenate([T.arms(slots, 0, slots * 8), T.arms(dual, 1, dual * 8 + 1)]))
    first, last = [], []
    for s, r in ((slots, 0), (dual, 1)):
        v = block_votes(cfg, g, s, r, s * 8 + r)           # one thrifty quorum per key, in key order
        q = len(v) // len(s)
        v = v.reshape(len(s), q)
        first.append(v[:, :q - 1].reshape(-1))
        last.append(v[:, q - 1])
    first = np.concatenate(first)
    first = first[g.permutation(len(first))]
    second = np.concatenate(last + [first[: len(first) // 4]])      # + re-deliveries of first votes
    second = second[g.permutation(len(second))]
    n = len(first)
    eng.set_counters(seq_base=TOP - n - 16)
    st, c = H.phase2b(eng, ora, first)
    assert st == 0 and len(c) == 0
    assert eng.counters()["seq_base"] == TOP - 16
    st, c = H.phase2b(eng, ora, second)
    assert st == 0 and len(c) == n_slots + len(dual)
    assert eng.counters()["seq_base"] == 1 + len(second)
    H.replica(eng, ora, c)
    H.compare_log(eng, ora, 0, n_slots)
    eng.close()


# --------------------------------------------------------------------------- replica rseq_base
def test_replica_log_numbers_renormalize_in_the_middle_of_a_trace():
    """replica_chosen calls of fresh slots mixed with Chosen records that carry another value for slots chosen
    in earlier calls, and followed by such records for slots of the same call; rseq_base starts so that the
    third of six calls renormalizes.  The first value of every slot wins on both sides of the collapse."""
    g = T.rng(3)
    n_slots = 3000
    eng, ora = H.make_pair(CFG2, n_slots)
    calls = []
    for k in range(6):
        fresh = np.arange(k * 400, (k + 1) * 400, dtype=np.int32)
        c = np.zeros(400 + 150 * (k > 0), dtype=CHOSEN)
        c["slot"] = np.concatenate([fresh, g.integers(0, max(k, 1) * 400, size=150 * (k > 0)).astype(np.int32)])
        c["value_id"] = c["slot"] * 10 + (np.arange(len(c)) >= 400) * (k + 1)
        d = np.zeros(50, dtype=CHOSEN)
        d["slot"] = fresh[g.integers(0, 400, size=50)]
        d["value_id"] = d["slot"] * 10 + 9
        calls.append(np.concatenate([c[g.permutation(len(c))], d]))
    at = 2
    eng.set_counters(rseq_base=start_for([len(c) for c in calls], at))
    for k, c in enumerate(calls):
        H.replica(eng, ora, c)
        rseq = eng.counters()["rseq_base"]
        assert (rseq == 1 + sum(len(x) for x in calls[at:k + 1])) == (k >= at), (k, rseq)
    log = eng.snapshot_log(0, n_slots)
    assert np.array_equal(log[:2400], np.arange(2400) * 10)
    H.compare_log(eng, ora, 0, n_slots)
    eng.close()


def _rechoose_steps(cfg, g, windows, W, n_again):
    """(arm, votes) per step: window w's slots in round 0, and the first n_again slots of window w-1 (chosen in
    the step before) armed and chosen again in round 1 with another value."""
    steps = []
    for w in range(windows):
        s = np.arange(w * W, (w + 1) * W, dtype=np.int32)
        arm = [T.arms(s, 0, s * 10)]
        v = [block_votes(cfg, g, s, 0, s * 10)]
        if w:
            x = np.arange((w - 1) * W, (w - 1) * W + n_again, dtype=np.int32)
            arm.append(T.arms(x, 1, x * 10 + 1))
            v.append(block_votes(cfg, g, x, 1, x * 10 + 1))
        v = np.concatenate(v)
        steps.append((np.concatenate(arm), v[g.permutation(len(v))]))
    return steps


def fused_step(eng, votes, arm=None, p2a=None):
    """fpx_step_dev; returns (sync result, Chosen stream)."""
    import torch
    dev = torch.device("cuda", 0)
    d_a = _td(arm) if arm is not None and len(arm) else None
    d_p = _td(p2a) if p2a is not None and len(p2a) else None
    d_v = _td(votes)
    n_p2a = 0 if d_p is None else len(p2a)
    o_b = torch.zeros((max(n_p2a, 1), 4), dtype=torch.int32, device=dev)
    o_n = torch.zeros((max(n_p2a, 1), 2), dtype=torch.int32, device=dev)
    o_c = torch.zeros((len(votes), 2), dtype=torch.int32, device=dev)
    d_wm = torch.zeros(1, dtype=torch.int32, device=dev)
    ptr = lambda t: t.data_ptr() if t is not None else None
    eng.step_dev(ptr(d_a), 0 if d_a is None else len(arm), ptr(d_p), n_p2a, o_b.data_ptr(), o_n.data_ptr(),
                 d_v.data_ptr(), len(votes), o_c.data_ptr(), d_wm.data_ptr())
    r = eng.sync()
    assert r.watermark == int(d_wm.item())
    return r, o_c[: r.n_chosen].cpu().numpy().view(CHOSEN).reshape(-1)


def last_dev_step(eng, votes):
    """proxyleader_phase2b_dev, then replica_chosen_last_dev on its output; returns the Chosen stream."""
    import torch
    d_v = _td(votes)
    d_c = torch.zeros((len(votes), 2), dtype=torch.int32, device=torch.device("cuda", 0))
    eng.proxyleader_phase2b_dev(d_v.data_ptr(), len(votes), d_c.data_ptr())
    eng.replica_chosen_last_dev(d_c.data_ptr())
    r = eng.sync()
    return d_c[: r.n_chosen].cpu().numpy().view(CHOSEN).reshape(-1)


@pytest.mark.parametrize("form", ["last_dev", "fused"])
def test_device_replica_forms_renormalize_in_the_middle_of_a_trace(form):
    """replica_chosen_last_dev (bound: the last tally call's vote count) and the fused step_dev (bound: twice the
    vote count) over four steps; every step re-chooses slots of the step before with another value.  rseq_base
    starts so that the third step renormalizes.  Chosen streams, watermark and log."""
    cfg = CFG2
    g = T.rng(11 + (form == "fused"))
    W = 2000
    eng, ora = H.make_pair(cfg, 4 * W, overflow_capacity=1 << 12)
    steps = _rechoose_steps(cfg, g, 4, W, 300)
    scale = 2 if form == "fused" else 1
    bounds = [scale * len(v) for _, v in steps]
    at = 2
    eng.set_counters(rseq_base=start_for(bounds, at))
    for k, (arm, votes) in enumerate(steps):
        if form == "fused":            # the arm batch rides in the fused call
            assert ora.arm(arm) == (0, -1)
        else:
            H.arm(eng, ora, arm)
        st, _, oc = ora.proxyleader_phase2b(votes)
        assert st == 0
        ora.replica_chosen(oc)
        if form == "fused":
            _, c = fused_step(eng, votes, arm=arm)
        else:
            c = last_dev_step(eng, votes)
        H.same(c, oc, f"Chosen stream, step {k}")
        assert eng.chosen_watermark() == ora.executed_watermark()
        rseq = eng.counters()["rseq_base"]
        assert (rseq == 1 + sum(bounds[at:k + 1])) == (k >= at), (k, rseq)
    log = eng.snapshot_log(0, 4 * W)
    assert np.array_equal(log[:4 * W], np.arange(4 * W) * 10)
    H.compare_log(eng, ora, 0, 4 * W)
    eng.close()


@pytest.mark.parametrize("path", ["auto", "exact"])
def test_fused_step_renormalizes_on_its_2n_bound(path):
    """A fused call of n votes numbers its co-located log puts below rseq_base + 2n (a launch of a split call
    numbers its records after the earlier launches' votes and their Chosen records).  With rseq_base =
    2^32 - 1 - n - 16 the n-bound fits and the 2n-bound does not: the step renormalizes.  The call is cut into
    256-vote launches and the slots chosen in the step before are chosen again, with another value, at the
    end of its stream; the log keeps the first value."""
    cfg = CFG1
    g = T.rng(21)
    eng, ora = H.make_pair(cfg, 4000, overflow_capacity=1 << 12, tally_max_sub=256)
    eng.set_tally_path(path == "exact")
    S = np.arange(500, dtype=np.int32)
    F = np.arange(500, 3500, dtype=np.int32)
    arm1, v1 = T.arms(S, 0, S * 10), block_votes(cfg, g, S, 0, S * 10)
    v1 = v1[g.permutation(len(v1))]
    arm2 = np.concatenate([T.arms(F, 0, F * 10), T.arms(S, 1, S * 10 + 1)])
    vf, vs = block_votes(cfg, g, F, 0, F * 10), block_votes(cfg, g, S, 1, S * 10 + 1)
    v2 = np.concatenate([vf[g.permutation(len(vf))], vs[g.permutation(len(vs))]])
    n1, n2 = len(v1), len(v2)
    eng.set_counters(rseq_base=TOP - n2 - 16 - 2 * n1)
    for k, (arm, votes) in enumerate([(arm1, v1), (arm2, v2)]):
        assert ora.arm(arm) == (0, -1)
        st, _, oc = ora.proxyleader_phase2b(votes)
        assert st == 0
        ora.replica_chosen(oc)
        _, c = fused_step(eng, votes, arm=arm)
        H.same(c, oc, f"Chosen stream, step {k}")
    if path == "exact":
        assert eng.last_tally_path == "exact"
    log = eng.snapshot_log(0, 4000)
    assert np.array_equal(log[S], S * 10)
    H.compare_log(eng, ora, 0, 4000)
    assert eng.counters()["rseq_base"] == 1 + 2 * n2
    eng.close()


def test_asynchronous_host_step_with_two_lanes_in_flight_across_the_collapse():
    """step_submit twice, then step_wait twice: the second submission renormalizes the log numbers while the
    first step's kernels are still queued ahead of it.  The second step re-chooses slots of the first with
    another value.  Phase2b and Chosen streams, watermark and log."""
    import torch
    cfg = CFG2
    g = T.rng(31)
    W = 2000
    eng, ora = H.make_pair(cfg, 2 * W, overflow_capacity=1 << 12)
    a1, p1, b1 = T.workload(41, cfg, W)
    a2, p2, b2 = T.workload(42, cfg, W, slot0=W)
    x = np.arange(300, dtype=np.int32)
    a2 = np.concatenate([a2, T.arms(x, 1, x + 7 * W)])
    b2 = np.concatenate([b2, block_votes(cfg, g, x, 1, x + 7 * W)])
    b2 = b2[g.permutation(len(b2))]
    pin = lambda r: torch.from_numpy(r.view(np.int32).reshape(len(r), -1).copy()).pin_memory()
    steps = [(a1, p1, b1), (a2, p2, b2)]
    eng.set_counters(rseq_base=start_for([2 * len(b) for _, _, b in steps], 1))
    held = []
    for a, p, b in steps:
        ha, hp, hb = pin(a), pin(p), pin(b)
        ob = torch.zeros((len(p), 4), dtype=torch.int32).pin_memory()
        on = torch.zeros((len(p), 2), dtype=torch.int32).pin_memory()
        oc = torch.zeros((len(b), 2), dtype=torch.int32).pin_memory()
        eng.step_submit(ha.data_ptr(), len(a), hp.data_ptr(), len(p), hb.data_ptr(), len(b), ob.data_ptr(),
                        on.data_ptr(), oc.data_ptr())
        held.append((ha, hp, hb, ob, on, oc))
    assert eng.counters()["rseq_base"] == 1 + 2 * len(b2)
    for k, (a, p, b) in enumerate(steps):
        n_p2b, n_nack, n_chosen, wm = eng.step_wait()
        assert ora.arm(a) == (0, -1)
        st, _, eb, en = ora.acceptor_phase2a(p)
        assert st == 0 and (n_p2b, n_nack) == (len(eb), len(en))
        st, _, ec = ora.proxyleader_phase2b(b)
        assert st == 0
        ora.replica_chosen(ec)
        _, _, _, ob, _, oc = held[k]
        H.same(ob[:n_p2b].numpy().view(P2B).reshape(-1), eb, f"Phase2b stream, step {k}")
        H.same(oc[:n_chosen].numpy().view(CHOSEN).reshape(-1), ec, f"Chosen stream, step {k}")
        assert wm == ora.executed_watermark()
    assert np.array_equal(eng.snapshot_log(0, 300), np.arange(300))
    H.compare_log(eng, ora, 0, 2 * W)
    eng.close()


# --------------------------------------------------------------------------- Mencius ranges
def _mencius(cap, LG=2, AG=2, per=3, f=1):
    eng = Engine(f, AG, per, num_leaders=2, num_replicas=2, slot_capacity=cap, max_batch=1 << 16, protocol=MENCIUS,
                 num_leader_groups=LG)
    return eng, O.MultiPaxos(f, AG, per, False, 2, 2, mencius_leader_groups=LG)


def test_range_votes_split_across_the_range_stamp_collapse():
    """NoopRanges of two leader groups over two acceptor groups, every acceptor voting, votes with duplicates in
    three calls; rng_seq_base starts so that the second call renormalizes.  Every range got votes in the
    first call, so every chosen range completes across the collapse.  ChosenNoopRange streams and the log."""
    LG, AG, per, cap = 2, 2, 3, 8192
    g = T.rng(51)
    eng, ora = _mencius(cap, LG, AG, per)
    ranges = [(lg + LG * 40 * k, lg + LG * 40 * (k + 1), 0) for lg in range(LG) for k in range(40)]
    arm = np.array([(s, e, r, -1) for s, e, r in ranges], dtype=P2A_RANGE)
    assert ora.arm_range(arm, cap) == (0, -1)
    eng.mencius_arm_range(arm)
    recs = np.array([(s, e, r, ((s % LG * AG + ag) << 16) | a) for s, e, r in ranges for ag in range(AG)
                     for a in range(per)], dtype=P2A_RANGE)
    recs = recs[g.permutation(len(recs))]
    st, _, ob, on = ora.acceptor_noop_range(recs, cap)
    assert st == 0 and len(on) == 0
    eb, en = eng.mencius_acceptor_noop_range(recs)
    H.same(eb, ob, "Phase2bNoopRange stream")
    # one vote of every range first, the rest shuffled with duplicates
    first = np.unique(ob["slot_start"], return_index=True)[1]
    rest = np.delete(ob, first)
    rest = np.concatenate([rest, rest[g.integers(0, len(rest), size=len(rest) // 4)]])
    rest = rest[g.permutation(len(rest))]
    h = len(rest) // 2
    chunks = [ob[first], rest[:h], rest[h:]]
    eng.set_counters(rng_seq_base=start_for([len(c) for c in chunks], 1))
    chosen = []
    for k, chunk in enumerate(chunks):
        st, _, oc = ora.range_phase2b(chunk)
        assert st == 0
        H.same(eng.mencius_range_phase2b(chunk), oc, f"ChosenNoopRange stream, call {k}")
        chosen.append(oc)
        rs = eng.counters()["rng_seq_base"]
        assert (rs == 1 + sum(len(c) for c in chunks[1:k + 1])) == (k >= 1), (k, rs)
    chosen = np.concatenate(chosen)
    assert len(chosen) == len(ranges)
    assert ora.replica_chosen_range(chosen, cap) == (0, -1)
    eng.mencius_replica_chosen_range(chosen)
    H.compare_log(eng, ora, 0, cap)
    eng.close()


@pytest.mark.parametrize("form", ["one_call", "first_fill"])
def test_range_fill_renormalizes_the_log_numbers(form):
    """Slots chosen at log numbers just below the wrap, then a range fill whose call renormalizes (the whole
    fill as one call, or its first-hit pass and its fill pass), then Chosen records with other values for
    slots of both: the values already in the log win."""
    LG, cap = 3, 1 << 14
    eng, ora = _mencius(cap, LG=LG, AG=1)
    ch = np.zeros(600, dtype=CHOSEN)
    ch["slot"] = np.arange(0, 6000, 10)
    ch["value_id"] = ch["slot"] + 1
    eng.set_counters(rseq_base=TOP - 16 - len(ch) - 2)
    H.replica(eng, ora, ch)
    assert eng.counters()["rseq_base"] == TOP - 18
    rng = np.array([(3, 9000), (4, 9000), (8, 12000)], dtype=CHOSEN_RANGE)
    assert ora.replica_chosen_range(rng, cap) == (0, -1)
    if form == "one_call":
        eng.mencius_replica_chosen_range(rng)
    else:
        first = eng.mencius_replica_range_first(rng)
        assert eng.counters()["rseq_base"] == TOP - 18          # the first-hit pass numbers nothing
        eng.mencius_replica_range_fill(rng, first)
    assert eng.counters()["rseq_base"] == 1 + len(rng)
    late = np.zeros(407, dtype=CHOSEN)
    late["slot"] = np.concatenate([np.arange(0, 8000, 20), [3, 6, 27, 4, 7, 8, 17]])
    late["value_id"] = 7
    H.replica(eng, ora, late)
    log = eng.snapshot_log(0, cap)
    assert log[10] == 11 and log[4000] == 4001 and log[6] == log[7] == log[17] == VALUE_NOOP
    H.compare_log(eng, ora, 0, cap)
    eng.close()


# --------------------------------------------------------------------------- EPaxos seq_base
def apply(gpu, ora, call, rows):
    """one call on both backends; replies and events must agree exactly"""
    rows = np.asarray(rows, dtype=np.int32)
    a = getattr(ora, call)(rows)
    if call in ("prepare_phase", "prepareok"):
        assert a[0] == 0, (call, a)
        a = a[2]
    elif call == "lead":
        assert a == (0, -1)
    c = getattr(gpu, call)(rows)
    if call not in ("lead", "commit"):
        assert np.asarray(c).tolist() == np.asarray(a).tolist(), (call, rows.tolist())
    return a


def check_entries(gpu, ora, insts):
    for rep, num in sorted(set(insts)):
        x, y = gpu.entry(rep, num), ora.entry(rep, num)
        assert (x[0].tolist(), int(x[1]), x[2].tolist()) == (y[0].tolist(), int(y[1]), y[2].tolist()), (rep, num)


STAMP_CALLS = ("preacceptok", "acceptok", "prepareok")


@pytest.mark.parametrize("f", [1, 2, 3])
def test_epaxos_mixed_traces_across_stamp_collapses(f):
    """Mixed traces of all eleven handlers (tests/epaxos_recovery_traces.py) against the recovery oracle.  Every
    60 calls the stamp numbering jumps forward to within a few batches of its wrap (as if calls without
    responses had run), so that PreAcceptOk, AcceptOk and PrepareOk quorums are collected across several
    collapses."""
    index = f % (2 * f + 1)
    gpu, ora = EpaxosReplica(f, index, 6, 1 << 12), R.EPaxos(f, index)
    trace = Trace(f, index, 6, 4100 + f, ora, max_batch=10)
    g = random.Random(f)
    collapses = 0
    for step in range(420):
        if step % 60 == 10:
            gpu.set_counters(seq_base=TOP - 16 - g.randint(20, 120))
        call, rows = trace.step()
        before = gpu.counters()["seq_base"]
        out = apply(gpu, ora, call, rows)
        trace.observe(call, np.asarray(rows), out)
        after = gpu.counters()["seq_base"]
        if call in STAMP_CALLS:
            collapses += after < before
            assert after == (1 + len(rows) if after < before else before + len(rows))
        check_entries(gpu, ora, [(int(r[0]), int(r[1])) for r in rows])
    assert collapses >= 5
    gpu.close()


def test_epaxos_quorums_split_across_the_collapse():
    """Directed: for each of PreAcceptOk (slow path), AcceptOk (commit) and PrepareOk (restart) the first
    responses of every instance are stamped in a call just below the wrap and the completing ones in the next
    call, which renormalizes.  Events, entries and largestBallot against the oracle."""
    f, idx = 2, 0
    n = 2 * f + 1
    K = 40
    gpu, ora = EpaxosReplica(f, idx, K, 1024), R.EPaxos(f, idx)
    A = [(0, k) for k in range(K)]
    B = [(1, k) for k in range(K)]
    z = [0] * n

    def split(call, first, second):
        gpu.set_counters(seq_base=start_for([len(first), len(second)], 1))
        apply(gpu, ora, call, first)
        assert gpu.counters()["seq_base"] > TOP - 16 - len(second)
        out = apply(gpu, ora, call, second)
        assert gpu.counters()["seq_base"] == 1 + len(second)
        return out

    apply(gpu, ora, "lead", [[r, k, 1, idx, k, 0, 1, 0] + z for r, k in A])     # avoid the fast path
    # own + replica 1 + replica 2 = the slow quorum f + 1
    ev = split("preacceptok", [[r, k, 1, idx, 1, k % 3] + [k % 2] * n for r, k in A],
               [[r, k, 1, idx, 2, 1] + [1] * n for r, k in A])
    assert all(e[0] == 2 for e in ev)
    ev = split("acceptok", [[r, k, 1, idx, 1, 0] for r, k in A], [[r, k, 1, idx, 2, 0] for r, k in A])
    assert all(e[0] == 4 for e in ev)
    ballots = apply(gpu, ora, "prepare_phase", [[r, k] for r, k in B])
    ok = lambda s: [[r, k, int(b[0]), int(b[1]), s, -1, -1, 0, 0] for (r, k), b in zip(B, ballots)]
    ev = split("prepareok", ok(1) + ok(2), ok(3))
    assert all(e[0] == 1 for e in ev)
    check_entries(gpu, ora, A + B)
    gpu.close()


# --------------------------------------------------------------------------- EPaxos batch tag
def _ep_rows(call, n, inst, b_ord, salt=0):
    r, k = inst
    if call == "lead":
        return [r, k, b_ord, 0, 5 + salt, 1, 0, 0] + [1] * n
    if call == "preaccept":
        return [r, k, b_ord, 1, 5 + salt, 1] + [1] * n + [2] * n
    return [r, k, 5 + salt, 2] + [3] * n                                        # commit


def test_epaxos_mixed_trace_across_the_tag_wrap():
    f, idx = 2, 1
    gpu, ora = EpaxosReplica(f, idx, 6, 1 << 12), R.EPaxos(f, idx)
    gpu.set_counters(tag=LAST_TAG - 40)
    trace = Trace(f, idx, 6, 91, ora, max_batch=10)
    wrapped = False
    for _ in range(120):
        call, rows = trace.step()
        before = gpu.counters()["tag"]
        out = apply(gpu, ora, call, rows)
        trace.observe(call, np.asarray(rows), out)
        after = gpu.counters()["tag"]
        assert after == (1 if before == LAST_TAG else before + 1)
        wrapped |= after == 1
        check_entries(gpu, ora, [(int(r[0]), int(r[1])) for r in rows])
    assert wrapped
    gpu.close()


@pytest.mark.parametrize("call", ["lead", "preaccept", "commit"])
def test_epaxos_duplicate_after_the_tag_wrap_is_reported(call):
    """Instance X is claimed by the last call of a cycle; in the first call of the next one, a second record for
    X in the same batch is a contract violation at its index (E1)."""
    f = 2
    n = 2 * f + 1
    X, Y, Z = (3, 0), (3, 1), (4, 2)
    gpu = EpaxosReplica(f, 0, 8, 1024)
    gpu.set_counters(tag=LAST_TAG)
    getattr(gpu, call)(np.asarray([_ep_rows(call, n, X, 1)], dtype=np.int32))
    assert gpu.counters()["tag"] == 1
    rows = [_ep_rows(call, n, Y, 2), _ep_rows(call, n, X, 2), _ep_rows(call, n, Z, 2), _ep_rows(call, n, X, 3, 1)]
    with pytest.raises(FpxError) as ei:
        getattr(gpu, call)(np.asarray(rows, dtype=np.int32))
    assert (ei.value.status, ei.value.index) == (-12, 3)
    gpu.close()


@pytest.mark.parametrize("call", ["lead", "preaccept", "commit"])
def test_epaxos_instance_claimed_with_the_same_tag_one_cycle_earlier(call):
    """Instance X is last claimed by the call with tag 1; the tag then runs through its cycle without touching X
    (jumped to its last value, one real call made there).  The next cycle's tag-1 call touches X once: a
    correct batch that must succeed, with the oracle's replies and entries."""
    f = 2
    n = 2 * f + 1
    X, Y, Z = (3, 0), (3, 1), (4, 2)
    gpu, ora = EpaxosReplica(f, 0, 8, 1024), R.EPaxos(f, 0)
    assert gpu.counters()["tag"] == 1
    apply(gpu, ora, call, [_ep_rows(call, n, X, 1)])
    gpu.set_counters(tag=LAST_TAG)
    apply(gpu, ora, call, [_ep_rows(call, n, Y, 1)])
    assert gpu.counters()["tag"] == 1
    apply(gpu, ora, call, [_ep_rows(call, n, Z, 2), _ep_rows(call, n, X, 2, 1)])
    check_entries(gpu, ora, [X, Y, Z])
    gpu.close()


def test_epaxos_lone_replacing_preacceptok_after_the_tag_wrap():
    """A PreAcceptOk of replica 1 for X counted under tag 2; a cycle later, under tag 2 again, replica 1's
    response with new content comes alone for X: it replaces the stored answer and is no contract violation."""
    f, idx = 2, 0
    n = 2 * f + 1
    X, Y, Z = (0, 0), (0, 1), (0, 2)
    gpu, ora = EpaxosReplica(f, idx, 8, 1024), R.EPaxos(f, idx)
    lead = lambda i: [i[0], i[1], 1, idx, 5, 0, 0, 0] + [0] * n
    apply(gpu, ora, "lead", [lead(X)])                                             # tag 1
    apply(gpu, ora, "preacceptok", [[X[0], X[1], 1, idx, 1, 1] + [1] * n])          # tag 2
    gpu.set_counters(tag=LAST_TAG)
    apply(gpu, ora, "lead", [lead(Y)])
    assert gpu.counters()["tag"] == 1
    apply(gpu, ora, "lead", [lead(Z)])                                             # tag 1
    assert gpu.counters()["tag"] == 2
    apply(gpu, ora, "preacceptok", [[X[0], X[1], 1, idx, 1, 2] + [0] * n])          # tag 2, replacing
    check_entries(gpu, ora, [X, Y, Z])
    gpu.close()


# --------------------------------------------------------------------------- vanilla Mencius batch tag
def _vanilla(f, cap):
    n = 2 * f + 1
    eng = Engine(f, 1, n, num_leaders=f + 1, num_replicas=f + 1, slot_capacity=cap, max_batch=1 << 15,
                 protocol=VANILLA_MENCIUS)
    return eng, O.VanillaMencius(f)


def test_vanilla_trace_across_the_tag_wrap():
    """vm_step_dev windows with stale re-deliveries of the previous window's Phase2as (to cells claimed by an
    earlier call), and vm_learn_chosen between them; the tag wraps after the second window.  Phase2a
    replies, Chosen streams, watermark and log."""
    import torch
    f, W = 1, 1000
    n = 2 * f + 1
    dev = torch.device("cuda", 0)
    eng, ora = _vanilla(f, 4 * W)
    eng.set_counters(vm_tag=LAST_TAG - 3)
    g = T.rng(61)
    prev = None
    tags = []
    for w in range(4):
        req, p, b = T.vanilla_cfg5(70 + w, f, W, slot_offset=w * W)
        if prev is not None:
            p = np.concatenate([p, prev[g.integers(0, len(prev), size=len(prev) // 4)]])
            p = p[g.permutation(len(p))]
            # re-delivered cells must be unique within the call (one Phase2a per (slot, server) per call)
            _, keep = np.unique(p["slot"].astype(np.int64) * n + p["dst"], return_index=True)
            p = p[np.sort(keep)]
        prev = p[p["slot"] >= w * W]
        assert ora.client_request(req) == (0, -1)
        _, _, orep = ora.phase2a(p)
        st, _, oc = ora.proxyleader_phase2b(b)
        assert st == 0 and len(oc) == W
        rep = torch.zeros((len(p), 4), dtype=torch.int32, device=dev)
        ch = torch.zeros((len(b), 2), dtype=torch.int32, device=dev)
        wm = torch.zeros(1, dtype=torch.int32, device=dev)
        d_req, d_p, d_b = _td(req), _td(p), _td(b)
        eng.vm_step_dev(d_req.data_ptr(), len(req), d_p.data_ptr(), len(p), rep.data_ptr(), d_b.data_ptr(), len(b),
                        ch.data_ptr(), wm.data_ptr())
        r = eng.sync()
        assert (r.status, r.n_chosen, r.watermark, int(wm.item())) == (0, W, (w + 1) * W, (w + 1) * W)
        H.same(rep.cpu().numpy().view(P2B).reshape(-1), orep, f"Phase2a replies, window {w}")
        H.same(ch[: r.n_chosen].cpu().numpy().view(CHOSEN).reshape(-1), oc, f"Chosen stream, window {w}")
        tags.append(eng.counters()["vm_tag"])
        lc = np.zeros(W // 2, dtype=P2B)
        lc["acceptor"] = (oc["slot"][: W // 2] + 1) % n
        lc["slot"] = oc["slot"][: W // 2]
        lc["round"] = oc["value_id"][: W // 2]
        ora.learn_chosen(lc)
        eng.vm_learn_chosen(lc)
        tags.append(eng.counters()["vm_tag"])
        log = eng.snapshot_log(w * W, W)
        assert np.array_equal(log[oc["slot"] - w * W], oc["value_id"])
    assert tags == [LAST_TAG - 2, LAST_TAG - 1, LAST_TAG, 1, 2, 3, 4, 5]
    # every server's entries against the oracle's after the wrap: a round-0 Phase2a to each non-owner's cell
    probe = np.array([(sl, 0, 0, s) for s in range(n) for sl in range(0, 4 * W, 97) if sl % n != s], dtype=P2A)
    H.same(eng.vm_phase2a(probe), ora.phase2a(probe)[2], "probe replies")
    eng.close()


def test_vanilla_duplicate_after_the_tag_wrap_is_reported():
    f = 1
    n = 2 * f + 1
    eng, _ = _vanilla(f, 256)
    eng.vm_client_request(np.array([(s, 0, s + 100, s % n) for s in range(30)], dtype=P2A))
    eng.set_counters(vm_tag=LAST_TAG)
    cell = lambda s, r: (s, r, s + 100, (s + 1) % n)
    eng.vm_phase2a(np.array([cell(4, 0)], dtype=P2A))
    assert eng.counters()["vm_tag"] == 1
    with pytest.raises(FpxError) as ei:
        eng.vm_phase2a(np.array([cell(5, 0), cell(4, 1), cell(6, 0), cell(4, 2)], dtype=P2A))
    assert (ei.value.status, ei.value.index) == (-12, 3)
    eng.close()


def test_vanilla_cell_claimed_with_the_same_tag_one_cycle_earlier():
    """A Phase2a to cell C under tag 1; the tag runs through its cycle without touching C (jumped to its last
    value, one real call made there); the next tag-1 call carries one correct Phase2a to C."""
    f = 1
    n = 2 * f + 1
    eng, ora = _vanilla(f, 256)
    req = np.array([(s, 0, s + 100, s % n) for s in range(30)], dtype=P2A)
    eng.vm_client_request(req)
    assert ora.client_request(req) == (0, -1)
    cell = lambda s, r: (s, r, s + 100, (s + 1) % n)
    both = lambda recs: H.same(eng.vm_phase2a(np.array(recs, dtype=P2A)),
                               ora.phase2a(np.array(recs, dtype=P2A))[2], "Phase2a replies")
    assert eng.counters()["vm_tag"] == 1
    both([cell(4, 0)])
    eng.set_counters(vm_tag=LAST_TAG)
    both([cell(9, 0)])
    assert eng.counters()["vm_tag"] == 1
    both([cell(10, 0), cell(4, 1)])
    eng.close()


# --------------------------------------------------------------------------- the aids themselves
def test_counter_aids_reject_values_the_counters_never_take():
    eng = Engine(slot_capacity=64, max_batch=1024, **CFG1)
    for bad in (0, TOP):
        for name in Engine.COUNTERS:
            with pytest.raises(FpxError) as ei:
                eng.set_counters(**{name: bad})
            assert ei.value.status == -1
    assert eng.counters() == {"seq_base": 1, "rseq_base": 1, "rng_seq_base": 1, "vm_tag": 1}
    eng.set_counters(seq_base=LAST_TAG, vm_tag=7)
    assert eng.counters() == {"seq_base": LAST_TAG, "rseq_base": 1, "rng_seq_base": 1, "vm_tag": 7}
    eng.close()
    ep = EpaxosReplica(1, 0, 4, 64)
    for kw in (dict(tag=0), dict(tag=TOP), dict(seq_base=0), dict(seq_base=TOP)):
        with pytest.raises(FpxError) as ei:
            ep.set_counters(**kw)
        assert ei.value.status == -1
    ep.set_counters(tag=LAST_TAG)
    assert ep.counters() == {"tag": LAST_TAG, "seq_base": 1}
    ep.close()
