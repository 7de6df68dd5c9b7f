"""Long-lived engines: fpx_retire_below on all three protocols, over logs ten times longer than slot_capacity,
against the oracle, which keeps everything.  Leader changes push secondary (slot, round) keys through a small
overflow table, lagging Mencius leader groups push noop ranges through the range table, and vanilla Mencius
slides its window with skips and stragglers for retired slots.  Every reply, Nack and Chosen stream, every error
status and index, and the live part of the acceptors and the log equal the oracle's.  Marked gpu."""
import numpy as np
import pytest

import harness as H
from frankenpaxos_b200 import (CHOSEN, MENCIUS, MULTIPAXOS, P2A, P2A_RANGE, P2B, VALUE_NOOP,
                               VANILLA_MENCIUS, VM_REPLY_CHOSEN, VM_REPLY_CHOSEN_RETIRED, VM_SKIP, Engine, FpxError)
from frankenpaxos_b200 import traces as T
from oracle import fpx_oracle_py as O

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True, params=["auto", "exact"])
def tally_path(request, monkeypatch):
    """Every test of this module runs twice: with the tally free to take its row sweep and forced onto the
    exact per-vote path (FPX_TALLY_PATH)."""
    monkeypatch.setenv("FPX_TALLY_PATH", request.param)
    return request.param


def both(eng_call, ora_result):
    """Run the engine call; (status, index) must equal the oracle's."""
    try:
        out = eng_call()
        est, eidx = 0, -1
    except FpxError as e:
        out, est, eidx = None, e.status, e.index
    assert (est, eidx) == (ora_result[0], ora_result[1]), f"engine {(est, eidx)} oracle {tuple(ora_result[:2])}"
    return out


def mp_oracle(cfg):
    return O.MultiPaxos(cfg["f"], cfg["num_acceptor_groups"], cfg["acceptors_per_group"], cfg["flexible"],
                        cfg["num_leaders"], cfg["num_replicas"])


SHAPES = {"cfg2": T.config_by_name("cfg2")[0], "grid2x3": T.config_by_name("cfg3")[0], "maj15": H.WIDE_SHAPES["maj15"]}


# --------------------------------------------------------------------------- 1. leader changes
@pytest.mark.parametrize("shards", [1, 3])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_leader_changes_through_a_sliding_window(tally_path, shape, shards):
    """40 windows of 1000 slots through engines of 4096 slots and a 256-entry overflow table (per shard).  In
    window w (round w) a new leader re-arms 50-62 slots that are still open in round w + 1: each such slot puts
    two keys into the table, so more than 4000 keys pass through it.  Stale round-w Phase2as are Nacked, votes
    of both rounds arrive interleaved, and the previous window is retired between the first and the second
    half of those votes, so the live keys must survive the table's rebuild and complete afterwards.  Every
    third window also carries stragglers of a retired window: arms of both rounds, Phase2as and votes for
    retired secondary keys.  One oracle per shard (each shard's acceptors see that shard's slots only)."""
    cfg = SHAPES[shape]
    cap, step, total = 4096, 1000, 40000
    g = T.rng(4100 + 7 * shards + len(shape))
    engs = [Engine(slot_capacity=cap, max_batch=1 << 14, overflow_capacity=1 << 8, shard_index=s, shard_count=shards,
                   **cfg) for s in range(shards)]
    oras = [mp_oracle(cfg) for _ in range(shards)]
    mine = lambda recs, s: recs[recs["slot"] % shards == s]
    grid = (cfg["f"], cfg["num_acceptor_groups"], cfg["acceptors_per_group"], cfg["flexible"])
    old = {}
    n_keys = n_nack = 0
    for w in range(total // step):
        r = w
        slots = np.arange(w * step, (w + 1) * step, dtype=np.int32)
        a = T.arms(slots, r, slots * 4 + (r & 3))
        p = T.phase2as(g, slots, *grid, r, a["value_id"])
        ob_all = T.votes_of(p)
        opened = np.sort(g.choice(slots, size=int(g.integers(50, 63)), replace=False)).astype(np.int32)
        is_open = np.isin(ob_all["slot"], opened)
        # one round-w vote per open slot now (never a quorum), the rest of them after the leader change
        rest_of_open = is_open & ~np.isin(np.arange(len(ob_all)), np.unique(ob_all["slot"], return_index=True)[1])
        held = ob_all[rest_of_open]
        early = T.shuffled(g, ob_all[~rest_of_open])
        a2 = T.arms(opened, r + 1, opened * 4 + ((r + 1) & 3))
        p2 = T.phase2as(g, opened, *grid, r + 1, a2["value_id"])
        stale = p[g.integers(0, len(p), size=30)]
        p2 = np.concatenate([p2, stale])[g.permutation(len(p2) + 30)]
        n_keys += 2 * len(opened)
        strag = old.get(w - 3) if w % 3 == 0 else None
        for s, (e, o) in enumerate(zip(engs, oras)):
            H.arm(e, o, mine(a, s))
            H.phase2a(e, o, T.shuffled(g, mine(p, s)))
            st, c1 = H.phase2b(e, o, mine(early, s))
            assert st == 0
            H.arm(e, o, mine(a2, s))                                   # the new leader's Phase2as (leader change)
            ob2, on2 = H.phase2a(e, o, mine(p2, s))
            n_nack += len(on2)
            late = T.shuffled(g, np.concatenate([mine(held, s), ob2]))
            half = len(late) // 2
            st, c2 = H.phase2b(e, o, late[:half])
            if w >= 1:
                e.retire_below(w * step)                               # the previous window goes, this one stays
            if strag is not None:                                      # stragglers of a window retired long ago
                sa, sa2, sp, sb = strag
                H.arm(e, o, mine(np.concatenate([sa[:20], sa2[:20]]), s))
                H.phase2a(e, o, mine(sp[:30], s))
                late = np.concatenate([late, mine(sb, s)])
            st, c3 = H.phase2b(e, o, late[half:])
            chosen = np.concatenate([c1, c2, c3])
            o.replica_chosen(chosen)
            e.replica_chosen(chosen)
            assert e.chosen_watermark() >= (w + 1) * step, (w, s)
        old[w] = (a, a2, p, T.votes_of(p2))
        old.pop(w - 4, None)
    assert n_keys > 4000 and n_nack > 0
    lo = total - step                                                  # the live part
    for e, o in zip(engs, oras):
        H.compare_acceptors(e, o, cfg, lo, step)
        H.compare_log(e, o, lo, step)
    if shards == 1:
        assert oras[0].executed_watermark() == total
    [e.close() for e in engs]


# --------------------------------------------------------------------------- 2. Mencius noop ranges
def mencius_plan(g, LG, total):
    """Per leader group, its slots of [0, total) cut into alternating runs of single-slot Phase2as and noop ranges
    (a range ends anywhere before the group's next slot).  Returns [(start_slot, kind, payload)] sorted by
    start: kind 0 = single slots (array), kind 1 = (start, end)."""
    items = []
    for lg in range(LG):
        s = lg
        single = bool(g.integers(0, 2))
        while s < total:
            k = int(g.integers(1, 9))
            run = s + LG * np.arange(k)
            run = run[run < total]
            if single:
                items.append((int(run[0]), 0, run.astype(np.int32)))
            else:
                items.append((int(run[0]), 1, (int(run[0]), int(min(total, run[-1] + 1 + int(g.integers(0, LG)))))))
            s = int(run[-1]) + LG
            single = not single
    items.sort(key=lambda x: x[0])
    return items


@pytest.mark.parametrize("LG,AG", [(2, 1), (3, 2)])
def test_mencius_ranges_through_a_sliding_window(tally_path, LG, AG):
    """A log ten times slot_capacity where every leader group closes half of its slots with Phase2aNoopRanges:
    more than 2000 ranges pass through the 1024-entry range table.  Ranges cross the window boundaries, so some
    straddle the retire point and keep their key.  After each retire, late arms and late votes of ranges of a
    retired window are ignored, as the oracle ignores them on a Done key."""
    f, per = 1, 3
    cap, step, total = 4096, 1024, 40960
    g = T.rng(5200 + LG * 10 + AG)
    eng = Engine(f, AG, per, num_leaders=2, num_replicas=2, slot_capacity=cap, max_batch=1 << 15,
                 overflow_capacity=1 << 8, protocol=MENCIUS, num_leader_groups=LG)
    ora = O.MultiPaxos(f, AG, per, False, 2, 2, mencius_leader_groups=LG)
    cfg = dict(num_acceptor_groups=LG * AG, acceptors_per_group=per)
    grp = lambda sl: (sl % LG) * AG + (sl // LG) % AG
    items = mencius_plan(g, LG, total)
    n_ranges = 0
    base = 0
    old = {}
    for w in range(total // step):
        lim = base + cap                                               # the engine's live window ends here
        its = [it for it in items if w * step <= it[0] < (w + 1) * step]
        singles = np.concatenate([it[2] for it in its if it[1] == 0] or [np.zeros(0, np.int32)]).astype(np.int32)
        ranges = [it[2] for it in its if it[1] == 1]
        n_ranges += len(ranges)
        # single slots: arm, acceptors (f+1 of the slot's group), votes
        H.arm(eng, ora, T.arms(singles, 0, singles * 4))
        q = np.zeros(len(singles) * (f + 1), dtype=P2A)
        acc = np.argsort(g.random((len(singles), per)), axis=1)[:, : f + 1].astype(np.int32)
        q["slot"] = np.repeat(singles, f + 1); q["round"] = 0; q["value_id"] = np.repeat(singles * 4, f + 1)
        q["dst"] = (np.repeat(grp(singles), f + 1) << 16) | acc.reshape(-1)
        ob, _ = H.phase2a(eng, ora, q[g.permutation(len(q))])
        st, oc = H.phase2b(eng, ora, ob[g.permutation(len(ob))])
        assert st == 0
        # ranges: arm, every acceptor group of the leader group votes with f+1 acceptors
        arm = np.array([(s, e, 0, -1) for (s, e) in ranges], dtype=P2A_RANGE)
        both(lambda: eng.mencius_arm_range(arm), ora.arm_range(arm, lim))
        recs = [(s, e, 0, (((s % LG) * AG + ag) << 16) | int(x)) for (s, e) in ranges for ag in range(AG)
                for x in g.permutation(per)[: f + 1]]
        recs = np.array([recs[i] for i in g.permutation(len(recs))], dtype=P2A_RANGE)
        st, err, rb, rn = ora.acceptor_noop_range(recs, lim)
        out = both(lambda: eng.mencius_acceptor_noop_range(recs), (st, err))
        H.same(out[0], rb, "Phase2bNoopRange stream"); H.same(out[1], rn, "range Nack stream")
        strag = old.get(w - 2)
        votes = rb[g.permutation(len(rb))]
        if strag is not None:                                          # late votes of retired ranges, mixed in
            votes = np.concatenate([strag[1][:40], votes])
        st, err, rc = ora.range_phase2b(votes)
        ec = both(lambda: eng.mencius_range_phase2b(votes), (st, err))
        H.same(ec, rc, "ChosenNoopRange stream")
        ora.replica_chosen(oc); eng.replica_chosen(oc)
        both(lambda: eng.mencius_replica_chosen_range(rc), ora.replica_chosen_range(rc, lim))
        assert eng.chosen_watermark() == ora.first_hole()
        if strag is not None:                                          # late arms of retired ranges
            late = strag[0][:40]
            both(lambda: eng.mencius_arm_range(late), ora.arm_range(late, lim))
        old[w] = (arm, rb)
        if w >= 1:
            base = (w - 1) * step + step // 2 if w % 2 else w * step   # retire points off and on window bounds
            base = min(base, eng.chosen_watermark())
            eng.retire_below(base)
            lim = base + cap
    assert n_ranges > 2000
    lo = total - step
    H.compare_acceptors(eng, ora, cfg, lo, step)
    H.compare_log(eng, ora, lo, step)
    eng.close()


# --------------------------------------------------------------------------- 3. vanilla Mencius
def vm_logs(eng, ora, n, lo, hi, keep):
    """Every server's log over [lo, hi) at the slots `keep` selects: ChosenEntry positions and values,
    pending rounds, vacancies."""
    for s in range(n):
        k, r, v = ora.snapshot(s, lo, hi - lo)
        _, _, vr, vv = eng.snapshot_acceptor(0, s, lo, hi - lo)
        k, r, v, vr, vv = k[keep], r[keep], v[keep], vr[keep], vv[keep]
        chosen = vr == 0x7fffffff
        assert np.array_equal(chosen, k == 3), f"server {s}: ChosenEntry positions"
        assert np.array_equal(vv[chosen], v[chosen]), f"server {s}: chosen values"
        pend = k == 2
        assert np.array_equal(vr[pend], r[pend]) and (vr[k == 0] == -1).all(), f"server {s}: pending entries"


@pytest.mark.parametrize("shards", [1, 2])
@pytest.mark.parametrize("f", [1, 3])
def test_vanilla_mencius_through_a_sliding_window(tally_path, f, shards):
    """n = 2f+1 servers (f = 3 is cfg5's 7), a log ten times slot_capacity, retired as it goes.  Even windows
    run through fpx_vm_step_dev, odd ones through the host calls.  In every window one server skips a run of
    its slots that crosses into the next window (own = 1 at the server, own = 0 at the others).  From the
    fourth window on, stragglers for retired slots arrive: Phase2as (kind 3 where the oracle answers Chosen,
    kind 2), Phase2bs, learn_chosen, own = 0 skips that straddle the retire point, own = 1 skips and client
    requests, with the oracle's statuses and indices."""
    import torch
    n = 2 * f + 1
    W, cap, total = 512, 2048, 20480
    K = 3 * n                                                          # skipped run: 2K slots around a boundary
    g = T.rng(6300 + 10 * f + shards)
    engs = [Engine(f, 1, n, num_leaders=f + 1, num_replicas=f + 1, slot_capacity=cap, max_batch=1 << 15,
                   protocol=VANILLA_MENCIUS, shard_index=s, shard_count=shards) for s in range(shards)]
    oras = [O.VanillaMencius(f) for _ in range(shards)]
    mine = lambda recs, s, key="slot": recs[recs[key] % shards == s]
    dev = torch.device("cuda", 0)
    td = lambda x: torch.from_numpy(np.ascontiguousarray(x).view(np.int32).reshape(len(x), -1).copy()).to(dev)
    skipped = {}                                                       # window -> (server, start, stop)
    hist = {}
    n_kind3 = 0                                                        # kind 3 replies checked
    for w in range(total // W):
        s0 = w % n
        lo_, hi_ = (w + 1) * W - K, (w + 1) * W + K
        start = lo_ + (s0 - lo_) % n
        skipped[w] = (s0, start, hi_)
        req, p, b = T.vanilla_cfg5(6400 + w, f, W, slot_offset=w * W)
        out_ = np.zeros(len(req), dtype=bool)
        for (sv, a_, z_) in (skipped[w], skipped.get(w - 1, (0, 0, 0))):
            out_ |= (req["slot"] >= a_) & (req["slot"] < z_) & (req["slot"] % n == sv)
        gone = req["slot"][out_]
        req = req[~out_]; p = p[~np.isin(p["slot"], gone)]; b = b[~np.isin(b["slot"], gone)]
        sk = [(s0, start, hi_, 1)] + [(o, start, hi_, 0) for o in range(n) if o != s0]
        sk = np.array(sk, dtype=VM_SKIP)[g.permutation(n)]
        noop = np.arange(start, hi_, n, dtype=np.int32)
        strag = hist.get(w - 3)
        for s, (e, o) in enumerate(zip(engs, oras)):
            rq, pp, bb = mine(req, s), mine(p, s), mine(b, s)
            if strag is not None:
                bb = np.concatenate([mine(strag[2], s)[:50], bb])      # Phase2bs for retired slots: ignored
            assert o.client_request(rq) == (0, -1)
            _, _, orep = o.phase2a(pp)
            st, _, oc = o.phase2b(bb)
            assert st == 0
            if w % 2 == 0:
                d_req, d_p, d_b = td(rq), td(pp), td(bb)
                rep = torch.zeros((max(len(pp), 1), 4), dtype=torch.int32, device=dev)
                ch = torch.zeros((max(len(bb), 1), 2), dtype=torch.int32, device=dev)
                wm = torch.zeros(1, dtype=torch.int32, device=dev)
                e.vm_step_dev(d_req.data_ptr(), len(rq), d_p.data_ptr(), len(pp), rep.data_ptr(), d_b.data_ptr(), len(bb),
                              ch.data_ptr(), wm.data_ptr())
                r = e.sync()
                assert r.status == 0
                erep = rep[: len(pp)].cpu().numpy().view(P2B).reshape(-1)
                ec = ch[: r.n_chosen].cpu().numpy().view(CHOSEN).reshape(-1)
            else:
                e.vm_client_request(rq)
                erep = e.vm_phase2a(pp)
                ec = e.proxyleader_phase2b(bb)
                e.replica_chosen(ec)
            H.same(erep, orep, f"Phase2a replies, window {w}")
            H.same(ec, oc, f"Chosen stream, window {w}")
            both(lambda: e.vm_skip(sk), o.skip(sk, max(0, (w - 2) * W) + cap))   # capacity: base + slot_capacity
            nm = mine(np.array([(x, VALUE_NOOP) for x in noop], dtype=CHOSEN), s)
            e.replica_chosen(nm)                                       # the shared log learns the skipped slots
            # some other servers learn some chosen slots
            lc = np.zeros(len(oc), dtype=P2B)
            lc["acceptor"] = (oc["slot"] + 1 + g.integers(0, n - 1, size=len(oc))) % n
            lc["slot"] = oc["slot"]; lc["round"] = oc["value_id"]
            lc = lc[g.random(len(lc)) < 0.3]
            e.vm_learn_chosen(lc); o.learn_chosen(lc)
            assert e.chosen_watermark() >= (w + 1) * W, (w, s)
            if strag is not None:
                n_kind3 += stragglers(e, o, g, strag, s, shards, n, w, W)
        hist[w] = (req, p, b, sk)
        hist.pop(w - 4, None)
        if w >= 1:
            for e in engs:
                e.retire_below((w - 1) * W)
    assert n_kind3 > 0
    lo = total - W
    for s, (e, o) in enumerate(zip(engs, oras)):
        keep = (np.arange(lo, total) % shards) == s
        vm_logs(e, o, n, lo, total, keep)
    with pytest.raises(FpxError) as ei:                                # beyond the window: base + capacity
        engs[0].vm_phase2a(np.array([(total + 2 * cap * shards, 0, 1, 1)], dtype=P2A))
    assert ei.value.status == -6
    [e.close() for e in engs]


def stragglers(e, o, g, strag, s, shards, n, w, W):
    """Messages for slots of window w - 3, which was retired two windows ago."""
    req, p, b, sk = strag
    mine = lambda recs, key="slot": recs[recs[key] % shards == s]
    # Phase2a where the oracle's entry is a ChosenEntry: kind 3 for its kind 2, the rest of the reply equal
    pp = mine(p)[:200]
    kinds = np.array([o.snapshot(int(x["dst"]), int(x["slot"]), 1)[0][0] for x in pp], dtype=np.int32)
    pp = pp[kinds == 3]
    _, _, orep = o.phase2a(pp)
    erep = e.vm_phase2a(pp)
    assert (orep["group"] == VM_REPLY_CHOSEN).all()
    exp = orep.copy()
    exp["group"] = VM_REPLY_CHOSEN_RETIRED
    exp["round"] = 0
    H.same(erep, exp, "Phase2a for retired slots")
    # learn_chosen for retired slots: ignored
    lc = np.zeros(20, dtype=P2B)
    lc["slot"] = mine(req)["slot"][:20] if len(mine(req)) >= 20 else 0
    lc["acceptor"] = g.integers(0, n, size=20); lc["round"] = 5
    lc = lc[lc["slot"] % shards == s]
    e.vm_learn_chosen(lc); o.learn_chosen(lc)
    # own = 0 skips (handleSkip) again, one of them straddling the retire point (w - 2) * W; own = 1: not vacant
    s0, start, stop = int(sk[sk["own"] == 1][0]["server"]), int(sk[0]["slot_start"]), int(sk[0]["slot_stop"])
    a_ = (w - 2) * W - 2 * n
    a_ += (s0 - a_) % n
    again = np.array([(o2, a_, a_ + 4 * n, 0) for o2 in range(n) if o2 != s0][:2], dtype=VM_SKIP)
    cap_ = 1 << 30
    both(lambda: e.vm_skip(again), o.skip(again, cap_))
    own = np.array([(s0, start, stop, 1)], dtype=VM_SKIP)
    r = o.skip(own, cap_)
    assert r[0] == -14
    both(lambda: e.vm_skip(own), r)
    # client requests for retired slots: dropped; one with a foreign coordinator: BAD_ACCEPTOR at its index
    rq = mine(req)[:10].copy()
    bad = rq.copy()
    if len(bad):
        bad["dst"][-1] = (bad["dst"][-1] + 1) % n
    both(lambda: e.vm_client_request(rq), o.client_request(rq))
    both(lambda: e.vm_client_request(bad), o.client_request(bad))
    # Phase2b for retired slots in a batch of its own
    bb = mine(b)[:30]
    st, _, oc = o.phase2b(bb)
    assert st == 0 and len(oc) == 0
    assert len(e.proxyleader_phase2b(bb)) == 0
    return len(pp)


# --------------------------------------------------------------------------- 4. steady state
def test_retire_launches_nothing_extra_in_the_steady_state(tally_path):
    """With no secondary key and no range ever armed, a retire is exactly one kernel launch, on all three
    protocols.  A leader change (or a noop range) makes the next retire rebuild its table: one more launch.
    Once the table is empty again, retiring is back to one launch."""
    cfg = SHAPES["cfg2"]
    for proto in (MULTIPAXOS, MENCIUS, VANILLA_MENCIUS):
        kw = dict(num_leader_groups=2) if proto == MENCIUS else {}
        if proto == VANILLA_MENCIUS:
            e = Engine(1, 1, 3, num_leaders=2, num_replicas=2, slot_capacity=4096, max_batch=1 << 14,
                       overflow_capacity=1 << 8, protocol=proto)
        else:
            e = Engine(slot_capacity=4096, max_batch=1 << 14, overflow_capacity=1 << 8, protocol=proto, **cfg, **kw)

        def window(k, leader_change=False, noop_range=False):
            sl = np.arange(k * 1000, (k + 1) * 1000, dtype=np.int32)
            if proto == VANILLA_MENCIUS:
                req, p, b = T.vanilla_cfg5(k, 1, 1000, slot_offset=k * 1000)
                e.vm_client_request(req); e.vm_phase2a(p)
                e.replica_chosen(e.proxyleader_phase2b(b))
                assert e.chosen_watermark() == (k + 1) * 1000         # publishes the watermark retire checks
                return
            grp_of = (lambda x: ((x % 2) << 16)) if proto == MENCIUS else (lambda x: 0)
            e.proxyleader_arm(T.arms(sl, 0))
            q = T.phase2as(T.rng(k), sl, 2, 1, 5, False, 0)
            q["dst"] |= grp_of(q["slot"])
            b, _ = e.acceptor_phase2a(q)
            if leader_change:
                e.proxyleader_arm(T.arms(sl[:10], 1, sl[:10] + 7))
            if noop_range:
                e.mencius_arm_range(np.array([(int(sl[0]) + 1000, int(sl[0]) + 1005, 0, -1)], dtype=P2A_RANGE))
            e.replica_chosen(e.proxyleader_phase2b(b))
            assert e.chosen_watermark() == (k + 1) * 1000

        def retire(k):
            c0 = e.launch_count
            e.retire_below(k * 1000)
            return e.launch_count - c0

        window(0); window(1)
        assert retire(1) == 1, proto
        if proto == VANILLA_MENCIUS:
            window(2)
            assert retire(2) == 1
        else:
            window(2, leader_change=True)
            assert retire(2) == 2, proto                               # window 2's keys are live: rebuilt, kept
            window(3)
            assert retire(3) == 2, proto                               # window 2's keys leave the table
            window(4)
            assert retire(4) == 1, proto                               # the table is empty again
        if proto == MENCIUS:
            window(5, noop_range=True)
            assert retire(5) == 2                                      # the range table holds [6000, 6005)
            window(6)
            assert retire(7) == 2                                      # ... until the range is retired
            assert retire(7) == 0                                      # nothing more to slide
        e.close()
