"""Wide quorum systems against the CPU oracle, bit for bit.  A proxy-leader row is {round, value, one stamp per
voter} padded to 8, 16 or 32 words (at most 6, 14 or 30 voters per slot), and the tally kernel is instantiated
once per row size; the acceptor kernel scans up to 32 acceptors, one per lane.  These cases reach the 16- and
32-word rows and up to 30 acceptors in ways the shape-parametrized tests elsewhere cannot: the row sweep at
every width, quorums decided by the far 32-byte sectors of a row alone, a hidden vote in a far sector, the
predicate kernel on wide masks, compartmentalized Mencius with 28 acceptors, the fused step, the slot ring and
the sweep's second emission pass on 32-word rows.  Marked gpu: needs an H100."""
import numpy as np
import pytest

import harness as H
from frankenpaxos_b200 import CHOSEN, MENCIUS, P2A, P2A_RANGE, P2B, Engine, FpxError
from frankenpaxos_b200 import traces as T
from oracle import fpx_oracle_py as O

pytestmark = pytest.mark.gpu

W = H.WIDE_SHAPES


@pytest.fixture(params=["auto", "exact"])
def tally_path(request, monkeypatch):
    """The test runs twice: with the tally free to take its row sweep and forced onto the exact per-vote
    path (FPX_TALLY_PATH, read when the engine is created)."""
    monkeypatch.setenv("FPX_TALLY_PATH", request.param)
    return request.param


def td(x):
    import torch
    return torch.from_numpy(x.view(np.int32).reshape(len(x), -1).copy()).to(torch.device("cuda", 0))


# --------------------------------------------------------------------------- the sweep at every width
@pytest.mark.parametrize("shape", list(W))
def test_sweep_at_every_width(tally_path, shape):
    """maj7, grid2x7 (16-word rows); maj15, groups2x15, maj29, grid5x6 (32-word rows): a steady-state
    one-round window, its votes shuffled and delivered in five batches, so that earlier batches' stamps decide
    completions.  In auto mode every batch takes the row sweep: a wide-row sweep that flagged an anomaly
    and fell back to the exact path would fail here."""
    cfg = W[shape]
    n_slots = 6000
    want = "sweep" if tally_path == "auto" else "exact"
    eng, ora = H.make_pair(cfg, n_slots, max_batch=1 << 17)
    a, p, b = T.workload(31 + len(shape), cfg, n_slots)
    H.arm(eng, ora, a)
    H.phase2a(eng, ora, p)
    total = 0
    for chunk in np.array_split(b, 5):
        st, c = H.phase2b(eng, ora, chunk)
        assert st == 0 and eng.last_tally_path == want
        total += len(c)
        H.replica(eng, ora, c)
    assert total == n_slots
    # duplicates of old votes only: nothing new is chosen, still the same path
    st, c = H.phase2b(eng, ora, b[:700])
    assert st == 0 and len(c) == 0 and eng.last_tally_path == want
    H.compare_log(eng, ora, 0, n_slots)
    eng.close()


# --------------------------------------------------------------------------- quorums from the far sectors only
def _order(b, order):
    if order == "by_slot":
        return b[np.argsort(b["slot"], kind="stable")]
    if order == "reversed":
        return b[np.argsort(b["slot"], kind="stable")][::-1].copy()
    return b[np.lexsort((b["slot"], b["group"] * 64 + b["acceptor"]))]        # one acceptor after another


@pytest.mark.parametrize("order", ["by_slot", "reversed", "by_acceptor"])
@pytest.mark.parametrize("shape", ["maj15", "maj29", "grid5x6"])
def test_quorum_from_the_far_sectors_only(tally_path, shape, order):
    """32-word rows; voter v's stamp is word 2 + v, so voters 0-5 live in the row's first 32-byte sector.
    maj15 (quorum 8) and maj29 (quorum 15): every slot's Phase2as go to f+1 voters drawn from voters 6 and
    up only, so a key is completed by stamps in the second to fourth sectors alone.  grid5x6: row 0 of the
    grid (voters 0-5) is the first sector; its vote is delivered first, so the completing vote always comes
    from rows 1-4.  Votes by slot, reversed, or one acceptor after another."""
    cfg = W[shape]
    n_slots = 8000
    g = T.rng(50 + len(shape))
    eng, ora = H.make_pair(cfg, n_slots, max_batch=1 << 18)
    slots = np.arange(n_slots, dtype=np.int32)
    a = T.arms(slots, 0, slots * 3 + 1)
    if cfg["flexible"]:
        p = T.phase2as(g, slots, cfg["f"], cfg["num_acceptor_groups"], cfg["acceptors_per_group"], True, 0,
                       slots * 3 + 1)
    else:
        A, q = cfg["acceptors_per_group"], cfg["f"] + 1
        acc = 6 + np.argsort(g.random((n_slots, A - 6)), axis=1)[:, :q].astype(np.int32)
        p = np.zeros(n_slots * q, dtype=P2A)
        p["slot"] = np.repeat(slots, q); p["value_id"] = np.repeat(slots * 3 + 1, q); p["dst"] = acc.reshape(-1)
    H.arm(eng, ora, a)
    ob, _ = H.phase2a(eng, ora, p[g.permutation(len(p))])
    b = _order(ob[g.permutation(len(ob))], order)
    if cfg["flexible"]:
        b = b[np.argsort(b["group"] != 0, kind="stable")]          # row 0's votes first
    else:
        assert (b["acceptor"] >= 6).all()
    st, c = H.phase2b(eng, ora, b)
    assert st == 0 and len(c) == n_slots
    if tally_path == "auto":
        assert eng.last_tally_path == "sweep"
    H.replica(eng, ora, c)
    H.compare_log(eng, ora, 0, n_slots)
    eng.close()


# --------------------------------------------------------------------------- a hidden vote in a far sector
def test_hidden_vote_in_a_far_sector_goes_to_the_exact_path(tally_path):
    """maj29, 32-word rows.  Window 0 is chosen in round 0 with voter 20 (stamp word 22, the third sector) in
    every slot's quorum; window 1 is armed in round 1.  A batch of round-1 votes for window 1 carries, in its
    middle, a round-1 vote of voter 20 for a window-0 slot: blind stamping keeps voter 20's older stamp, so
    only the row's round word shows the vote has no key.  The batch must take the exact path and report
    FPX_ERR_UNKNOWN_SLOT_ROUND at the oracle's index."""
    cfg = W["maj29"]
    n, A, q = 2000, cfg["acceptors_per_group"], cfg["f"] + 1
    g = T.rng(77)
    eng, ora = H.make_pair(cfg, 2 * n, max_batch=1 << 17)

    def p2as(slots, rnd):
        others = np.array([v for v in range(A) if v != 20])
        acc = np.concatenate([np.full((len(slots), 1), 20), others[np.argsort(g.random((len(slots), A - 1)), axis=1)[:, :q - 1]]], axis=1)
        p = np.zeros(len(slots) * q, dtype=P2A)
        p["slot"] = np.repeat(slots, q); p["round"] = rnd; p["value_id"] = np.repeat(slots * 2 + rnd, q)
        p["dst"] = acc.reshape(-1)
        return p[g.permutation(len(p))]
    s0 = np.arange(n, dtype=np.int32)
    s1 = s0 + n
    H.arm(eng, ora, T.arms(s0, 0, s0 * 2))
    ob, _ = H.phase2a(eng, ora, p2as(s0, 0))
    st, c = H.phase2b(eng, ora, ob[g.permutation(len(ob))])
    assert st == 0 and len(c) == n
    H.replica(eng, ora, c)
    H.arm(eng, ora, T.arms(s1, 1, s1 * 2 + 1))
    ob1, _ = H.phase2a(eng, ora, p2as(s1, 1))
    v = ob1[g.permutation(len(ob1))]
    hidden = np.array([(0, 20, n - 1, 1)], dtype=P2B)
    k = len(v) // 2
    st, _ = H.phase2b(eng, ora, np.concatenate([v[:k], hidden, v[k:]]))
    assert st == -4 and eng.last_tally_path == "exact"
    eng.close()


# --------------------------------------------------------------------------- quorum predicates
@pytest.mark.parametrize("shape", ["grid2x7", "grid5x6", "maj15", "maj29"])
def test_quorum_predicates_on_wide_masks(shape):
    """fpx_quorum_eval against the oracle's Grid / SimpleMajority with the same members.  grid2x7: 14
    members (2 rows of 7); grid5x6: 30 members (5 rows of 6); maj15 and maj29: 15 and 29 members.  A few
    thousand random masks of every density, whole grid rows, and masks with a foreign bit at and above the
    member count (bits up to 31)."""
    cfg = W[shape]
    G, A, flexible = cfg["num_acceptor_groups"], cfg["acceptors_per_group"], cfg["flexible"]
    members = G * A if flexible else A
    g = T.rng(400 + members)
    n = 3000
    dens = g.random(n)[:, None]
    bits = g.random((n, members)) < dens
    masks = (bits.astype(np.uint64) << np.arange(members, dtype=np.uint64)).sum(axis=1).astype(np.uint32)
    extra = []
    if flexible:
        row = (1 << A) - 1
        extra += [row << (r * A) for r in range(G)]                          # exactly one row: a read quorum
        extra += [sum(1 << (r * A + int(g.integers(0, A))) for r in range(G)) for _ in range(50)]   # one per row
    extra += [(1 << members) - 1, 0, 1 << (members - 1)]
    extra = np.array(extra, dtype=np.uint32)
    foreign = masks[:400] | (np.uint32(1) << g.integers(members, 32, size=400).astype(np.uint32))
    edge = np.array([(1 << members) - 1 | (1 << b) for b in range(members, 32)], dtype=np.uint32)
    masks = np.concatenate([masks, extra, foreign, edge])
    ids = list(range(members))
    ora_members = [ids[r * A:(r + 1) * A] for r in range(G)] if flexible else ids
    kind = "grid" if flexible else "simple_majority"
    eng = Engine(slot_capacity=8, max_batch=1024, **cfg)
    for which in range(4):
        got = eng.quorum_eval(which, masks)
        for m, r in zip(masks.tolist(), got.tolist()):
            xs = [b if b < members else 1000 + b for b in range(32) if (m >> b) & 1]
            want = O.quorum_eval(kind, ora_members, which, xs)
            assert r == want, (shape, which, hex(m), r, want)
    eng.close()


# --------------------------------------------------------------------------- compartmentalized Mencius, 28 acceptors
MEN_F, MEN_LG, MEN_AG, MEN_PER = 3, 2, 2, 7


def _mencius_pair(cap):
    eng = Engine(MEN_F, MEN_AG, MEN_PER, num_leaders=MEN_F + 1, num_replicas=MEN_F + 1, slot_capacity=cap,
                 max_batch=1 << 17, protocol=MENCIUS, num_leader_groups=MEN_LG)
    ora = O.MultiPaxos(MEN_F, MEN_AG, MEN_PER, False, MEN_F + 1, MEN_F + 1, mencius_leader_groups=MEN_LG)
    return eng, ora


def test_mencius_with_28_acceptors(tally_path):
    """mencius2x2x7: 2 leader groups x 2 acceptor groups x 7 acceptors = 28 acceptors, f = 3, 7 voters per
    slot (16-word rows).  Slot s -> leader group s % 2, acceptor group (s / 2) % 2; arm, a round bump on every
    7th slot, Phase2as in three chunks with Nacks, shuffled votes in four batches, replica log."""
    f, LG, AG, per = MEN_F, MEN_LG, MEN_AG, MEN_PER
    n_slots = 5000
    g = T.rng(170)
    eng, ora = _mencius_pair(n_slots)
    slots = np.arange(n_slots, dtype=np.int32)
    grp = (slots % LG) * AG + (slots // LG) % AG

    def p2as(sl, rnd, thrifty=True):
        q = f + 1 if thrifty else per
        acc = np.argsort(g.random((len(sl), per)), axis=1)[:, :q].astype(np.int32)
        out = np.zeros(len(sl) * q, dtype=P2A)
        out["slot"] = np.repeat(sl, q); out["round"] = rnd; out["value_id"] = np.repeat(sl, q) * 4 + rnd
        out["dst"] = (np.repeat(grp[sl], q) << 16) | acc.reshape(-1)
        return out
    H.arm(eng, ora, T.arms(slots, 0, slots * 4))
    bump = slots[::7]
    H.arm(eng, ora, T.arms(bump, 1, bump * 4 + 1))
    mix = np.concatenate([p2as(slots, 0), p2as(bump, 1, thrifty=False)])
    mix = mix[g.permutation(len(mix))]
    votes = []
    n_nack = 0
    for chunk in np.array_split(mix, 3):
        ob, on = H.phase2a(eng, ora, chunk)
        votes.append(ob)
        n_nack += len(on)
    assert n_nack > 0
    cfg = dict(num_acceptor_groups=LG * AG, acceptors_per_group=per)
    H.compare_acceptors(eng, ora, cfg, 0, n_slots)
    v = np.concatenate(votes)
    v = v[g.permutation(len(v))]
    for chunk in np.array_split(v, 4):
        st, c = H.phase2b(eng, ora, chunk)
        assert st == 0
        H.replica(eng, ora, c)
    H.compare_log(eng, ora, 0, n_slots)
    with pytest.raises(FpxError) as ei:           # a Phase2a delivered to the wrong acceptor group
        eng.acceptor_phase2a(np.array([(0, 0, 0, (3 << 16) | 0)], dtype=P2A))
    assert ei.value.status == -5
    eng.close()


def test_mencius_noop_range_with_14_stamps():
    """mencius2x2x7: a Phase2aNoopRange's entry keeps one stamp per (acceptor group, acceptor) of its leader
    group, 2 x 7 = 14 stamps; quorum f+1 = 4 in each acceptor group.  Ranges of both leader groups, all 7 or
    only 5 acceptors of each group answering, votes shuffled with duplicates; acceptors and log vs the oracle."""
    from test_ranges_gpu import both, range_round_trip
    f, LG, AG, per = MEN_F, MEN_LG, MEN_AG, MEN_PER
    cap = 6000
    g = T.rng(171)
    eng, ora = _mencius_pair(cap)
    n_chosen = 0
    for ranges, k in (([(0, 1200, 0), (1, 2401, 0)], None), ([(2400, 4000, 1), (2401, 3001, 1)], 5)):
        chosen, on = range_round_trip(eng, ora, g, ranges, cap, LG, AG, per, voters_per_group=k)
        assert len(on) == 0
        n_chosen += len(chosen)
        both(lambda: eng.mencius_replica_chosen_range(chosen), ora.replica_chosen_range(chosen, cap))
        assert eng.chosen_watermark() == ora.first_hole()
    assert n_chosen == 4
    H.compare_acceptors(eng, ora, dict(num_acceptor_groups=LG * AG, acceptors_per_group=per), 0, cap)
    H.compare_log(eng, ora, 0, cap)
    eng.close()


# --------------------------------------------------------------------------- the fused step at 32-word rows
def test_fused_step_on_rebased_windows_with_32_word_rows(tally_path):
    """maj15 (15 voters, 32-word rows): fpx_step_dev -- arm, acceptor, tally with the replica's log put and
    the watermark fused into it -- over three windows of 2^18 slots of one log, windows 1 and 2 above
    committed ones.  Phase2b and Chosen streams, counts, the fused watermark, acceptors and log vs the oracle."""
    import torch
    cfg = W["maj15"]
    Wn, wins = 1 << 18, 3
    q = cfg["f"] + 1
    eng, ora = H.make_pair(cfg, wins * Wn, max_batch=q * Wn, overflow_capacity=1 << 10)
    dev = torch.device("cuda", 0)
    d_p2b = torch.zeros((q * Wn, 4), dtype=torch.int32, device=dev)
    d_nack = torch.zeros((q * Wn, 2), dtype=torch.int32, device=dev)
    d_ch = torch.zeros((q * Wn, 2), dtype=torch.int32, device=dev)
    d_wm = torch.zeros(1, dtype=torch.int32, device=dev)
    for w in range(wins):
        a, p, b = T.workload(90 + w, cfg, Wn, slot0=w * Wn)
        ora.arm(a)
        _, _, ob, on = ora.acceptor_phase2a(p)
        _, _, oc = ora.proxyleader_phase2b(b)
        ora.replica_chosen(oc)
        d_a, d_p, d_b = td(a), td(p), td(b)
        eng.step_dev(d_a.data_ptr(), len(a), d_p.data_ptr(), len(p), d_p2b.data_ptr(), d_nack.data_ptr(),
                     d_b.data_ptr(), len(b), d_ch.data_ptr(), d_wm.data_ptr())
        r = eng.sync()
        assert (r.status, r.n_p2b, r.n_nack, r.n_chosen) == (0, len(ob), 0, len(oc)) and len(oc) == Wn
        assert r.watermark == ora.executed_watermark() == int(d_wm.item()) == (w + 1) * Wn
        H.same(d_p2b[: r.n_p2b].cpu().numpy().view(P2B).reshape(-1), ob, f"Phase2b stream, window {w}")
        H.same(d_ch[: r.n_chosen].cpu().numpy().view(CHOSEN).reshape(-1), oc, f"Chosen stream, window {w}")
    H.compare_acceptors(eng, ora, cfg, (wins - 1) * Wn, Wn)
    H.compare_log(eng, ora, 0, wins * Wn)
    eng.close()


# --------------------------------------------------------------------------- the slot ring at 32-word rows
def test_ring_window_slides_with_32_word_rows(tally_path):
    """maj15 (32-word rows, 15 vote cells per slot) through fpx_retire_below: a log ten times longer than
    slot_capacity, the executed prefix retired as it goes, so recycle_kernel resets 32-word rows and 15 cells
    per slot; late messages for retired slots are ignored.  Streams, log and acceptors vs the oracle."""
    cfg = W["maj15"]
    cap, step, total = 4096, 1000, 40000
    eng = Engine(slot_capacity=cap, max_batch=1 << 15, overflow_capacity=1 << 8, **cfg)
    ora = O.MultiPaxos(cfg["f"], 1, cfg["acceptors_per_group"], False, cfg["num_leaders"], cfg["num_replicas"])
    old = None
    for w in range(total // step):
        a, p, b = T.workload(500 + w, cfg, step, slot0=w * step)
        if old is not None and w % 3 == 0:         # stragglers of a window that is retired by now
            oa, op, ob_ = old
            a, p, b = np.concatenate([oa[:20], a]), np.concatenate([op[:30], p]), np.concatenate([b[:500], ob_[:40], b[500:]])
        ora.arm(a)
        _, _, ob, on = ora.acceptor_phase2a(p)
        _, _, oc = ora.proxyleader_phase2b(b)
        ora.replica_chosen(oc)
        eng.proxyleader_arm(a)
        eb, en = eng.acceptor_phase2a(p)
        assert len(en) == 0
        H.same(eb, ob, f"Phase2b stream, window {w}")
        ec = eng.proxyleader_phase2b(b)
        H.same(ec, oc, f"Chosen stream, window {w}")
        eng.replica_chosen(ec)
        assert eng.chosen_watermark() == (w + 1) * step
        if w >= 2:
            eng.retire_below((w - 1) * step)           # keep the last two windows
            old = T.workload(500 + w - 2, cfg, step, slot0=(w - 2) * step)
    assert ora.executed_watermark() == total
    H.compare_acceptors(eng, ora, cfg, total - step, step)
    H.compare_log(eng, ora, total - step, step)
    eng.close()


# --------------------------------------------------------------------------- the sweep's second emission pass
def test_sweep_emits_in_a_second_pass_when_rows_exceed_shared_memory(tally_path):
    """maj15, 32-word rows.  The sweep keeps a CTA's completed {vote, value} entries in shared memory between
    its phases B and D; when a CTA's share of the window exceeds keep_cap, phase D sweeps the rows again.

    keep_cap = (200 KiB - 4 B per 1024-vote chunk) / 8 B: with 900,000 votes (879 chunks) it is 25,160
    rows.  The window spans 112,500 armed slots 32 apart, 3,599,969 rows; over H100's 132 single-CTA tally
    grid that is 27,273 rows per CTA, rounded up to 27,648 -- above keep_cap.  The sweep runs only when the
    window is at most 4 rows per vote (+ 4096): 900,000 votes = f + 1 = 8 per armed slot allow 3,604,096.
    Which pass emitted cannot be read back; the Chosen stream, its order and the log are checked."""
    cfg = W["maj15"]
    n_armed, gap = 112500, 32
    slots = (np.arange(n_armed, dtype=np.int64) * gap).astype(np.int32)
    cap = int(slots[-1]) + 1
    q = cfg["f"] + 1
    assert n_armed * q == 900000 and cap - 1 <= 4 * n_armed * q + 4096
    g = T.rng(4242)
    eng, ora = H.make_pair(cfg, cap, max_batch=n_armed * q, overflow_capacity=1 << 10)
    a = T.arms(slots, 0, slots // gap + 7)
    p = T.phase2as(g, slots, cfg["f"], 1, cfg["acceptors_per_group"], False, 0, slots // gap + 7)
    b = T.shuffled(g, T.votes_of(p))
    H.arm(eng, ora, a)
    st, c = H.phase2b(eng, ora, b)
    assert st == 0 and len(c) == n_armed
    if tally_path == "auto":
        assert eng.last_tally_path == "sweep"
    H.replica(eng, ora, c)
    H.compare_log(eng, ora, 0, cap)
    eng.close()
