"""A tally call of more votes than one launch takes (10,485,760: the shared-memory scan of the per-chunk
counts) is cut into several cooperative launches (tally_launch, fpx_engine.cu).  The launches of one call
carry state from one to the next: the Chosen stream's append offset, the vote sequence numbers, the
co-located replica's log numbering, the fused watermark (settled by the last launch only, published once
per call) and the largest chosen slot; error indices are call indices.  Engine.set_tally_max_sub cuts
small batches the same way, so every boundary case runs at sizes the oracle answers quickly; the last two
tests run the real split at its default size.  Everything is compared bit for bit with the oracle."""
import functools

import numpy as np
import pytest

import harness as H
from frankenpaxos_b200 import CHOSEN, NACK, P2A, P2B, VANILLA_MENCIUS, Engine, FpxError
from frankenpaxos_b200 import traces as T
from oracle import fpx_oracle_py as O

pytestmark = pytest.mark.gpu

DEFAULT_MAX_SUB = (40 * 1024 // 4) * 1024
CFG1, _ = T.config_by_name("cfg1")
CFG2, _ = T.config_by_name("cfg2")
SHAPES = {
    "cfg1": CFG1,
    "cfg2": CFG2,
    "grid2x3": dict(f=1, num_acceptor_groups=2, acceptors_per_group=3, flexible=True, num_leaders=2, num_replicas=2),
    "maj15": H.WIDE_SHAPES["maj15"],
}
# one vote per launch, less than a warp, one rank chunk exactly, one vote past a chunk, a ragged tail
SUBS = [1, 31, 1024, 1025, 4097]


@pytest.fixture(autouse=True, params=["auto", "exact"])
def tally_path(request, monkeypatch):
    """Every test runs with the tally free to take its row sweep and forced onto the exact per-vote path."""
    monkeypatch.setenv("FPX_TALLY_PATH", request.param)
    return request.param


def launches(n, sub):
    return -(-n // sub)


def _td(x):
    import torch
    return torch.from_numpy(x.view(np.int32).reshape(len(x), -1).copy()).to(torch.device("cuda", 0))


def _ptr(t):
    return t.data_ptr() if t is not None else None


def fused_step(eng, votes, arm=None, p2a=None):
    """fpx_step_dev: acceptor batch, arm batch, then the tally with the co-located replica's log put and the
    watermark fused into it.  Returns (sync result, Phase2b stream, Nack stream, Chosen stream, d_watermark)."""
    import torch
    dev = torch.device("cuda", 0)
    n_arm = 0 if arm is None else len(arm)
    n_p2a = 0 if p2a is None else len(p2a)
    d_a = _td(arm) if n_arm else None
    d_p = _td(p2a) if n_p2a else None
    d_v = _td(votes) if len(votes) else None
    o_b = torch.zeros((max(n_p2a, 1), 4), dtype=torch.int32, device=dev)
    o_n = torch.zeros((max(n_p2a, 1), 2), dtype=torch.int32, device=dev)
    o_c = torch.zeros((max(len(votes), 1), 2), dtype=torch.int32, device=dev)
    d_wm = torch.full((1,), -7, dtype=torch.int32, device=dev)
    eng.step_dev(_ptr(d_a), n_arm, _ptr(d_p), n_p2a, o_b.data_ptr(), o_n.data_ptr(), _ptr(d_v), len(votes),
                 o_c.data_ptr(), d_wm.data_ptr())
    r = eng.sync()
    view = lambda t, k, dt: t[:k].cpu().numpy().view(dt).reshape(-1)
    return r, view(o_b, r.n_p2b, P2B), view(o_n, r.n_nack, NACK), view(o_c, r.n_chosen, CHOSEN), int(d_wm.item())


def oracle_step(ora, votes, arm=None, p2a=None):
    ob = on = None
    if arm is not None:
        assert ora.arm(arm) == (0, -1)
    if p2a is not None:
        st, _, ob, on = ora.acceptor_phase2a(p2a)
        assert st == 0
    st, idx, oc = ora.proxyleader_phase2b(votes)
    assert st == 0, (st, idx)
    ora.replica_chosen(oc)
    return ob, on, oc, ora.executed_watermark()


def tally_and_compare(form, eng, ora, votes, arm=None):
    """One tally call of `votes` (host form: proxyleader_phase2b + replica_chosen; fused: fpx_step_dev with the
    arm batch in the same call), its Chosen stream and watermark against the oracle's."""
    if form == "host":
        if arm is not None:
            H.arm(eng, ora, arm)
        st, c = H.phase2b(eng, ora, votes)
        assert st == 0
        H.replica(eng, ora, c)
        return c
    _, _, oc, wm = oracle_step(ora, votes, arm=arm)
    r, _, _, c, d_wm = fused_step(eng, votes, arm=arm)
    assert (r.status, r.n_chosen) == (0, len(oc))
    H.same(c, oc, "Chosen stream")
    assert r.watermark == d_wm == wm
    return c


def block_votes(cfg, g, slots, round_=0, values=None, thrifty=True):
    return T.votes_of(T.phase2as(g, slots, cfg["f"], cfg["num_acceptor_groups"], cfg["acceptors_per_group"],
                                 cfg["flexible"], round_, values, thrifty=thrifty))


# --------------------------------------------------------------------------- 1. adversarial traces
@pytest.mark.parametrize("sub", SUBS)
@pytest.mark.parametrize("shape", list(SHAPES))
def test_adversarial_traces_over_many_launches(shape, sub):
    """Stale and fresh rounds, duplicates, late votes, several live rounds per slot (rows poisoned, keys in
    the overflow table), non-thrifty fan-out; every tally call cut into launches of `sub` votes."""
    cfg = SHAPES[shape]
    wide = shape == "maj15"
    H.adversarial(cfg, 77 * sub + len(shape), 3000, 600 if sub == 1 else 2500,
                  max_batch=1 << 18 if wide else 1 << 16, tally_max_sub=sub)


# --------------------------------------------------------------------------- 2. order across boundaries
@pytest.mark.parametrize("form", ["host", "fused"])
@pytest.mark.parametrize("order", ["by_slot", "shuffled"])
@pytest.mark.parametrize("sub", SUBS)
def test_order_across_launch_boundaries(tally_path, sub, order, form):
    """Slot-sorted votes give every launch a narrow window (the sweep runs in each); shuffled votes give small
    launches a window far wider than themselves (the exact path).  Chosen stream, log and watermark."""
    n_slots = 3000 if sub == 1 else 20000
    eng, ora = H.make_pair(CFG2, n_slots, max_batch=1 << 17, tally_max_sub=sub)
    a, p, b = T.workload(11 + sub, CFG2, n_slots)
    if order == "by_slot":
        b = b[np.argsort(b["slot"], kind="stable")]
    c = tally_and_compare(form, eng, ora, b, arm=a)
    assert len(c) == n_slots
    if tally_path == "auto":
        last = b[(len(b) - 1) // sub * sub:]
        span = int(last["slot"].max()) - int(last["slot"].min())
        assert eng.last_tally_path == ("sweep" if span <= 4 * len(last) + 4096 else "exact")
        if order == "by_slot":
            assert eng.last_tally_path == "sweep"
        elif sub in (31, 1024, 1025):
            assert eng.last_tally_path == "exact"
    else:
        assert eng.last_tally_path == "exact"
    H.compare_log(eng, ora, 0, n_slots)
    eng.close()


@pytest.mark.parametrize("form", ["host", "fused"])
@pytest.mark.parametrize("revote", [False, True])
@pytest.mark.parametrize("keys", [1, 11, 341, 1366])
def test_completion_in_the_launch_after_the_first_votes(keys, revote, form):
    """Launch k carries the first f votes of `keys` keys, launch k+1 their completing votes.  With revote,
    launch k+2 also carries the other acceptors' votes and a duplicate completing vote for those keys,
    which find them Done.  Consecutive key groups are consecutive slots, so every launch's window is narrow."""
    cfg, f = CFG2, CFG2["f"]
    n_groups = 12
    g = T.rng(keys + 100 * revote)
    n_slots = keys * n_groups
    sub = (6 if revote else 3) * keys
    first, complete, late = [], [], []
    for j in range(n_groups):
        slots = np.arange(j * keys, (j + 1) * keys, dtype=np.int32)
        v = block_votes(cfg, g, slots, values=slots * 3 + 1, thrifty=False).reshape(keys, cfg["acceptors_per_group"])
        first.append(v[:, :f].reshape(-1))
        complete.append(v[:, f])
        late.append(np.concatenate([v[:, f + 1:].reshape(-1), v[:, f]]))
    blocks = []
    for j in range(n_groups + 2):
        parts = []
        if 0 <= j - 1 < n_groups:
            parts.append(complete[j - 1])
        if j < n_groups:
            parts.append(first[j])
        if revote and 0 <= j - 2 < n_groups:
            parts.append(late[j - 2])
        if not parts:
            continue
        blk = np.concatenate(parts)
        blk = blk[g.permutation(len(blk))]
        if len(blk) < sub and j < n_groups + (1 if revote else 0):
            # pad to one launch with re-deliveries of this launch's own votes (a voter's second delivery)
            blk = np.concatenate([blk, blk[g.integers(0, len(blk), size=sub - len(blk))]])
        assert len(blk) == sub or j == n_groups + (1 if revote else 0)
        blocks.append(blk)
    votes = np.concatenate(blocks)
    eng, ora = H.make_pair(cfg, n_slots, max_batch=1 << 17, tally_max_sub=sub)
    a = T.arms(np.arange(n_slots, dtype=np.int32), 0, np.arange(n_slots, dtype=np.int32) * 3 + 1)
    c = tally_and_compare(form, eng, ora, votes, arm=a)
    assert len(c) == n_slots
    H.compare_log(eng, ora, 0, n_slots)
    eng.close()


# --------------------------------------------------------------------------- 3. two rounds of one slot
@pytest.mark.parametrize("sub", [31, 1024, 1025])
def test_two_rounds_of_one_slot_chosen_in_different_launches_of_one_call(sub):
    """Slots armed in rounds 0 and 1 with different values (poisoned rows: the exact path) are chosen twice in
    one fpx_step_dev call, each round in a different launch, between launches of plain slot-sorted slots (the
    sweep, under auto).  The co-located log keeps the value of the earlier Chosen in the stream
    (S/multipaxos/Replica.scala:580-588), so the log numbers must grow from launch to launch on both paths."""
    cfg = CFG2
    g = T.rng(sub)
    n_plain, n_dual = 3000, 300
    plain = np.arange(n_plain, dtype=np.int32)
    dual = np.arange(n_plain, n_plain + n_dual, dtype=np.int32)
    x, y = dual[: n_dual // 2], dual[n_dual // 2:]
    arm = np.concatenate([T.arms(plain, 0, plain * 10), T.arms(dual, 0, dual * 10), T.arms(dual, 1, dual * 10 + 1)])
    sort = lambda v: v[np.argsort(v["slot"], kind="stable")]
    shuf = lambda v: v[g.permutation(len(v))]
    pv = sort(block_votes(cfg, g, plain, 0, plain * 10))
    half = len(pv) // 2
    votes = np.concatenate([
        pv[:half],
        shuf(np.concatenate([block_votes(cfg, g, x, 1, x * 10 + 1), block_votes(cfg, g, y, 0, y * 10)])),
        pv[half:],
        shuf(np.concatenate([block_votes(cfg, g, x, 0, x * 10), block_votes(cfg, g, y, 1, y * 10 + 1)])),
    ])
    eng, ora = H.make_pair(cfg, n_plain + n_dual, max_batch=1 << 16, overflow_capacity=1 << 12, tally_max_sub=sub)
    c = tally_and_compare("fused", eng, ora, votes, arm=arm)
    assert len(c) == n_plain + 2 * n_dual
    log = eng.snapshot_log(0, n_plain + n_dual)
    assert np.array_equal(log[x], x * 10 + 1) and np.array_equal(log[y], y * 10)
    H.compare_log(eng, ora, 0, n_plain + n_dual)
    eng.close()


# --------------------------------------------------------------------------- 4. error indices
ERROR_SUBS = [31, 1000, 1024, 1025]
N_ERR_SLOTS, N_EXTRA, ERR_CAPACITY = 3000, 16, 4096


def _error_trace(kind):
    """(engine factory, oracle factory, setup, votes, fatal(j) -> a fatal record on pending key j)."""
    if kind == "vanilla_round":
        f = 1
        n = 2 * f + 1
        req, p, b = T.vanilla_cfg5(5, f, N_ERR_SLOTS)
        extra = np.arange(N_ERR_SLOTS, N_ERR_SLOTS + N_EXTRA, dtype=np.int32)
        xr = np.zeros(N_EXTRA, dtype=P2A)
        xr["slot"] = extra; xr["value_id"] = extra * 3 + 1; xr["dst"] = extra % n
        req = np.concatenate([req, xr])
        mk_eng = lambda: Engine(f, 1, n, num_leaders=f + 1, num_replicas=f + 1, slot_capacity=ERR_CAPACITY,
                                max_batch=1 << 15, protocol=VANILLA_MENCIUS)
        mk_ora = lambda: O.VanillaMencius(f)

        def setup(eng, ora):
            eng.vm_client_request(req)
            assert ora.client_request(req) == (0, -1)
            H.same(eng.vm_phase2a(p), ora.phase2a(p)[2], "vanilla Phase2a replies")
        # a larger round than the pending entry's: checkEq (Server.scala:1116)
        fatal = lambda j: (0, (int(extra[j]) + 1) % n, int(extra[j]), 5)
        return mk_eng, mk_ora, setup, b, fatal
    # a non-member voter is the grid's `require(xs subsetOf nodes)` (Grid.scala:44-47)
    cfg = SHAPES["grid2x3"] if kind == "non_member" else CFG2
    a, _, b = T.workload(6, cfg, N_ERR_SLOTS)
    extra = np.arange(N_ERR_SLOTS, N_ERR_SLOTS + N_EXTRA, dtype=np.int32)
    a = np.concatenate([a, T.arms(extra, 0)])
    mk_eng = lambda: Engine(slot_capacity=ERR_CAPACITY, max_batch=1 << 15, overflow_capacity=1 << 8, **cfg)
    mk_ora = lambda: O.MultiPaxos(cfg["f"], cfg["num_acceptor_groups"], cfg["acceptors_per_group"], cfg["flexible"],
                                  cfg["num_leaders"], cfg["num_replicas"])

    def setup(eng, ora):
        H.arm(eng, ora, a)
    fatal = {
        "unarmed_round": lambda j: (0, 0, int(extra[j]), 9),                  # ProxyLeader.scala:220-225
        "non_member": lambda j: (5, 0, int(extra[j]), 0),                    # a pending key: the quorum test runs
        "past_window": lambda j: (0, 0, ERR_CAPACITY + 5 + j, 0),            # beyond the live window
    }[kind]
    return mk_eng, mk_ora, setup, b, fatal


EXPECT_CODE = {"unarmed_round": -4, "non_member": -5, "past_window": -6, "vanilla_round": -4}


def _plant(votes, fatal, where, sub):
    v = votes.copy()
    if where == "launch_start":
        at = [2 * sub]                         # the first vote of the third launch
    elif where == "last":
        at = [len(v) - 1]
    else:
        at = [sub - 2, sub + 1]                # a large index of the first launch, a small one of the second
    for j, i in enumerate(at):
        v[i] = fatal(j)
    return v, at[0]


def _dev_tally(eng, votes):
    import torch
    d_v = _td(votes)
    d_c = torch.zeros((len(votes), 2), dtype=torch.int32, device=torch.device("cuda", 0))
    eng.proxyleader_phase2b_dev(d_v.data_ptr(), len(votes), d_c.data_ptr())
    r = eng.sync(check=False)
    return r.status, r.err_index


@pytest.mark.parametrize("form", ["host", "dev"])
@pytest.mark.parametrize("kind", list(EXPECT_CODE))
@pytest.mark.parametrize("sub", ERROR_SUBS)
def test_error_index_is_the_call_index_of_the_first_offender(sub, kind, form):
    """A fatal vote at the first vote of a non-first launch, at the last vote of the call, and two fatal votes
    of which the later one has the smaller index within its launch: the status and the index are the
    oracle's, i.e. the call index of the first offending vote in delivery order (DESIGN section 1)."""
    mk_eng, mk_ora, setup, votes, fatal = _error_trace(kind)
    code = EXPECT_CODE[kind]
    eng = mk_eng()
    eng.set_tally_max_sub(sub)
    for where in ("launch_start", "last", "two"):
        eng.reset()
        ora = mk_ora()
        setup(eng, ora)
        v, first = _plant(votes, fatal, where, sub)
        ost, oidx, _ = ora.proxyleader_phase2b(v)
        # the oracle has no live window: a slot beyond it is simply never armed there (-4)
        assert (ost, oidx) == (-4 if code == -6 else code, first), (where, ost, oidx)
        if form == "host":
            with pytest.raises(FpxError) as ei:
                eng.proxyleader_phase2b(v)
            got = (ei.value.status, ei.value.index)
        else:
            got = _dev_tally(eng, v)
        assert got == (code, first), (where, got)
    eng.close()


def test_error_index_through_the_asynchronous_host_step():
    """fpx_step_submit / fpx_step_wait report the call index too."""
    import torch
    sub = 1000
    mk_eng, mk_ora, setup, votes, fatal = _error_trace("unarmed_round")
    eng, ora = mk_eng(), mk_ora()
    eng.set_tally_max_sub(sub)
    setup(eng, ora)
    v, first = _plant(votes, fatal, "two", sub)
    assert ora.proxyleader_phase2b(v)[:2] == (-4, first)
    hv = torch.from_numpy(v.view(np.int32).reshape(len(v), 4).copy()).pin_memory()
    oc = torch.zeros((len(v), 2), dtype=torch.int32).pin_memory()
    eng.step_submit(None, 0, None, 0, hv.data_ptr(), len(v), None, None, oc.data_ptr())
    with pytest.raises(FpxError) as ei:
        eng.step_wait()
    assert (ei.value.status, ei.value.index) == (-4, first)
    eng.close()


# --------------------------------------------------------------------------- 5. fused step across launches
@pytest.mark.parametrize("order", ["by_slot", "shuffled"])
@pytest.mark.parametrize("sub", [1000, 1025, 4097])
def test_fused_step_on_a_rebased_window(sub, order):
    """fpx_step_dev over four windows of a log twice as long as slot_capacity, retire_below between them; the
    votes of one slot per window arrive one call late, so the watermark stops inside the window and jumps at
    the next call.  Phase2b stream, Chosen stream, d_watermark and sync().watermark, acceptors and log."""
    cfg = CFG2
    W, wins = 3000, 4
    g = T.rng(sub)
    eng, ora = H.make_pair(cfg, 2 * W, max_batch=1 << 16, tally_max_sub=sub)
    held = np.zeros(0, dtype=P2B)
    for w in range(wins):
        a, p, b = T.workload(500 + w, cfg, W, slot0=w * W)
        hole = w * W + 77 + 31 * w
        late, b = b[b["slot"] == hole], b[b["slot"] != hole]
        b = np.concatenate([held, b])
        if order == "by_slot":
            b = b[np.argsort(b["slot"], kind="stable")]
        else:
            b = b[g.permutation(len(b))]
        held = late
        ob, on, oc, wm = oracle_step(ora, b, arm=a, p2a=p)
        r, eb, en, ec, d_wm = fused_step(eng, b, arm=a, p2a=p)
        assert (r.status, r.n_p2b, r.n_nack, r.n_chosen) == (0, len(ob), len(on), len(oc))
        H.same(eb, ob, f"Phase2b stream, window {w}")
        H.same(ec, oc, f"Chosen stream, window {w}")
        assert wm == hole
        assert r.watermark == d_wm == wm, (w, r.watermark, d_wm, wm)
        H.compare_acceptors(eng, ora, cfg, w * W, W)
        H.compare_log(eng, ora, w * W, W)
        if w >= 1:
            eng.retire_below(w * W)
    eng.close()


@pytest.mark.parametrize("sub", [1000, 4097])
def test_two_shards_publish_once_per_call(sub):
    """Two shards on one GPU (exchange_attach_local), every fused call cut into several launches: the
    exchange epoch advances by exactly one per call (no launch but the last publishes), and the global
    watermark is the oracle's, a hole in the first call included."""
    cfg = CFG2
    n_slots, P, calls = 6000, 2, 2
    a, p, b = T.workload(23, cfg, n_slots)
    hole = 1234
    ora = O.MultiPaxos(2, 1, 5, False, 3, 3)
    engs = [Engine(slot_capacity=n_slots, max_batch=1 << 16, shard_index=s, shard_count=P, **cfg) for s in range(P)]
    for e in engs:
        e.set_tally_max_sub(sub)
        for s, peer in enumerate(engs):
            e.exchange_attach_local(s, peer)
    per = n_slots // calls
    for k in range(calls):
        part = lambda r: r[(r["slot"] >= k * per) & (r["slot"] < (k + 1) * per)]
        ak, pk, bk = part(a), part(p), part(b)
        if k == 0:
            bk = bk[bk["slot"] != hole]
        else:
            bk = np.concatenate([bk, b[b["slot"] == hole]])
        bk = bk[np.argsort(bk["slot"], kind="stable")]
        ora.arm(ak); ora.acceptor_phase2a(pk)
        _, _, oc = ora.proxyleader_phase2b(bk)
        ora.replica_chosen(oc)
        for s, e in enumerate(engs):
            mine = lambda r: r[r["slot"] % P == s]
            r, _, _, c, d_wm = fused_step(e, mine(bk), arm=mine(ak), p2a=mine(pk))
            assert r.status == 0 and r.watermark == d_wm
            H.same(c, mine(oc), f"Chosen stream, call {k}, shard {s}")
            assert launches(len(mine(bk)), sub) > 1
            assert e.exchange_epoch == k + 1
        for e in engs:
            g_wm, fr = e.global_watermark(epoch=k + 1)
            assert g_wm == ora.executed_watermark() == (hole if k == 0 else n_slots)
            # nothing beyond the publications the host counted was published
            with pytest.raises(FpxError) as ei:
                e.global_watermark(epoch=k + 2, timeout_ms=20)
            assert ei.value.status == -16
    [e.close() for e in engs]


# --------------------------------------------------------------------------- 6. vanilla Mencius
@pytest.mark.parametrize("sub", [31, 1025])
@pytest.mark.parametrize("f", [1, 3])
def test_vanilla_step_across_launches(f, sub):
    """fpx_vm_step_dev with every tally call cut into launches: a ChosenEntry made in an earlier launch
    absorbs the later votes for its slot (Server.scala:1090-1093).  Two windows, the second carrying stale
    duplicates of the first's votes and delivered in slot order.  Against the oracle and against an engine
    whose calls are one launch each (log, servers' state)."""
    import torch
    n, W = 2 * f + 1, 3000
    dev = torch.device("cuda", 0)
    mk = lambda: Engine(f, 1, n, num_leaders=f + 1, num_replicas=f + 1, slot_capacity=2 * W,
                        max_batch=3 * (n - 1) * W, protocol=VANILLA_MENCIUS)
    one, ref, ora = mk(), mk(), O.VanillaMencius(f)
    one.set_tally_max_sub(sub)
    prev = None
    for w in range(2):
        req, p, b = T.vanilla_cfg5(80 + f + w, f, W, slot_offset=w * W)
        b = np.concatenate([b, b[: len(b) // 3]])                 # re-deliveries: later ones find ChosenEntry
        if prev is not None:
            b = np.concatenate([prev[: len(prev) // 2], b])
            b = b[np.argsort(b["slot"], kind="stable")]
        prev = b
        assert ora.client_request(req) == (0, -1)
        _, _, orep = ora.phase2a(p)
        st, _, oc = ora.proxyleader_phase2b(b)
        assert st == 0 and len(oc) == W
        d_req, d_p, d_b = _td(req), _td(p), _td(b)
        res = []
        for e in (one, ref):
            rep = torch.zeros((len(p), 4), dtype=torch.int32, device=dev)
            ch = torch.zeros((len(b), 2), dtype=torch.int32, device=dev)
            wm = torch.zeros(1, dtype=torch.int32, device=dev)
            e.vm_step_dev(d_req.data_ptr(), len(req), d_p.data_ptr(), len(p), rep.data_ptr(), d_b.data_ptr(), len(b),
                          ch.data_ptr(), wm.data_ptr())
            r = e.sync()
            assert (r.status, r.n_chosen, r.watermark, int(wm.item())) == (0, W, (w + 1) * W, (w + 1) * W)
            H.same(rep.cpu().numpy().view(P2B).reshape(-1), orep, f"Phase2a replies, window {w}")
            H.same(ch[: r.n_chosen].cpu().numpy().view(CHOSEN).reshape(-1), oc, f"Chosen stream, window {w}")
        log = one.snapshot_log(0, 2 * W)
        H.same(log, ref.snapshot_log(0, 2 * W), "log")
        assert np.array_equal(log[oc["slot"]], oc["value_id"])
    for s in range(n):
        x, y = one.snapshot_acceptor(0, s, 0, 2 * W), ref.snapshot_acceptor(0, s, 0, 2 * W)
        assert x[:2] == y[:2]
        H.same(x[2], y[2], f"server {s} voteRound"); H.same(x[3], y[3], f"server {s} voteValue")
    one.close(); ref.close()


# --------------------------------------------------------------------------- 7. launch count
@pytest.mark.parametrize("sub", SUBS)
def test_a_call_of_n_votes_takes_ceil_n_over_sub_launches(sub):
    eng, ora = H.make_pair(CFG2, 8192, tally_max_sub=sub)
    for n_slots in (1, 342, 1700):
        eng.reset()
        ora = O.MultiPaxos(2, 1, 5, False, 3, 3)
        a, _, b = T.workload(n_slots, CFG2, n_slots)
        H.arm(eng, ora, a)
        before = eng.launch_count
        st, c = H.phase2b(eng, ora, b)
        assert eng.launch_count - before == launches(len(b), sub)
        assert len(c) == n_slots
    eng.close()


def test_the_aid_rejects_sizes_outside_one_to_the_default():
    eng = Engine(slot_capacity=64, max_batch=1024, **CFG2)
    for bad in (-1, DEFAULT_MAX_SUB + 1):
        with pytest.raises(FpxError) as ei:
            eng.set_tally_max_sub(bad)
        assert ei.value.status == -1
    eng.set_tally_max_sub(DEFAULT_MAX_SUB)
    eng.set_tally_max_sub(0)
    eng.close()


# --------------------------------------------------------------------------- 8. full size, default limit
FULL_SLOTS = 3_600_000      # 10,800,000 votes: one launch of 10,485,760, then 314,240
FULL_FATAL = 10_500_000


@functools.lru_cache(maxsize=1)
def _full_trace():
    return T.workload(0, CFG2, FULL_SLOTS)


def _full_pair():
    eng, ora = H.make_pair(CFG2, FULL_SLOTS, max_batch=3 * FULL_SLOTS, overflow_capacity=1 << 10)
    return eng, ora


def test_full_size_call_split_at_the_default_limit(tally_path):
    """cfg2 with 3.6 M slots: 10.8 M shuffled votes in one call are two launches; the second one's window is
    far wider than its 314,240 votes (the exact path).  Chosen stream and log against the oracle."""
    if tally_path == "exact":
        pytest.skip("runs once (oracle time); the split itself is covered under both paths above")
    a, _, b = _full_trace()
    assert launches(len(b), DEFAULT_MAX_SUB) == 2
    eng, ora = _full_pair()
    H.arm(eng, ora, a)
    before = eng.launch_count
    st, c = H.phase2b(eng, ora, b)
    assert eng.launch_count - before == 2
    assert st == 0 and len(c) == FULL_SLOTS and eng.last_tally_path == "exact"
    H.replica(eng, ora, c)
    H.compare_log(eng, ora, 0, FULL_SLOTS)
    eng.close()


def test_full_size_error_index_in_the_second_launch(tally_path):
    """The same call with the vote at index 10,500,000 (the second launch's 14,240th) in a round that was
    never armed: (-4, 10500000), as the oracle says."""
    if tally_path == "exact":
        pytest.skip("runs once (oracle time)")
    a, _, b = _full_trace()
    bad = b.copy()
    bad["round"][FULL_FATAL] = 7
    eng, ora = _full_pair()
    H.arm(eng, ora, a)
    assert ora.proxyleader_phase2b(bad)[:2] == (-4, FULL_FATAL)
    with pytest.raises(FpxError) as ei:
        eng.proxyleader_phase2b(bad)
    assert (ei.value.status, ei.value.index) == (-4, FULL_FATAL)
    eng.close()
