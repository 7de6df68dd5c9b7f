"""fpx_reads_* on the GPU against the CPU oracle, bit for bit: the Client's and the ReadBatcher's read-quorum
tallies, and the replica's deferred reads released by the engine's own watermark."""
import numpy as np
import pytest

import harness as H
import reads_oracle as RO
import reads_traces as RT
from frankenpaxos_b200 import Engine, FpxError, Reads, READS_CLIENT, READS_READ_BATCHER
from frankenpaxos_b200 import traces as T
from oracle import fpx_oracle_py as O

pytestmark = pytest.mark.gpu

STRIDE_KEYS = 132 * 1024 * 4   # past one grid stride of any launch the handle makes on an H100


def engine(cfg, **kw):
    return Engine(slot_capacity=1 << 12, max_batch=1 << 12, overflow_capacity=1 << 8, **cfg, **kw)


def oracle_tally(cfg, kind):
    return RO.ReadTally(kind, cfg["f"], cfg["num_acceptor_groups"], cfg["acceptors_per_group"], cfg["flexible"])


def tally_pair(cfg, kind, key_capacity, max_batch):
    eng = engine(cfg)
    return eng, Reads(eng, kind, key_capacity=key_capacity, pending_capacity=16, max_batch=max_batch), oracle_tally(cfg, kind)


@pytest.mark.parametrize("shape", ["cfg1", "maj5", "grid2x3", "maj15", "grid5x6"])
@pytest.mark.parametrize("kind", [READS_CLIENT, READS_READ_BATCHER])
def test_tally_matches_oracle(shape, kind):
    cfg = RT.SHAPES[shape]
    eng, r, ora = tally_pair(cfg, kind, 4096, 1 << 15)
    trace = RT.tally_trace(7 + kind, cfg, kind, 4096, 8, 1 << 15, hot_keys=3)
    a, b = RT.run_tally(r, trace), RT.run_tally(ora, trace)
    RT.same_outputs(a, b, f"{shape} kind {kind}")
    assert sum(len(x) for x in a) > 1000
    r.close(); eng.close()


@pytest.mark.parametrize("kind", [READS_CLIENT, READS_READ_BATCHER])
def test_tally_2p20_replies_past_one_grid_stride(kind):
    """cfg2's shape (f = 2): batches of 2^20 replies over keys past one grid stride, with duplicates, late
    replies, stale ids and unopened keys."""
    cfg = RT.SHAPES["maj5"]
    cap = 1 << 21
    assert cap > STRIDE_KEYS
    eng, r, ora = tally_pair(cfg, kind, cap, 1 << 20)
    trace = RT.tally_trace(99, cfg, kind, cap, 3, 1 << 20, slot_hi=1 << 30)
    a, b = RT.run_tally(r, trace), RT.run_tally(ora, trace)
    RT.same_outputs(a, b, f"kind {kind}")
    assert max(int(x["key"].max()) for x in a if len(x)) > STRIDE_KEYS
    r.close(); eng.close()


@pytest.mark.parametrize("shape", ["maj5", "grid5x6"])
@pytest.mark.parametrize("kind", [READS_CLIENT, READS_READ_BATCHER])
def test_one_key_over_many_tiles(shape, kind):
    """A read with more than 3000 replies: one voter repeats itself across several 1024-reply tiles (its
    LATEST slot counts, and it is smaller than the earlier ones), the quorum completes in a later tile, and the
    replies after it are ignored.  Other keys' replies are interleaved, so the segment's tile boundaries fall
    anywhere."""
    cfg = RT.SHAPES[shape]
    G, A = cfg["num_acceptor_groups"], cfg["acceptors_per_group"]
    g = np.random.default_rng(5)
    for n_hot in (3000, 1024 * 3, 1024 * 3 + 1, 1024 * 4 - 1):
        eng, r, ora = tally_pair(cfg, kind, 1 << 12, 1 << 14)
        keys = np.arange(1 << 12, dtype=np.int32)
        for h in (r, ora):
            h.open(keys, np.ones(len(keys), np.int32))
        # the hot key 17: voter (0, 0) over and over with decreasing slots, then the rest of a quorum
        first = RT.voter(0, 0)
        quorum = [RT.voter(0, a) for a in range(1, A)] if kind == READS_CLIENT and cfg["flexible"] else \
            [RT.voter(0, a) for a in range(1, cfg["f"] + 1)]
        hot = np.zeros(n_hot, RO.MAX_SLOT_REPLY)
        hot["key"], hot["id"] = 17, 1
        hot["voter"] = first
        hot["slot"] = np.arange(n_hot, 0, -1) + 5000
        hot["slot"][-len(quorum) - 1] = 1      # voter (0, 0)'s latest slot is its smallest
        hot["voter"][-len(quorum):] = quorum
        hot["slot"][-len(quorum):] = 3
        late = np.zeros(50, RO.MAX_SLOT_REPLY)
        late["key"], late["id"], late["voter"], late["slot"] = 17, 1, RT.voter(0, A - 1), 1 << 29
        cold = np.zeros(5000, RO.MAX_SLOT_REPLY)
        cold["key"] = g.integers(0, 1 << 12, len(cold))
        cold["id"] = 1
        cold["voter"] = RT.voter(g.integers(0, G, len(cold)) if cfg["flexible"] else 0, g.integers(0, A, len(cold)))
        cold["slot"] = g.integers(0, 1 << 20, len(cold))
        cold = cold[cold["key"] != 17]
        recs = np.concatenate([hot, late, cold])
        order = np.sort(g.choice(len(recs), len(hot) + len(late), replace=False))
        mixed = np.empty_like(recs)
        mask = np.zeros(len(recs), bool); mask[order] = True
        mixed[mask] = np.concatenate([hot, late])
        mixed[~mask] = cold
        a = r.max_slot_replies(mixed)
        st, err, b = ora.max_slot_replies(mixed)
        assert st == 0
        H.same(a, b, f"{shape} kind {kind} n_hot {n_hot}")
        row = a[a["key"] == 17]
        assert len(row) == 1 and row["slot"][0] == 3 + (0 if kind == READS_CLIENT and cfg["flexible"] else G - 1)
        r.close(); eng.close()


def test_flexible_client_non_member_and_bad_keys():
    cfg = RT.SHAPES["grid2x3"]
    eng, r, ora = tally_pair(cfg, READS_CLIENT, 64, 1024)
    for h in (r, ora):
        h.open([0, 1], [0, 0])
    recs = np.zeros(4, RO.MAX_SLOT_REPLY)
    recs[:] = [(1, 7, 3, 0), (0, 0, 0, 1), (0, 0, 3, 2), (0, 0, 1 << 16 | 7, 2)]
    st, err, _ = ora.max_slot_replies(recs)
    with pytest.raises(FpxError) as ei:
        r.max_slot_replies(recs)
    assert (ei.value.status, ei.value.index) == (st, err) == (-5, 2)
    with pytest.raises(FpxError) as ei:
        r.open([3, 64], [0, 0])
    assert (ei.value.status, ei.value.index) == (-1, 1)
    r.close(); eng.close()


def deferred_pair(pending, max_batch, eng=None):
    eng = eng or engine(RT.SHAPES["cfg1"])
    return eng, Reads(eng, READS_CLIENT, key_capacity=1, pending_capacity=pending, max_batch=max_batch), \
        RO.DeferredReads(pending)


@pytest.mark.parametrize("spread", [96, 1 << 16])
def test_replica_matches_oracle(spread):
    eng, r, ora = deferred_pair(1 << 20, 1 << 14)
    trace = RT.replica_trace(3, 40, 1 << 14, step=spread // 2, spread=spread)
    a, b = RT.run_replica(r, trace), RT.run_replica(ora, trace)
    RT.same_outputs(a, b, f"spread {spread}")
    assert sum(len(x) for x in a[1::2]) > 10000
    r.close(); eng.close()


def test_replica_2p20_batch_and_release():
    eng, r, ora = deferred_pair(1 << 20, 1 << 20)
    g = np.random.default_rng(11)
    req = np.zeros(1 << 20, RO.READ_REQUEST)
    req["slot"] = g.integers(0, 1 << 18, len(req))
    req["handle"] = np.arange(len(req))
    trace = [("req", req[:1000]), ("adv", 10), ("req", req[1000:]), ("adv", 1 << 17), ("adv", 1 << 18)]
    a, b = RT.run_replica(r, trace), RT.run_replica(ora, trace)
    RT.same_outputs(a, b, "2^20")
    assert len(a[-1]) + len(a[-2]) + len(a[1]) > (1 << 20) - 2000
    r.close(); eng.close()


def test_replica_overflow_applies_nothing():
    eng, r, ora = deferred_pair(1000, 1 << 12)
    g = np.random.default_rng(2)
    first = np.zeros(900, RO.READ_REQUEST)
    first["slot"], first["handle"] = g.integers(100, 200, 900), np.arange(900)
    batch = np.zeros(2048, RO.READ_REQUEST)
    batch["slot"] = g.integers(-1, 300, 2048)
    batch["slot"][:1100] = g.integers(-1, 50, 1100)   # answered now: the overflow lies past the first tile
    batch["handle"] = 1000 + np.arange(2048)
    r.advance(50); ora.advance(50)
    RT.same_outputs([r.replica(first)], [ora.replica(first)[2]], "fill")
    st, err, _ = ora.replica(batch)
    assert st == -8 and err > 1024       # the read that does not fit lies in the batch's second tile
    with pytest.raises(FpxError) as ei:
        r.replica(batch)
    assert (ei.value.status, ei.value.index) == (st, err)
    # nothing applied: the pool still releases exactly the first batch's reads
    RT.same_outputs([r.advance(1000)], [ora.advance(1000)[1]], "after overflow")
    with pytest.raises(FpxError) as ei:
        r.advance(999)
    assert ei.value.status == -1
    r.close(); eng.close()


def test_reads_released_by_engine_steps():
    """Reads wait for slots of a real cfg2 log: arm -> phase2a -> phase2b -> replica_chosen in slot windows,
    the host watermark releases them; then the same through fpx_step_dev's d_watermark and advance_dev."""
    import torch
    cfg, _ = T.config_by_name("cfg2")
    n_slots = 8192
    a, p, b = T.workload(4, cfg, n_slots)
    dev = torch.device("cuda", 0)
    td = lambda x: torch.from_numpy(np.ascontiguousarray(x).view(np.int32).reshape(len(x), -1).copy()).to(dev)
    g = np.random.default_rng(4)
    for use_dev in (False, True):
        eng = Engine(slot_capacity=n_slots, max_batch=1 << 16, **cfg)
        ora_log = O.MultiPaxos(2, 1, 5, False, 3, 3)
        r = Reads(eng, READS_CLIENT, key_capacity=1, pending_capacity=1 << 16, max_batch=1 << 14)
        ora = RO.DeferredReads(1 << 16)
        handle = 0
        for lo in range(0, n_slots, 1024):
            sel = lambda x: x[(x["slot"] >= lo) & (x["slot"] < lo + 1024)]
            req = np.zeros(3000, RO.READ_REQUEST)
            req["slot"] = g.integers(-1, min(lo + 2048, n_slots), len(req))
            req["handle"] = handle + np.arange(len(req)); handle += len(req)
            RT.same_outputs([r.replica(req)], [ora.replica(req)[2]], f"requests {lo}")
            ora_log.arm(sel(a)); ora_log.acceptor_phase2a(sel(p))
            _, _, oc = ora_log.proxyleader_phase2b(sel(b))
            ora_log.replica_chosen(oc)
            W = ora_log.executed_watermark()
            if not use_dev:
                eng.proxyleader_arm(sel(a)); eng.acceptor_phase2a(sel(p))
                eng.replica_chosen(eng.proxyleader_phase2b(sel(b)))
                out = r.advance(eng.chosen_watermark())
            else:
                da, dp, db = td(sel(a)), td(sel(p)), td(sel(b))
                o1 = torch.zeros((len(dp), 4), dtype=torch.int32, device=dev)
                o2 = torch.zeros((len(dp), 2), dtype=torch.int32, device=dev)
                o3 = torch.zeros((len(db), 2), dtype=torch.int32, device=dev)
                wm = torch.zeros(1, dtype=torch.int32, device=dev)
                d_out = torch.zeros((1 << 16, 4), dtype=torch.int32, device=dev)
                eng.step_dev(da.data_ptr(), len(da), dp.data_ptr(), len(dp), o1.data_ptr(), o2.data_ptr(),
                             db.data_ptr(), len(db), o3.data_ptr(), wm.data_ptr())
                r.advance_dev(wm.data_ptr(), d_out.data_ptr())   # same stream: no host round trip in between
                s = r.sync()
                eng.sync()
                assert s.watermark == W
                out = d_out[:s.n_released].cpu().numpy().reshape(-1).view(RO.READ_REPLY)
            st, want = ora.advance(W)
            RT.same_outputs([out], [want], f"release at {lo} (dev {use_dev})")
        assert W == n_slots and ora.pending == 0
        r.close(); eng.close()


def test_reads_across_retire_below():
    """The handle keeps working while the engine slides its window: reads for slots beyond the first window."""
    cfg, _ = T.config_by_name("cfg1")
    cap = 2048
    eng = Engine(slot_capacity=cap, max_batch=1 << 14, **cfg)
    ora_log = O.MultiPaxos(1, 1, 3, False, 2, 2)
    r = Reads(eng, READS_CLIENT, key_capacity=1, pending_capacity=1 << 14, max_batch=1 << 14)
    ora = RO.DeferredReads(1 << 14)
    g = np.random.default_rng(8)
    total = 4 * cap
    a, p, b = T.workload(8, cfg, total)
    for lo in range(0, total, cap // 2):
        sel = lambda x: x[(x["slot"] >= lo) & (x["slot"] < lo + cap // 2)]
        req = np.zeros(1000, RO.READ_REQUEST)
        req["slot"] = g.integers(max(lo - 100, -1), lo + cap, len(req))
        req["handle"] = lo * 10 + np.arange(len(req))
        RT.same_outputs([r.replica(req)], [ora.replica(req)[2]], f"requests {lo}")
        eng.proxyleader_arm(sel(a)); eng.acceptor_phase2a(sel(p))
        eng.replica_chosen(eng.proxyleader_phase2b(sel(b)))
        ora_log.arm(sel(a)); ora_log.acceptor_phase2a(sel(p))
        ora_log.replica_chosen(ora_log.proxyleader_phase2b(sel(b))[2])
        W = eng.chosen_watermark()
        assert W == ora_log.executed_watermark()
        RT.same_outputs([r.advance(W)], [ora.advance(W)[1]], f"release {lo}")
        eng.retire_below(W)
    assert W == total
    r.close(); eng.close()


def test_tally_dev_form_and_sync_counts():
    import torch
    cfg = RT.SHAPES["grid2x3"]
    eng, r, ora = tally_pair(cfg, READS_CLIENT, 256, 4096)
    trace = RT.tally_trace(12, cfg, READS_CLIENT, 256, 3, 4096)
    dev = torch.device("cuda", 0)
    for op in trace:
        if op[0] == "open":
            r.open(op[1], op[2]); ora.open(op[1], op[2])
            continue
        d_in = torch.from_numpy(op[1].view(np.int32).reshape(-1, 4).copy()).to(dev)
        d_out = torch.zeros((len(op[1]), 4), dtype=torch.int32, device=dev)
        r.max_slot_replies_dev(d_in.data_ptr(), len(op[1]), d_out.data_ptr())
        s = r.sync()
        got = d_out[:s.n_slots].cpu().numpy().reshape(-1).view(RO.READ_SLOT)
        RT.same_outputs([got], [ora.max_slot_replies(op[1])[2]], "dev form")
    r.close(); eng.close()


def test_engine_destroyed_first_with_work_queued():
    """The engine goes first, with the reads handle's device-form batches still queued on its stream; then the
    reads handle goes, and a new pair on the same device matches the oracle."""
    import torch
    cfg = RT.SHAPES["grid2x3"]
    eng, r, ora = tally_pair(cfg, READS_CLIENT, 256, 4096)
    trace = RT.tally_trace(12, cfg, READS_CLIENT, 256, 3, 4096)
    dev = torch.device("cuda", 0)
    queued = []
    for op in trace:
        if op[0] == "open":
            r.open(op[1], op[2]); ora.open(op[1], op[2])
            continue
        d_in = torch.from_numpy(op[1].view(np.int32).reshape(-1, 4).copy()).to(dev)
        d_out = torch.zeros((len(op[1]), 4), dtype=torch.int32, device=dev)
        torch.cuda.synchronize()
        r.max_slot_replies_dev(d_in.data_ptr(), len(op[1]), d_out.data_ptr())
        queued.append((d_in, d_out, ora.max_slot_replies(op[1])[2]))
    eng.close()   # drains the engine's stream: every queued batch has run
    for _, d_out, want in queued:
        got = d_out.cpu().numpy()
        RT.same_outputs([got[:len(want)].reshape(-1).view(RO.READ_SLOT)], [want], "queued dev form")
        assert not got[len(want):].any()
    assert sum(len(w) for _, _, w in queued) > 0
    r.close()
    eng, r, ora = tally_pair(cfg, READS_CLIENT, 256, 4096)
    RT.same_outputs(RT.run_tally(r, trace), RT.run_tally(ora, trace), "after the engine went first")
    r.close(); eng.close()


def test_create_checks():
    eng = engine(RT.SHAPES["cfg1"])
    with pytest.raises(FpxError) as ei:
        Reads(eng, 7)
    assert ei.value.status == -1
    eng.close()
    m = Engine(slot_capacity=1024, max_batch=1024, protocol=1, num_leader_groups=2, f=1, num_acceptor_groups=1,
               acceptors_per_group=3)
    with pytest.raises(FpxError) as ei:
        Reads(m)
    assert ei.value.status == -11
    m.close()
