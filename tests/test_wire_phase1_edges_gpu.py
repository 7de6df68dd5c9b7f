"""The Phase 1 wire paths at the edges of their own kernels, on the GPU against the CPU oracles
(tests/wire_phase1_oracle.cc, tests/wire_mencius_phase1_oracle.cc) and tests/vm_revoke_model.py: the leader's walk
window, oneof handling, entry placement, parse / max / first grid strides and emit CTA cap, int32 slot edges; the
acceptors' 1024-slot tiles, count-scan chunks, record limit and 30 keys; the Phase1b and Phase2a encoders' length
widths, scan chunk and capacity; the vanilla Mencius walk's 256-slot chunks.  Batches come from
tests/wire_phase1_edges.py."""
import numpy as np
import pytest

import wire_mencius_phase1_oracle as MO
import wire_phase1_edges as E
import wire_phase1_oracle as O
from frankenpaxos_b200 import MENCIUS, P2A, P2B, VALUE_NOOP, VANILLA_MENCIUS, Engine, FpxError, dst
from vm_revoke_model import Server

pytestmark = pytest.mark.gpu
SENTINEL = 0x5a


def status_of(fn, *a, **kw):
    try:
        return 0, -1, fn(*a, **kw)
    except FpxError as e:
        return e.status, e.index, None


def mp_same(eng, buf, offs, cw, cap, f=1, groups=1, per_group=3, round_=9, base=40):
    """the engine's leader call against fpo_leader_phase1b -> the oracle's tuple"""
    o = O.leader_phase1b(f, groups, per_group, 0, round_, cw, buf, offs, base, cap)
    st, idx, got = status_of(eng.leader_phase1b_wire, round_, cw, buf, offs, base, cap)
    assert (st, idx) == (o[0], o[1])
    if st == 0:
        complete, max_slot, recs, spans = got
        assert (complete, max_slot) == (o[2], o[3])
        assert np.array_equal(recs.view(np.int32), o[4].view(np.int32)) and np.array_equal(spans, o[5])
    return o


def mencius_same(eng, buf, offs, lg, cw, rec, cap, f=1, lgroups=3, agroups=2, round_=9, base=40):
    o = MO.leader_phase1b(f, lgroups, agroups, 2 * f + 1, lg, round_, cw, buf, offs, rec, base, cap)
    st, idx, got = status_of(eng.mencius_leader_phase1b_wire, lg, round_, cw, buf, offs, rec, base, cap)
    assert (st, idx) == (o[0], o[1])
    if st == 0:
        complete, max_slot, next_slot, recs, spans = got
        assert (complete, max_slot, next_slot) == (o[2], o[3], o[4])
        assert np.array_equal(recs.view(np.int32), o[5].view(np.int32)) and np.array_equal(spans, o[6])
    return o


def leader_dev(eng, buf, offs, cw, cap, mencius=None, round_=9, base=40):
    """the _dev form over sentinel-filled outputs -> (status, result, records int32[k, 4], spans, untouched tail)"""
    import torch
    dev = torch.device("cuda", 0)
    d_buf, d_offs = torch.from_numpy(buf).to(dev), torch.from_numpy(offs).to(dev)
    d_out = torch.full((max(cap, 1) + 4, 4), SENTINEL, dtype=torch.int32, device=dev)
    d_sp = torch.full((max(cap, 1) + 4, 2), SENTINEL, dtype=torch.int32, device=dev)
    d_res = torch.full((4,), SENTINEL, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    try:
        if mencius is None:
            eng.leader_phase1b_wire_dev(round_, cw, d_buf.data_ptr(), len(buf), d_offs.data_ptr(), len(offs) - 1, base,
                                        d_out.data_ptr(), d_sp.data_ptr(), cap, d_res.data_ptr())
        else:
            lg, rec = mencius
            eng.mencius_leader_phase1b_wire_dev(lg, round_, cw, rec, d_buf.data_ptr(), len(buf), d_offs.data_ptr(),
                                                len(offs) - 1, base, d_out.data_ptr(), d_sp.data_ptr(), cap,
                                                d_res.data_ptr())
        eng.sync()
        st = 0
    except FpxError as e:
        st = e.status
    res = d_res.cpu().numpy()
    k = int(res[2]) if st == 0 else 0
    out, sp = d_out.cpu().numpy(), d_sp.cpu().numpy()
    untouched = (out[k:] == SENTINEL).all() and (sp[k:] == SENTINEL).all()
    return st, res, out[:k], sp[:k], untouched


@pytest.fixture(scope="module")
def mp():
    e = Engine(1, 1, 3, slot_capacity=1 << 12, max_batch=1 << 12)
    yield e
    e.close()


@pytest.fixture(scope="module")
def big():
    e = Engine(1, 1, 3, slot_capacity=1 << 12, max_batch=1 << 24)
    yield e
    e.close()


@pytest.fixture(scope="module")
def mp5():
    e = Engine(2, 1, 5, slot_capacity=1 << 12, max_batch=1 << 12)
    yield e
    e.close()


@pytest.fixture(scope="module")
def men():
    e = Engine(1, 2, 3, protocol=MENCIUS, num_leader_groups=3, slot_capacity=1 << 12, max_batch=1 << 12)
    yield e
    e.close()


@pytest.fixture(scope="module")
def men1():
    e = Engine(1, 1, 3, protocol=MENCIUS, num_leader_groups=1, slot_capacity=1 << 12, max_batch=1 << 12)
    yield e
    e.close()


# --------------------------------------------------------------------------- p1_walk_kernel: the window's end
@pytest.mark.parametrize("target", ["info", "scalar", "member"])
@pytest.mark.parametrize("d", E.WINDOW_DISTANCES, ids=[f"16384-{d}" for d in E.WINDOW_DISTANCES])
def test_walk_header_at_window_end(mp, d, target):
    g = np.random.default_rng(d + 7)
    for tag_w, len_w in [(1, None), (1, 10), (5, 10), (10, 10)]:
        for lead in (0, 5, 33):
            buf, offs, m, pos, head, infos = E.window_batch(d, target, tag_w, len_w, lead, g)
            o = mp_same(mp, buf, offs, 0, 64)
            assert o[0] == 0 and o[2] == 1 and len(o[4]) == 22        # slots 0 .. 21 re-proposed from the edge message


# --------------------------------------------------------------------------- the walk's oneof handling
@pytest.mark.parametrize("case", sorted(E.oneof_cases()))
def test_walk_oneof_members(mp, men1, case):
    msg, want = E.oneof_cases()[case]
    buf, offs = E.oneof_batch(msg)
    o = mp_same(mp, buf, offs, 0, 64)
    assert o[0] == (E.ERR_WIRE if want == "bad" else 0)
    if isinstance(want, tuple):
        assert len(o[4]) == max(s for s, _, _ in want[3]) + 1
    msg, want = E.oneof_cases(nack=7)[case]
    buf, offs = E.oneof_batch(msg)
    mencius_same(men1, buf, offs, 0, 0, -1, 64, lgroups=1, agroups=1)


# --------------------------------------------------------------------------- entry placement, tightest packing
@pytest.mark.parametrize("lead", range(16))
def test_tight_infos_at_every_offset(mp5, lead):
    buf, offs = E.tight_batch(lead, np.random.default_rng(lead + 100))
    o = mp_same(mp5, buf, offs, 0, 256, f=2, per_group=5)
    assert o[0] == 0 and o[2] == len(offs) - 2 and len(o[4]) > 0
    assert (o[4]["value_id"] != VALUE_NOOP).sum() > 0


# --------------------------------------------------------------------------- p1_parse / p1_max / p1_first strides
@pytest.mark.parametrize("k", E.PARSE_EDGES)
def test_parse_grid_stride_one_phase1b(big, k):
    """one Phase1b of k infos: its entries past 262 144 take the second grid-stride step; the highest slot is the
    last info, and acceptor 2's Phase1b ties and outvotes it around the stride edge"""
    g = np.random.default_rng(k)
    slots = np.arange(k, dtype=np.int64)
    whole = E.many_infos(0, 9, slots, g)
    near = np.arange(max(0, E.PARSE_STRIDE - 40), k, dtype=np.int64)
    other = E.many_infos(2, 9, near, g)
    buf, offs = E.pack([whole, other], 3)
    o = mp_same(big, buf, offs, 0, k)
    assert o[0] == 0 and o[3] == k - 1 and len(o[4]) == k
    st, res, recs, spans, untouched = leader_dev(big, buf, offs, 0, k)
    assert st == 0 and res[:3].tolist() == [1, k - 1, k] and untouched
    assert np.array_equal(recs.reshape(-1), o[4].view(np.int32).reshape(-1)) and np.array_equal(spans, o[5])


@pytest.mark.parametrize("fill", [E.GRID_Y - 1, E.GRID_Y, E.GRID_Y + 1])
def test_parse_grid_y_many_messages(big, fill):
    """`fill` messages of no member, then the quorum's Phase1bs at indices >= 65 534: past gridDim.y = 65 535"""
    g = np.random.default_rng(fill)
    stale = E.phase1b(0, 0, 8, [(900, 1, E.VALUES[1])])
    q = [E.many_infos(a, 9, np.sort(g.choice(300, 120, replace=False)), g) for a in (0, 2)]
    late = E.phase1b(0, 1, 9, [(5000, 1, E.VALUES[1])])
    msgs = [stale] + [b""] * (fill - 1) + q + [late]
    buf, offs = E.pack(msgs, 1)
    o = mp_same(big, buf, offs, 0, 400)
    assert o[0] == 0 and o[2] == fill + 1 and o[3] < 300
    st, res, recs, spans, untouched = leader_dev(big, buf, offs, 0, 400)
    assert st == 0 and res[:3].tolist() == [fill + 1, o[3], len(o[4])] and untouched
    assert np.array_equal(recs.reshape(-1), o[4].view(np.int32).reshape(-1)) and np.array_equal(spans, o[5])


# --------------------------------------------------------------------------- p1_emit: 4096 CTAs, grid-stride
@pytest.mark.parametrize("count", E.EMIT_EDGES)
def test_emit_rows_at_the_cta_cap(big, count):
    cw = 77
    buf, offs = E.emit_batch(count, cw)
    o = mp_same(big, buf, offs, cw, count)
    assert o[0] == 0 and len(o[4]) == count and o[4]["slot"][-1] == cw + count - 1
    st, res, recs, spans, untouched = leader_dev(big, buf, offs, cw, count)
    assert st == 0 and res[:3].tolist() == [1, cw + count - 1, count] and untouched
    assert np.array_equal(recs.reshape(-1), o[4].view(np.int32).reshape(-1)) and np.array_equal(spans, o[5])
    # one row short: refused at `complete`, nothing written
    assert mp_same(big, buf, offs, cw, count - 1)[:2] == (E.ERR_INVALID_ARG, 1)
    st, res, _, _, untouched = leader_dev(big, buf, offs, cw, count - 1)
    assert st == E.ERR_INVALID_ARG and untouched


def test_phase2a_past_the_scan_chunk(big):
    """the re-proposed Phase2a of more than SCAN_CHUNK x ENC_TILE records through the gathering encoder"""
    n = E.BIG_P2A
    buf, offs = E.p2a_chunk_batch(n)
    o = mp_same(big, buf, offs, 0, n)
    assert len(o[4]) == n
    hb, hoffs = big.wire_encode_phase2a(o[4], buf, o[5], 40)
    ost, _, ob, ooffs = O.encode_phase2a(o[4], buf, o[5], 40)
    assert ost == 0 and np.array_equal(hoffs, ooffs) and bytes(hb) == bytes(ob)


# --------------------------------------------------------------------------- int32 slot edges
@pytest.mark.parametrize("case", sorted(E.mp_slot_cases()))
def test_mp_slot_extremes(mp, case):
    msgs, cw = E.mp_slot_cases()[case]
    buf, offs = O.pack(msgs)
    o = mp_same(mp, buf, offs, cw, 64)
    assert o[0] == 0


@pytest.mark.parametrize("case", sorted(E.mencius_slot_cases()))
def test_mencius_slot_extremes(men, case):
    """DESIGN §7: a next_slot past INT32_MAX is refused (FPX_ERR_SLOT_RANGE at complete) where the reference's Int
    would wrap; exactly INT32_MAX is accepted"""
    lg, cw, rec, msgs = E.mencius_slot_cases()[case]
    buf, offs = O.pack(msgs)
    o = mencius_same(men, buf, offs, lg, cw, rec, 64)
    want = E.MENCIUS_SLOT_STATUS.get(case, 0)
    assert o[0] == want
    if case in ("next_slot_int32_max", "recover_next_slot_int32_max"):
        assert o[4] == E.INT_MAX
    st, res, recs, spans, untouched = leader_dev(men, buf, offs, cw, 64, mencius=(lg, rec))
    assert st == want and untouched
    if st == 0:
        assert res.tolist() == [o[2], o[3], len(o[5]), o[4]]
        assert np.array_equal(recs.reshape(-1), o[5].view(np.int32).reshape(-1)) and np.array_equal(spans, o[6])
    if st == 0 and len(o[5]):                        # their Phase2a bytes, slots up to INT32_MAX included
        hb, hoffs = men.wire_encode_mencius_phase2a(o[5], buf, o[6], 40)
        ost, _, ob, ooffs = MO.encode_phase2a(o[5], buf, o[6], 40)
        assert ost == 0 and np.array_equal(hoffs, ooffs) and bytes(hb) == bytes(ob)


def test_cross_group_votes_are_not_read():
    """MultiPaxos 2 x 3: group 1's higher votes on group 0's slots raise max_slot only; safeValue reads the slot's
    own group (Leader.scala:552)"""
    with Engine(1, 2, 3, slot_capacity=1 << 10, max_batch=1 << 12) as e:
        buf, offs = O.pack(E.cross_group_mp())
        o = mp_same(e, buf, offs, 0, 64, groups=2)
        assert (o[0], o[2], o[3], len(o[4])) == (0, 3, 6, 7)
        assert o[4]["value_id"][6] == VALUE_NOOP and (o[5][[0, 2, 4], 1] == len(E.VALUES[1])).all()
        st, res, recs, spans, untouched = leader_dev(e, buf, offs, 0, 64)
        assert st == 0 and untouched and np.array_equal(recs.reshape(-1), o[4].view(np.int32).reshape(-1))


# --------------------------------------------------------------------------- the acceptors' side
VALS = [b"\x0a\x00", b"\x0a\x07\x0a\x05\x0a\x01a\x10\x01"]


def arena_of(values):
    a = np.frombuffer(b"".join(values) + b"\0", np.uint8)[:sum(len(v) for v in values)].copy()
    return a, np.concatenate([[0], np.cumsum([len(v) for v in values])]).astype(np.int32)


def phase1a(round_, cw):
    return E.field(1, E.fint(1, round_) + E.fint(2, cw))


def phase1a_batch(reqs, dests):
    """AcceptorInbound{phase1a} bytes and the records fpx_wire_decode_inbound writes for them"""
    msgs = [phase1a(r, cw) for r, cw in reqs]
    buf, offs = O.pack(msgs)
    recs = np.zeros(len(msgs), O.WIRE_REC)
    recs["a"] = dests
    recs["c"] = offs[:-1] + 2
    recs["d"] = [len(m) - 2 for m in msgs]
    assert all(len(m) < 130 for m in msgs)
    return buf, np.ones(len(msgs), np.int32), recs


def acceptor_same(e, o, reqs, dests, arena, voffs, first_held=0, mencius=False, keys=None):
    buf, kind, recs = phase1a_batch(reqs, dests)
    ost, oidx, ob, ooffs = o.phase1a_wire(first_held, buf, kind, recs, arena, voffs)
    call = e.mencius_acceptor_phase1a_wire if mencius else e.acceptor_phase1a_wire
    st, idx, got = status_of(call, buf, kind, recs, arena, voffs)
    assert (st, idx) == (ost, oidx)
    if st == 0:
        assert bytes(got[0]) == bytes(ob) and np.array_equal(got[1], ooffs)
    for k in keys:
        assert e.snapshot_acceptor(*k)[0] == o.round(*k)
    return st, got, (buf, kind, recs)


def votes(slots, acceptor_keys, round_, value):
    p = np.zeros(len(slots) * len(acceptor_keys), O.P2A)
    p["slot"] = np.repeat(slots, len(acceptor_keys))
    p["round"] = round_
    p["value_id"] = value
    p["dst"] = np.tile([int(dst(*k)) for k in acceptor_keys], len(slots))
    return p


def test_acceptor_tile_offsets():
    """voted slots at tile offsets 1023 / 1024 / 1025 from chosen_watermark, a range of exactly one slot, an empty
    one and the last slot of the live window"""
    S = 4096
    a, voffs = arena_of(VALS)
    keys = [(0, c) for c in range(3)]
    with Engine(1, 1, 3, slot_capacity=S, max_batch=1 << 13) as e:
        o = O.Acceptors(1, 1, 3)
        for cw in (0, 1, 1000):
            p = votes(np.array([cw + 1023, cw + 1024, cw + 1025, cw + 2047, cw + 2048]), keys[:1], 1 + cw % 3, 1)
            e.acceptor_phase2a(p); o.phase2a(p)
        p = votes(np.array([S - 1]), keys[1:2], 2, 0)
        e.acceptor_phase2a(p); o.phase2a(p)
        reqs = [(5, 0), (5, 1), (5, 1000), (6, 1023), (6, 3048), (6, 3049), (7, S - 1), (7, S - 2)]
        dests = [int(dst(0, 0))] * 6 + [int(dst(0, 1))] * 2
        assert acceptor_same(e, o, reqs, np.array(dests, np.int32), a, voffs, keys=keys)[0] == 0


@pytest.mark.parametrize("total", E.SCAN_EDGES)
def test_acceptor_count_scan_chunk(total):
    """n x tiles (record, tile) counters of 4095 / 4096 / 4097: one tile per record at 512 slots"""
    a, voffs = arena_of(VALS)
    keys = [(0, c) for c in range(3)]
    g = np.random.default_rng(total)
    with Engine(1, 1, 3, slot_capacity=512, max_batch=1 << 13) as e:
        o = O.Acceptors(1, 1, 3)
        p = votes(np.sort(g.choice(512, 40, replace=False)), keys, 1, 1)
        e.acceptor_phase2a(p); o.phase2a(p)
        reqs = [(2 + i // 500, int(g.integers(0, 512))) for i in range(total)]
        dests = g.integers(0, 3, total).astype(np.int32)
        assert acceptor_same(e, o, reqs, dests, a, voffs, keys=keys)[0] == 0
    with Engine(1, 1, 3, slot_capacity=16 * E.P1A_TILE, max_batch=1 << 13) as e:     # 17 tiles x 241 = 4097
        o = O.Acceptors(1, 1, 3)
        p = votes(np.sort(g.choice(16 * E.P1A_TILE, 300, replace=False)), keys, 1, 0)
        e.acceptor_phase2a(p); o.phase2a(p)
        n = 241 if total == E.SCAN_CHUNK + 1 else 240
        reqs = [(2 + i // 50, int(g.integers(0, 16 * E.P1A_TILE))) for i in range(n)]
        assert acceptor_same(e, o, reqs, g.integers(0, 3, n).astype(np.int32), a, voffs, keys=keys)[0] == 0


@pytest.mark.parametrize("shape", [(1, 3, 1), (1, 2, 3)], ids=["LG3xAG1", "LG2xAG3"])
def test_mencius_scan_over_the_whole_window(shape):
    """local_slots / (LG * AG) = 1024 with a remainder: residues below it hold 1025 slots, the last in the `+ 1`
    tile; every residue's acceptor answers a Phase1a from slot 0 with votes at its first and last slots"""
    f, lgroups, agroups = shape
    stride = lgroups * agroups
    S = 1024 * stride + stride - 1
    a, voffs = arena_of(VALS)
    with Engine(f, agroups, 3, protocol=MENCIUS, num_leader_groups=lgroups, slot_capacity=S, max_batch=1 << 14) as e:
        o = MO.Acceptors(f, lgroups, agroups)
        keys = [(gr, c) for gr in range(stride) for c in range(3)]
        slots = np.array(sorted({s for r in range(stride) for s in (r, S - 1 - (S - 1 - r) % stride)}))
        grp = (slots % lgroups) * agroups + (slots // lgroups) % agroups
        p = np.zeros(len(slots), O.P2A)
        p["slot"], p["round"], p["value_id"], p["dst"] = slots, 1, 1, dst(grp, 0)
        e.acceptor_phase2a(p); o.phase2a(p)
        reqs = [(3, 0)] * stride
        dests = np.array([int(dst(gr, 0)) for gr in range(stride)], np.int32)
        st, got, _ = acceptor_same(e, o, reqs, dests, a, voffs, mencius=True, keys=keys)
        assert st == 0
        assert max(len(got[0][got[1][i]:got[1][i + 1]]) for i in range(stride)) > 20


def test_acceptor_slid_window_across_the_ring_end():
    S = 1024
    a, voffs = arena_of(VALS)
    keys = [(0, c) for c in range(3)]
    with Engine(1, 1, 3, slot_capacity=S, max_batch=1 << 13) as e:
        o = O.Acceptors(1, 1, 3)
        recs = np.zeros(600, O.P2A)
        recs["slot"] = np.arange(600); recs["round"] = 1; recs["value_id"] = 0
        e.proxyleader_arm(recs)
        acc = np.repeat(recs, 3)
        acc["dst"] = dst(0, np.tile(np.arange(3), 600))
        p2b, _ = e.acceptor_phase2a(acc)
        o.phase2a(acc)
        e.replica_chosen(e.proxyleader_phase2b(p2b))
        assert e.chosen_watermark() == 600           # the scan publishes the executed prefix retire_below checks
        e.retire_below(500)
        p = votes(np.array([1000, 1023, 1024, 1025, 1500, 1523]), keys[:2], 2, 1)
        e.acceptor_phase2a(p); o.phase2a(p)
        reqs = [(3, 500), (3, 1020), (4, 1024), (4, 1523)]
        dests = np.array([int(dst(0, 0))] * 2 + [int(dst(0, 1))] * 2, np.int32)
        assert acceptor_same(e, o, reqs, dests, a, voffs, first_held=500, keys=keys)[0] == 0


def test_acceptor_record_limit():
    """65 535 records (gridDim.y of count and fill) are answered; 65 536 are refused with nothing applied"""
    a, voffs = arena_of(VALS)
    keys = [(0, c) for c in range(3)]
    with Engine(1, 1, 3, slot_capacity=1 << 10, max_batch=1 << 17) as e:
        o = O.Acceptors(1, 1, 3)
        p = votes(np.array([3, 700]), keys, 1, 1)
        e.acceptor_phase2a(p); o.phase2a(p)
        n = E.P1A_MAX_N
        reqs = [(5 if i in (0, n - 1, n - 2) else 2, 0) for i in range(n)]
        dests = (np.arange(n) % 3).astype(np.int32)
        dests[n - 1] = int(dst(0, 1))
        st, got, _ = acceptor_same(e, o, reqs, dests, a, voffs, keys=keys)
        assert st == 0 and got[1][n] > 0
        before = [e.snapshot_acceptor(*k)[0] for k in keys]
        buf, kind, recs = phase1a_batch([(9, 0)] * (n + 1), np.zeros(n + 1, np.int32))
        assert status_of(e.acceptor_phase1a_wire, buf, kind, recs, a, voffs)[0] == E.ERR_INVALID_ARG
        assert [e.snapshot_acceptor(*k)[0] for k in keys] == before


@pytest.mark.parametrize("shape", [(7, 2, 15, 0), (1, 10, 3, 0), (2, 5, 6, 1), (14, 1, 29, 0), ("m", 1, 2, 5),
                                   ("m", 7, 1, 2)], ids=["2x15", "10x3", "flex5x6", "maj29", "LG2AG5", "LG1AG2f7"])
def test_acceptor_thirty_keys(shape):
    """p1a_apply_kernel's one thread per key at its widest: 30 acceptors, the last key 29 included"""
    a, voffs = arena_of(VALS)
    g = np.random.default_rng(len(str(shape)))
    if shape[0] == "m":
        _, f, lgroups, agroups = shape
        e = Engine(f, agroups, 2 * f + 1, protocol=MENCIUS, num_leader_groups=lgroups, slot_capacity=1 << 10,
                   max_batch=1 << 12)
        o = MO.Acceptors(f, lgroups, agroups)
        groups, per, mencius = lgroups * agroups, 2 * f + 1, True
    else:
        f, groups, per, flexible = shape
        e = Engine(f, groups, per, flexible=bool(flexible), slot_capacity=1 << 10, max_batch=1 << 12)
        o = O.Acceptors(f, groups, per, bool(flexible))
        mencius = False
    keys = [(gr, c) for gr in range(groups) for c in range(per)]
    assert len(keys) >= 29                      # a single group holds at most 29 acceptors (2f + 1)
    with e:
        for rnd in range(3):
            picks = list(range(len(keys))) + [int(x) for x in g.integers(0, len(keys), 20)]
            reqs = [(int(g.integers(0, 4)) + 2 * rnd, 0) for _ in picks]
            dests = np.array([int(dst(*keys[k])) for k in picks], np.int32)
            assert acceptor_same(e, o, reqs, dests, a, voffs, mencius=mencius, keys=keys)[0] == 0


@pytest.mark.parametrize("body", E.BODY_EDGES)
def test_phase1b_body_length_widths(body):
    """an acceptor's Phase1b whose body is 127 / 128, 16 383 / 16 384, 2^21 - 1 / 2^21 bytes; then the same reply
    into an output of exactly its size and one byte short"""
    import torch
    dev = torch.device("cuda", 0)
    vlen = E.phase1b_value_len(body, 0, 0, 5, 0, 1)
    a, voffs = arena_of([bytes(vlen)])               # value bytes are copied, not parsed
    outs = []
    for cap_delta in (None, 0, -1):
        with Engine(1, 1, 3, slot_capacity=1 << 10, max_batch=1 << 12) as e:
            o = O.Acceptors(1, 1, 3)
            p = votes(np.array([0]), [(0, 0)], 1, 0)
            e.acceptor_phase2a(p); o.phase2a(p)
            if cap_delta is None:
                st, got, (buf, kind, recs) = acceptor_same(e, o, [(5, 0)], np.array([0], np.int32), a, voffs,
                                                           keys=[(0, 0)])
                assert st == 0 and E.body_len_widths(got[0], got[1]) == {E.width_of(body)}
                need = len(got[0])
                outs.append(bytes(got[0]))
                continue
            d = {k: torch.from_numpy(np.ascontiguousarray(v).view(np.uint8).reshape(-1).copy()).to(dev)
                 for k, v in (("buf", buf), ("kind", kind), ("rec", recs), ("arena", a), ("voffs", voffs))}
            cap = need + cap_delta
            d_out = torch.full((cap + 64,), SENTINEL, dtype=torch.uint8, device=dev)
            d_offs = torch.zeros(2, dtype=torch.int32, device=dev)
            torch.cuda.synchronize()
            st, _, _ = status_of(lambda: (e.acceptor_phase1a_wire_dev(
                d["buf"].data_ptr(), len(buf), d["kind"].data_ptr(), d["rec"].data_ptr(), 1, d["arena"].data_ptr(),
                d["voffs"].data_ptr(), 1, d_out.data_ptr(), cap, d_offs.data_ptr()), e.sync()))
            out = d_out.cpu().numpy()
            if cap_delta == 0:
                assert st == 0 and bytes(out[:need]) == outs[0] and (out[cap:] == SENTINEL).all()
            else:
                # the gathering encoder writes nothing when the replies do not fit; the rounds are those the records
                # left (include/fpx.h fpx_acceptor_phase1a_wire: only malformed bodies, bad voters and retired
                # watermarks change no round)
                assert st == E.ERR_INVALID_ARG and (out == SENTINEL).all()
                assert e.snapshot_acceptor(0, 0)[0] == 5


@pytest.mark.parametrize("rnd", E.ROUND_EDGES)
def test_phase1b_slot_and_round_widths(rnd):
    a, voffs = arena_of(VALS)
    slots = np.array([0, 127, 128, 16383, 16384, (1 << 21) - 1])
    with Engine(1, 1, 3, slot_capacity=(1 << 21) + 8, max_batch=1 << 12) as e:
        o = O.Acceptors(1, 1, 3)
        p = votes(slots, [(0, 0)], 0, 1)
        p["round"] = np.minimum(rnd, [0, 127, 128, 16383, 16384, (1 << 21) - 1])
        e.acceptor_phase2a(p); o.phase2a(p)
        st, got, _ = acceptor_same(e, o, [(rnd, 0), (rnd, 128)], np.array([0, 0], np.int32), a, voffs, keys=[(0, 0)])
        assert st == 0


# --------------------------------------------------------------------------- vanilla Mencius: the walk's chunks
def vm_phase1a(round_, start, stop):
    return E.field(2, E.fint(1, round_) + E.fint(2, start) + E.fint(3, stop))


def vm_value(v, vals):
    return b"\x12\x00" if v == VALUE_NOOP else vals[v]


def vm_reply(server, reply, vals):
    """ServerInbound bytes of the model's reply: Phase1b (member 3) or Phase1Nack (member 8)"""
    if reply[0] == "nack":
        _, start, stop, rnd = reply
        return E.field(8, E.fint(1, start) + E.fint(2, stop) + E.fint(3, rnd))
    _, rnd, start, stop, infos = reply
    body = E.fint(1, server) + E.fint(2, rnd) + E.fint(3, start) + E.fint(4, stop)
    for slot, kind, x, y in infos:
        if kind == "pending":
            inner = E.field(2, E.fint(1, x) + E.field(2, vm_value(y, vals)))
        else:
            inner = E.field(3, E.field(1, vm_value(x, vals)) + E.fint(2, int(y)))
        body += E.field(5, E.fint(1, slot) + inner)
    return E.field(3, body)


def vm_run(eng, model, reqs, next_slot, vals, arena, voffs):
    """reqs [(receiving server, round, start, stop)] -> compares replies, skips and next_slot with the model"""
    msgs = [vm_phase1a(r, a, b) for _, r, a, b in reqs]
    buf, offs = O.pack(msgs)
    kind, rec, _ = eng.wire_decode_vm_server_inbound(buf, offs)
    rec = rec.copy()
    rec["a"] = [s for s, _, _, _ in reqs]
    replies, skips = eng.vm_phase1a_wire(buf, kind, rec, next_slot, arena, voffs)
    for i, (s, r, a, b) in enumerate(reqs):
        want, skip = model[s].phase1a(r, a, b)
        assert replies[i] == vm_reply(s, want, vals), (i, want[0])
        if skip is not None:
            assert (int(skips[i]["slot_start"]), int(skips[i]["slot_stop"])) == skip
    assert next_slot.tolist() == [m.next_slot for m in model]


def vm_check(eng, model, upto):
    for s, m in enumerate(model):
        got = eng.vm_entries(s, 0, upto)
        want = np.array([m.entry_row(x) for x in range(upto)], dtype=np.int32)
        bad = np.nonzero((got != want).any(axis=1))[0]
        assert len(bad) == 0, (s, int(bad[0]), got[bad[0]].tolist(), want[bad[0]].tolist())


VM_VALS = [b"\x0a\x00", b"\x0a\x03\x0a\x01z"]


@pytest.mark.parametrize("stale_at", [0, 255, 256, 257, -1, None], ids=["k0", "k255", "k256", "k257", "last", "none"])
@pytest.mark.parametrize("count", [255, 256, 257, 513])
def test_vm_walk_chunks(count, stale_at):
    """server 1 answers a revocation of `count` of server 0's slots; one entry is stale (round above the Phase1a's) at
    k, or none: the raise before it is kept across the earlier chunks, the later chunks untouched"""
    n = 3
    arena, voffs = arena_of(VM_VALS)
    with Engine(1, 1, n, slot_capacity=2048, max_batch=1 << 12, protocol=VANILLA_MENCIUS) as eng:
        model = [Server(s, n) for s in range(n)]
        next_slot = np.array([3 * count + s for s in range(n)], np.int32)
        for s in range(n):
            model[s].next_slot = int(next_slot[s])
        k = np.arange(0, count, 3)
        p2a = [(int(3 * x), 0, int(x % 2), 1) for x in k]
        if stale_at is not None:
            at = stale_at % count
            p2a = [r for r in p2a if r[0] != 3 * at] + [(3 * at, 9, 1, 1)]
        eng.vm_phase2a(np.array(p2a, dtype=P2A))
        for r in p2a:
            model[1].phase2a(r[0], r[1], r[2])
        eng.vm_choose(np.array([(1, 1, 3 * 7, 0)], dtype=P2B)); model[1].choose(21, 0, True)
        vm_run(eng, model, [(1, 5, 0, 3 * count), (1, 4, 0, 3 * count)], next_slot, VM_VALS, arena, voffs)
        vm_check(eng, model, 3 * count + 6)


@pytest.mark.parametrize("fills", [255, 256, 257])
def test_vm_self_revocation_fill(fills):
    n = 3
    with Engine(1, 1, n, slot_capacity=2048, max_batch=1 << 12, protocol=VANILLA_MENCIUS) as eng:
        model = [Server(s, n) for s in range(n)]
        next_slot = np.array([0, 1, 2], np.int32)
        vm_run(eng, model, [(2, 4, 2, 2 + 3 * fills), (2, 6, 2 + 3 * fills, 2 + 3 * fills + 4)], next_slot, [],
               *arena_of([b"\x0a\x00"]))
        vm_check(eng, model, 3 * fills + 12)


def test_vm_many_phase1a_records():
    """more than SCAN_CHUNK Phase1a records: their walked-slot counts span two chunks of the count scan"""
    n = 3
    g = np.random.default_rng(4)
    arena, voffs = arena_of(VM_VALS)
    with Engine(1, 1, n, slot_capacity=1 << 12, max_batch=1 << 14, protocol=VANILLA_MENCIUS) as eng:
        model = [Server(s, n) for s in range(n)]
        next_slot = np.array([3000, 3001, 3002], np.int32)
        for s in range(n):
            model[s].next_slot = int(next_slot[s])
        p2a = np.array([(int(x), int(g.integers(0, 3)), int(x % 2), int(g.integers(0, n))) for x in range(0, 600, 2)],
                       dtype=P2A)
        eng.vm_phase2a(p2a)
        for r in p2a:
            model[int(r["dst"])].phase2a(int(r["slot"]), int(r["round"]), int(r["value_id"]))
        reqs = []
        for i in range(E.SCAN_CHUNK + 1):
            rv = int(g.integers(0, 2))
            start = rv + 3 * int(g.integers(0, 190))
            reqs.append((int(g.integers(0, n)), 1 + i // 800, start, start + int(g.integers(0, 30))))
        vm_run(eng, model, reqs, next_slot, VM_VALS, arena, voffs)
        vm_check(eng, model, 640)


def test_vm_range_across_the_ring_wrap():
    from frankenpaxos_b200 import CHOSEN
    n = 3
    cap = 1024
    with Engine(1, 1, n, slot_capacity=cap, max_batch=1 << 12, protocol=VANILLA_MENCIUS) as eng:
        model = [Server(s, n) for s in range(n)]
        eng.replica_chosen(np.array([(s, VALUE_NOOP) for s in range(300)], dtype=CHOSEN))
        assert eng.chosen_watermark() >= 300
        eng.retire_below(300)
        next_slot = np.array([3000, 3001, 3002], np.int32)
        for s in range(n):
            model[s].next_slot = int(next_slot[s])
        arena, voffs = arena_of(VM_VALS)
        # votes and chosen entries on both sides of the ring's end, on the residues the two walks read: server 0's
        # slots (993 + 3k) at server 2, server 1's (301 + 3k) at server 0
        p2a = np.array([(s, 1, s % 2, 2) for s in range(cap - 31, cap + 60, 3)] +
                       [(s, 2, s % 2, 0) for s in range(cap - 24, cap + 60, 6)], dtype=P2A)
        eng.vm_phase2a(p2a)
        for r in p2a:
            model[int(r["dst"])].phase2a(int(r["slot"]), int(r["round"]), int(r["value_id"]))
        ch = np.array([(1, 2, cap - 1, 0), (0, 2, cap + 2, VALUE_NOOP), (1, 0, cap + 3, 1)], dtype=P2B)
        eng.vm_choose(ch)
        for rev, s, slot, v in ch.tolist():
            model[s].choose(slot, v, rev)
        start = cap - 31
        vm_run(eng, model, [(2, 4, start, start + 300), (0, 4, 301, cap + 299)], next_slot, VM_VALS, arena, voffs)
        for s in (0, 2):
            got = eng.vm_entries(s, 301, cap - 2)
            want = np.array([model[s].entry_row(x) for x in range(301, cap + 299)], dtype=np.int32)
            assert np.array_equal(got, want), s


@pytest.mark.parametrize("body", E.BODY_EDGES)
def test_vm_phase1b_body_length_widths(body):
    """VmP1bCodec: server 1's Phase1b of one pending info whose body is 127 / 128, 16 383 / 16 384, 2^21 - 1 / 2^21
    bytes, into an output of exactly its size and of one byte less"""
    import torch
    dev = torch.device("cuda", 0)
    n, rnd = 3, 5
    vlen = E.vm_phase1b_value_len(body, 1, rnd, 0, 3, 0, 0)
    vals = [bytes(vlen)]                             # value bytes are copied, not parsed
    arena, voffs = arena_of(vals)

    def dev_of(x):
        return torch.from_numpy(np.ascontiguousarray(x).view(np.uint8).reshape(-1).copy()).to(dev)
    for short in (False, True):
        with Engine(1, 1, n, slot_capacity=1 << 10, max_batch=1 << 12, protocol=VANILLA_MENCIUS) as eng:
            model = [Server(s, n) for s in range(n)]
            eng.vm_phase2a(np.array([(0, 0, 0, 1)], dtype=P2A))
            model[1].phase2a(0, 0, 0)
            before = eng.vm_entries(1, 0, 3).copy()
            # refused before anything is applied: a walk past the live window in the same batch
            buf, offs = O.pack([vm_phase1a(rnd, 0, 3), vm_phase1a(rnd, 0, (1 << 10) + 3)])
            kind, rec, _ = eng.wire_decode_vm_server_inbound(buf, offs)
            rec = rec.copy()
            rec["a"] = 1
            assert status_of(eng.vm_phase1a_wire, buf, kind, rec, np.array([0, 1, 2], np.int32), arena,
                             voffs)[:2] == (E.ERR_SLOT_RANGE, 1)
            assert np.array_equal(eng.vm_entries(1, 0, 3), before)
            want, _ = model[1].phase1a(rnd, 0, 3)
            reply = vm_reply(1, want, vals)
            assert E.body_len_widths(np.frombuffer(reply, np.uint8), [0, len(reply)]) == {E.width_of(body)}
            cap = len(reply) - short
            d_buf, d_kind, d_rec, d_arena, d_voffs = (dev_of(x) for x in (buf, kind[:1], rec[:1], arena, voffs))
            d_ns = dev_of(np.array([0, 1, 2], np.int32))
            d_out = torch.full((cap + 64,), SENTINEL, dtype=torch.uint8, device=dev)
            d_offs = torch.zeros(2, dtype=torch.int32, device=dev)
            d_skips = torch.zeros(4, dtype=torch.int32, device=dev)
            torch.cuda.synchronize()
            st, idx, _ = status_of(lambda: (eng.vm_phase1a_wire_dev(
                d_buf.data_ptr(), len(buf), d_kind.data_ptr(), d_rec.data_ptr(), 1, d_arena.data_ptr(),
                d_voffs.data_ptr(), 1, d_ns.data_ptr(), d_out.data_ptr(), cap, d_offs.data_ptr(), d_skips.data_ptr()),
                eng.sync()))
            out = d_out.cpu().numpy()
            assert d_ns.cpu().numpy().view(np.int32).tolist() == [0, 1, 2]
            if short:
                # include/fpx.h fpx_vm_phase1a_wire: replies longer than out_capacity are found after the entries
                # are raised; nothing is written
                assert (st, idx) == (E.ERR_INVALID_ARG, 0) and (out == SENTINEL).all()
            else:
                assert st == 0 and out[:cap].tobytes() == reply and (out[cap:] == SENTINEL).all()
                assert d_offs.cpu().tolist() == [0, len(reply)]
            vm_check(eng, model, 6)


def test_acceptor_phase1b_past_the_scan_chunk():
    """one acceptor's Phase1b of 4 195 329 infos: more than SCAN_CHUNK x ENC_TILE records through P1bCodec"""
    n = E.BIG_P2A
    a, voffs = arena_of(VALS)
    with Engine(1, 1, 3, slot_capacity=n + 16, max_batch=1 << 23) as e:
        o = O.Acceptors(1, 1, 3)
        p = votes(np.arange(n), [(0, 0)], 1, 0)
        p["value_id"][::3] = VALUE_NOOP
        e.acceptor_phase2a(p); o.phase2a(p)
        st, got, _ = acceptor_same(e, o, [(4, 0), (3, 0)], np.array([0, 0], np.int32), a, voffs, keys=[(0, 0)])
        assert st == 0 and got[1][1] > 10 * n
