"""GPU parity of the leader's Phase-1 wire path (fpx_leader_phase1b_wire, fpx_wire_encode_phase2a) against the golden
vectors and the CPU oracle (tests/wire_phase1_oracle.cc), and the leader change end to end at 2^20 slots in flight."""
import numpy as np
import pytest

import wire_phase1_cases as W
import wire_phase1_oracle as O
from frankenpaxos_b200 import MENCIUS, WIRE_PROXYLEADER_INBOUND, Engine, FpxError, VALUE_NOOP, dst

pytestmark = pytest.mark.gpu


def status_of(fn, *a, **kw):
    try:
        return 0, -1, fn(*a, **kw)
    except FpxError as e:
        return e.status, e.index, None


def same_leader(eng, f, groups, per_group, flexible, round_, cw, msgs, base=0, cap=1 << 12, buf=None, offs=None):
    if buf is None:
        buf, offs = O.pack(msgs)
    o = O.leader_phase1b(f, groups, per_group, flexible, round_, cw, buf, offs, base, cap)
    st, idx, got = status_of(eng.leader_phase1b_wire, round_, cw, buf, offs, base, cap)
    assert (st, idx) == (o[0], o[1])
    if st == 0:
        complete, max_slot, recs, spans = got
        assert (complete, max_slot) == (o[2], o[3])
        assert np.array_equal(recs.view(np.int32), o[4].view(np.int32)) and np.array_equal(spans, o[5])
    return o, buf


@pytest.fixture(scope="module")
def eng():
    e = Engine(W.F, W.GROUPS, W.PER_GROUP, slot_capacity=1 << 12, max_batch=1 << 12)
    yield e
    e.close()


def test_golden_decode_and_encode(eng):
    for case in W.GOLD["decode"]:
        msgs, round_ = W.golden_batch(case)
        same_leader(eng, W.F, W.GROUPS, W.PER_GROUP, 0, round_, 0, msgs, 40)
    for case in W.GOLD["phase2a"]:
        payload = np.frombuffer(bytes.fromhex(case["payload_hex"]), np.uint8).copy()
        rec = np.zeros(1, O.P2A)
        rec["slot"], rec["round"], rec["dst"] = case["slot"], case["round"], 7
        rec["value_id"] = VALUE_NOOP if case["noop"] else 3
        out, offs = eng.wire_encode_phase2a(rec, payload, [[0, len(payload)]], 3)
        assert bytes(out) == bytes.fromhex(case["hex"]) and list(offs) == [0, len(out)]


@pytest.mark.parametrize("shape", [(1, 1, 3, 0), (1, 2, 3, 0), (1, 2, 3, 1), (2, 1, 5, 0)])
def test_random_batches_against_oracle(shape):
    f, groups, per_group, flexible = shape
    g = np.random.Generator(np.random.PCG64(7 + groups * 10 + flexible))
    a, voffs = W.arena(g, 64)
    with Engine(f, groups, per_group, flexible=bool(flexible), slot_capacity=1 << 12, max_batch=1 << 12) as e:
        for _ in range(40):
            msgs = W.random_phase1b_batch(g, groups, per_group, 9, 300, int(g.integers(1, 14)), a, voffs)
            same_leader(e, f, groups, per_group, flexible, 9, int(g.integers(0, 350)), msgs, int(g.integers(0, 1000)))
        # Phase2a of the last records, host form against the oracle
        msgs = W.random_phase1b_batch(g, groups, per_group, 9, 300, 12, a, voffs, extra=False)
        buf, offs = O.pack(msgs)
        o = O.leader_phase1b(f, groups, per_group, flexible, 9, 0, buf, offs, 100, 1 << 12)
        if o[0] == 0 and len(o[4]):
            ost, _, ob, ooffs = O.encode_phase2a(o[4], buf, o[5], 100)
            hb, hoffs = e.wire_encode_phase2a(o[4], buf, o[5], 100)
            assert ost == 0 and bytes(hb) == bytes(ob) and np.array_equal(hoffs, ooffs)


def test_flexible_row_differs_from_safe_values():
    """A 2x3 grid: the reference's fill-in reads phase1bs(slot % rows) only; fpx_leader_safe_values takes every
    responder.  Row 1 holds the higher vote of slot 0, row 0 is the full row that completes the read quorum."""
    a = np.frombuffer(b"\x0a\x00AB", np.uint8).copy()
    voffs = np.array([0, 2, 4], np.int32)
    low = [O.encode_phase1b(0, c, 4, [0], [1], [0], a, voffs) for c in range(3)]
    high = O.encode_phase1b(1, 0, 4, [0], [3], [1], a, voffs)
    msgs = [high] + low
    with Engine(1, 2, 3, flexible=True, slot_capacity=1 << 10, max_batch=1 << 10) as e:
        o, buf = same_leader(e, 1, 2, 3, 1, 4, 0, msgs)
        assert o[2] == 3 and len(o[4]) == 1
        k = o[5][0]
        assert bytes(buf[k[0]: k[0] + k[1]]) == b"\x0a\x00"            # row 0's vote (round 1), not row 1's (round 3)
        # the same votes in the engine's cells: fpx_leader_safe_values answers round 3
        p2a = np.zeros(4, O.P2A)
        p2a["slot"], p2a["round"], p2a["value_id"] = 0, [1, 1, 1, 3], [10, 10, 10, 11]
        p2a["dst"] = dst([0, 0, 0, 1], [0, 1, 2, 0])
        e.acceptor_phase2a(p2a[:3])
        e.acceptor_phase2a(p2a[3:])
        vr, vv, _ = e.leader_safe_values(0b1111, 0, 1)
        assert vr[0] == 3 and vv[0] == 11


def test_device_forms_capacity_and_mutations(eng):
    import torch
    dev = torch.device("cuda", 0)
    g = np.random.Generator(np.random.PCG64(31))
    a, voffs = W.arena(g, 32)
    msgs = W.random_phase1b_batch(g, 2, 3, 9, 2000, 10, a, voffs, extra=False)
    msgs += [W.empty_phase1b(gr, c, 9) for gr in range(2) for c in range(3)]
    buf, offs = O.pack(msgs)
    complete, max_slot, recs, spans = eng.leader_phase1b_wire(9, 5, buf, offs, 50, 4096)
    assert complete >= 0 and len(recs) == max_slot - 4
    # device form
    d_buf, d_offs = torch.from_numpy(buf).to(dev), torch.from_numpy(offs).to(dev)
    d_out, d_sp, d_res = (torch.zeros(s, dtype=torch.int32, device=dev) for s in ((4096, 4), (4096, 2), (3,)))
    torch.cuda.synchronize()
    eng.leader_phase1b_wire_dev(9, 5, d_buf.data_ptr(), len(buf), d_offs.data_ptr(), len(msgs), 50, d_out.data_ptr(),
                                d_sp.data_ptr(), 4096, d_res.data_ptr())
    eng.sync()
    assert d_res.cpu().tolist() == [complete, max_slot, len(recs)]
    assert np.array_equal(d_out[:len(recs)].cpu().numpy().reshape(-1), recs.view(np.int32).reshape(-1))
    assert np.array_equal(d_sp[:len(recs)].cpu().numpy(), spans)
    hb, hoffs = eng.wire_encode_phase2a(recs, buf, spans, 50)
    d_recs = torch.from_numpy(recs.view(np.int32).reshape(-1, 4).copy()).to(dev)
    d_bytes = torch.zeros(len(hb) + 64, dtype=torch.uint8, device=dev)
    d_o = torch.zeros(len(recs) + 1, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    eng.wire_encode_phase2a_dev(d_recs.data_ptr(), len(recs), d_buf.data_ptr(), len(buf), d_sp.data_ptr(), len(recs), 50,
                                d_bytes.data_ptr(), len(d_bytes), d_o.data_ptr())
    eng.sync()
    assert np.array_equal(d_o.cpu().numpy(), hoffs) and bytes(d_bytes[:len(hb)].cpu().numpy()) == bytes(hb)
    # one record / one byte short: refused, nothing written
    st, idx, _ = status_of(eng.leader_phase1b_wire, 9, 5, buf, offs, 50, len(recs) - 1)
    assert (st, idx) == (-1, complete)
    n = len(recs)
    out = np.zeros(len(hb) - 1, np.uint8)
    o2 = np.zeros(n + 1, np.int32)
    st = eng._L.fpx_wire_encode_phase2a(eng.h, recs.ctypes.data, n, buf.ctypes.data, len(buf), spans.ctypes.data, n, 50,
                                        out.ctypes.data, len(out), o2.ctypes.data, None)
    assert st == -1 and not out.any()
    # 300 mutations of Phase1b bytes: status and first index as the oracle's
    small = W.random_phase1b_batch(g, 2, 3, 9, 40, 8, a, voffs, extra=False)
    for _ in range(300):
        i = int(g.integers(0, len(small)))
        raw = bytearray(small[i])
        kind = int(g.integers(0, 3))
        if kind == 0 and raw:
            raw[int(g.integers(0, len(raw)))] = int(g.integers(0, 256))
        elif kind == 1 and raw:
            del raw[int(g.integers(0, len(raw))):]
        else:
            p = int(g.integers(0, len(raw) + 1))
            raw[p:p] = bytes(g.integers(0, 256, size=int(g.integers(1, 4)), dtype=np.uint8))
        batch = small[:i] + [bytes(raw)] + small[i + 1:]
        same_leader(eng, W.F, W.GROUPS, W.PER_GROUP, 0, 9, 0, batch, 3)


def test_spans_many_encode_tiles(eng):
    """One Phase1b of 5000 infos (many walk windows) and the Phase2a of its 5000 slots (five encode tiles)."""
    g = np.random.Generator(np.random.PCG64(77))
    a, voffs = W.arena(g, 100)
    n = 4000
    big = [O.encode_phase1b(gr, c, 9, np.arange(gr, n, 2), np.full(len(range(gr, n, 2)), 8),
                            g.integers(0, 100, len(range(gr, n, 2))), a, voffs) for gr in range(2) for c in range(2)]
    o, buf = same_leader(eng, W.F, W.GROUPS, W.PER_GROUP, 0, 9, 0, big, 0, 4096)
    assert o[2] == 3 and len(o[4]) == n
    hb, hoffs = eng.wire_encode_phase2a(o[4], buf, o[5], 0)
    ost, _, ob, ooffs = O.encode_phase2a(o[4], buf, o[5], 0)
    assert ost == 0 and bytes(hb) == bytes(ob) and np.array_equal(hoffs, ooffs)


def test_unsupported():
    with Engine(1, 1, 3, protocol=MENCIUS, num_leader_groups=1, slot_capacity=1 << 10, max_batch=1 << 10) as e:
        buf, offs = O.pack([W.empty_phase1b(0, 0, 1)])
        assert status_of(e.leader_phase1b_wire, 1, 0, buf, offs)[0] == -11
    with Engine(1, 1, 3, slot_capacity=1 << 10, max_batch=1 << 10, shard_count=2) as e:
        assert status_of(e.leader_phase1b_wire, 1, 0, buf, offs)[0] == -11


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_leader_change_end_to_end_2e20(seed):
    """cfg2's shape (f = 2, one group of five) with 2^20 slots in flight: three acceptors' votes, their Phase1b bytes
    from Phase1a bytes, the new leader's call, its Phase2a bytes decoded again, then arm -> acceptor -> tally; the
    Phase1b bytes, the Chosen stream and the log carry exactly the oracle's values."""
    g = np.random.Generator(np.random.PCG64(seed))
    S = 1 << 20
    a, voffs = W.arena(g, 4096)
    o = O.Acceptors(2, 1, 5)
    with Engine(2, 1, 5, slot_capacity=1 << 21, max_batch=1 << 22, overflow_capacity=1 << 14) as e:
        votes = []
        for c in range(3):
            voted = np.nonzero(g.random(S) < 0.9)[0].astype(np.int32)
            p = np.zeros(len(voted), O.P2A)
            p["slot"], p["round"], p["dst"] = voted, g.integers(0, 7, len(voted)), dst(0, c)
            p["value_id"] = np.where(g.random(len(voted)) < 0.05, VALUE_NOOP, g.integers(0, 4096, len(voted)))
            votes.append(p)
        p = np.concatenate(votes)
        e.acceptor_phase2a(p)
        o.phase2a(p)
        # Phase1a{round 7, chosen_watermark 0} to acceptors 0, 1, 2 -> their Phase1b bytes
        req, roffs = O.pack([phase1a(7, 0)] * 3)
        kind, recs1a = e.wire_decode_inbound(1, req, roffs)
        recs1a = recs1a.copy()
        recs1a["a"] = dst(0, np.arange(3))
        ost, _, ob, _ = o.phase1a_wire(0, req, kind, recs1a, a, voffs)
        p1b, p1offs = e.acceptor_phase1a_wire(req, kind, recs1a, a, voffs)
        assert ost == 0 and bytes(p1b) == bytes(ob)
        msgs = O.split(p1b, p1offs)
        o2, buf = same_leader(e, 2, 1, 5, 0, 7, 0, msgs, 0, S)
        recs, spans = o2[4], o2[5]
        assert o2[2] == 2 and len(recs) == o2[3] + 1
        p2a, poffs = e.wire_encode_phase2a(recs, buf, spans, 0)
        ost, _, ob, _ = O.encode_phase2a(recs, buf, spans, 0)
        assert ost == 0 and bytes(p2a) == bytes(ob)
        kind, dec = e.wire_decode_inbound(WIRE_PROXYLEADER_INBOUND, p2a, poffs)
        assert (kind == 1).all() and np.array_equal(dec["a"], recs["slot"]) and np.array_equal(dec["b"], recs["round"])
        e.proxyleader_arm(recs)
        acc = np.repeat(recs, 3)
        acc["dst"] = dst(0, np.tile(np.arange(3), len(recs)))
        p2b, nack = e.acceptor_phase2a(acc)
        assert len(nack) == 0 and len(p2b) == len(acc)
        chosen = e.proxyleader_phase2b(p2b)
        assert np.array_equal(np.sort(chosen["slot"]), recs["slot"])
        want = dict(zip(recs["slot"].tolist(), recs["value_id"].tolist()))
        assert all(want[s] == v for s, v in zip(chosen["slot"].tolist(), chosen["value_id"].tolist()))
        e.replica_chosen(chosen)
        assert np.array_equal(e.snapshot_log(0, len(recs)), recs["value_id"])


# ---- the acceptor's side: Phase1a bytes in, Phase1b / Nack bytes out
# canonical CommandBatchOrNoops, which the runtime re-serializes unchanged: Noop, an empty batch, one command
_CMD_ID = b"\x0a\x01a\x10\x01\x18\x01"
_CMD = b"\x0a" + bytes([len(_CMD_ID)]) + _CMD_ID + b"\x12\x02xy"
_BATCH = b"\x0a" + bytes([len(_CMD)]) + _CMD
VALUES = [b"\x0a\x00", b"\x0a" + bytes([len(_BATCH)]) + _BATCH]


def value_arena():
    a = np.frombuffer(b"".join(VALUES), np.uint8).copy()
    return a, np.concatenate([[0], np.cumsum([len(v) for v in VALUES])]).astype(np.int32)


def _varint(v):
    v &= (1 << 64) - 1
    out = b""
    while v >= 0x80:
        out += bytes([(v & 0x7f) | 0x80]); v >>= 7
    return out + bytes([v])


def phase1a(round_, cw):
    body = b"\x08" + _varint(round_) + b"\x10" + _varint(cw)
    return b"\x0a" + bytes([len(body)]) + body      # AcceptorInbound{phase1a = 1}


def runtime():
    import importlib.util
    import os
    spec = importlib.util.spec_from_file_location("mk", os.path.join(W.HERE, "golden", "make_wire_phase1_golden.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    return mk


def trace(g, e, o, groups, per_group, flexible, n_slots, batches=3, size=2000):
    """Random Phase2a batches through the engine's acceptors and the oracle's."""
    for _ in range(batches):
        p2a = np.zeros(size, O.P2A)
        p2a["slot"] = g.integers(0, n_slots, size)
        p2a["round"] = g.integers(0, 6, size)
        p2a["value_id"] = np.where(g.random(size) < 0.2, VALUE_NOOP, g.integers(0, len(VALUES), size))
        grp = g.integers(0, groups, size) if flexible else p2a["slot"] % groups
        p2a["dst"] = dst(grp, g.integers(0, per_group, size))
        e.acceptor_phase2a(p2a)
        o.phase2a(p2a)


def same_acceptor(e, o, msgs, dests, first_held=0, mk=None):
    a, voffs = value_arena()
    buf, offs = O.pack(msgs)
    kind, recs = e.wire_decode_inbound(1, buf, offs)           # WIRE_ACCEPTOR_INBOUND
    recs = recs.copy()
    recs["a"] = dests
    ost, oidx, ob, ooffs = o.phase1a_wire(first_held, buf, kind, recs, a, voffs)
    st, idx, got = status_of(e.acceptor_phase1a_wire, buf, kind, recs, a, voffs)
    assert (st, idx) == (ost, oidx)
    if st == 0:
        gb, goffs = got
        assert bytes(gb) == bytes(ob) and np.array_equal(goffs, ooffs)
        if mk is not None:
            for raw in O.split(gb, goffs):
                if raw:
                    m = mk.cls("LeaderInbound")()
                    m.ParseFromString(raw)
                    assert m.SerializeToString() == raw
    for gr in range(o.groups):
        for c in range(o.per_group):
            assert e.snapshot_acceptor(gr, c)[0] == o.round(gr, c)
    return st


@pytest.mark.parametrize("shape", [(1, 1, 3, 0), (2, 1, 5, 0), (1, 2, 3, 1)], ids=["cfg1", "cfg2", "grid2x3"])
def test_acceptor_phase1a_against_oracle(shape):
    f, groups, per_group, flexible = shape
    g = np.random.Generator(np.random.PCG64(50 + groups + f))
    mk = runtime()
    S = 3000
    with Engine(f, groups, per_group, flexible=bool(flexible), slot_capacity=1 << 13, max_batch=1 << 13) as e:
        o = O.Acceptors(f, groups, per_group, flexible)
        trace(g, e, o, groups, per_group, flexible, S)
        keys = [(gr, c) for gr in range(groups) for c in range(per_group)]
        for rnd in range(12):
            msgs, dests = [], []
            for _ in range(int(g.integers(1, 12))):
                gr, c = keys[int(g.integers(0, len(keys)))]
                cw = int(g.choice([0, S // 2, S + 50, int(g.integers(0, S))]))
                msgs.append(phase1a(int(g.integers(0, 4)) + rnd // 3 * 2, cw))          # stale ones and repeats
                dests.append(int(dst(gr, c)))
            if g.random() < 0.3:                                 # another member: a zero-length reply
                msgs.insert(0, bytes.fromhex("1208080110021a021200"))
                dests.insert(0, 0)
            same_acceptor(e, o, msgs, np.array(dests, np.int32), 0, mk)
        # a malformed body and a non-member refuse the call; no round changes
        assert same_acceptor(e, o, [phase1a(9, 0), b"\x0a\x02\x08\x01"], np.array([0, 1], np.int32)) == -15
        assert same_acceptor(e, o, [phase1a(9, 0)], np.array([int(dst(groups, 0))], np.int32)) == -1


def test_acceptor_phase1a_below_retired_base():
    g = np.random.Generator(np.random.PCG64(3))
    with Engine(1, 1, 3, slot_capacity=1 << 10, max_batch=1 << 12) as e:
        o = O.Acceptors(1, 1, 3)
        recs = np.zeros(200, O.P2A)
        recs["slot"] = np.arange(200); recs["round"] = 1; recs["value_id"] = g.integers(0, 2, 200)
        e.proxyleader_arm(recs)
        acc = np.repeat(recs, 3)
        acc["dst"] = dst(0, np.tile(np.arange(3), 200))
        p2b, _ = e.acceptor_phase2a(acc)
        o.phase2a(acc)
        e.replica_chosen(e.proxyleader_phase2b(p2b))
        assert e.chosen_watermark() == 200
        e.retire_below(128)
        d = np.array([int(dst(0, 1))], np.int32)
        assert same_acceptor(e, o, [phase1a(5, 3)], d, 128) == -6           # SLOT_RANGE, nothing applied
        assert e.snapshot_acceptor(0, 1)[0] == 1
        assert same_acceptor(e, o, [phase1a(5, 128)], d, 128) == 0
        assert same_acceptor(e, o, [phase1a(6, 150)], d, 128) == 0
