"""GPU wire codec of Compartmentalized Mencius' noop ranges and replica, and the replica's mixed Chosen /
ChosenNoopRange call (fpx_mencius_replica_inbound): the golden vectors, the CPU oracle (tests/wire_mencius_oracle.cc),
the device forms against the host forms, the codec's window / chunk / capacity edges, and protobuf bytes through the
acceptor, the proxy leader and the replica end to end."""
import ctypes as C
import json
import os
import sys

import numpy as np
import pytest
import torch

from frankenpaxos_b200 import (CHOSEN, CHOSEN_RANGE, MENCIUS, MENCIUS_CHOSEN, NACK, P2A_RANGE, P2B_RANGE, VALUE_NOOP,
                               WIRE_MENCIUS_PROXYLEADER_INBOUND, Engine, FpxError)
import wire_mencius_oracle as O

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import make_wire_mencius_golden as M  # noqa: E402

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
CASES = json.load(open(os.path.join(HERE, "golden", "wire_mencius.json")))["cases"]
WIRE, SLOT_RANGE, UNSUPPORTED, INVALID_ARG = -15, -6, -11, -1
LG, AG, PER = 3, 3, 3


def of_type(t):
    return [c for c in CASES if c["type"] == t]


def mencius(lg=LG, ag=AG, **kw):
    kw.setdefault("slot_capacity", 1 << 14)
    kw.setdefault("max_batch", 1 << 14)
    return Engine(1, ag, PER, num_leaders=2, num_replicas=2, protocol=MENCIUS, num_leader_groups=lg, **kw)


@pytest.fixture(scope="module")
def eng():
    e = mencius()
    yield e
    e.close()


def same_decode(eng, buf, offs, base=0):
    """Engine and oracle agree: status, first offending index, and every row."""
    st, err, okind, orecs, ovals = O.decode(buf, offs, base)
    try:
        kind, recs, vals = eng.wire_decode_mencius_replica_inbound(buf, offs, base)
        est, eidx = 0, -1
    except FpxError as e:
        est, eidx = e.status, e.index
    assert (est, eidx) == (st, err)
    if st == 0:
        assert np.array_equal(kind, okind) and np.array_equal(vals, ovals)
        assert np.array_equal(recs.view(np.int32), orecs.view(np.int32))
    return st


def test_decode_golden(eng):
    cs = of_type("chosen") + of_type("chosen_noop_range")
    buf, offs = O.pack([bytes.fromhex(c["hex"]) for c in cs])
    assert same_decode(eng, buf, offs, base=7) == 0
    kind, recs, vals = eng.wire_decode_mencius_replica_inbound(buf, offs, 7)
    for i, c in enumerate(cs):
        if c["type"] == "chosen":
            assert kind[i] == 1 and recs[i]["slot_start"] == c["slot"] and recs[i]["value_id"] == 7 + i
            assert bytes(buf[vals[i][0]: vals[i][0] + vals[i][1]]).hex() == c["value_hex"]
        else:
            assert kind[i] == 2 and (recs[i]["slot_start"], recs[i]["slot_end"], recs[i]["value_id"]) == \
                (c["start"], c["end"], VALUE_NOOP)
    for c in of_type("robustness"):
        same_decode(eng, *O.pack([bytes.fromhex(c["hex"])]))


def test_encode_golden(eng):
    cr = of_type("chosen_noop_range")
    out, offs = eng.wire_encode_mencius_chosen_range(np.array([(c["start"], c["end"]) for c in cr], dtype=CHOSEN_RANGE))
    assert [bytes(out[offs[i]: offs[i + 1]]).hex() for i in range(len(cr))] == [c["hex"] for c in cr]
    nk = of_type("nack")
    out, offs = eng.wire_encode_nack(np.array([(1, c["round"]) for c in nk], dtype=NACK))
    assert [bytes(out[offs[i]: offs[i + 1]]).hex() for i in range(len(nk))] == [c["hex"] for c in nk]
    pr = [c for c in of_type("phase2b_noop_range") if 0 <= c["acceptor_group_index"] < AG]
    recs = np.array([((c["acceptor_group_index"] << 16) | (c["acceptor_index"] & 0xffff), c["start"], c["end"], c["round"])
                     for c in pr if 0 <= c["acceptor_index"] < 0x10000], dtype=P2B_RANGE)
    want = [c["hex"] for c in pr if 0 <= c["acceptor_index"] < 0x10000]
    out, offs = eng.wire_encode_mencius_phase2b_range(recs)
    assert [bytes(out[offs[i]: offs[i + 1]]).hex() for i in range(len(recs))] == want


def test_mencius_nack_is_leader_inbound_nack(eng):
    """On a Mencius engine the Nack is LeaderInbound.nack = 7: field 6 is leader_info_request_batcher."""
    rounds = [0, 1, 127, 128, 1 << 20, (1 << 31) - 1, -1, -(1 << 31)]
    out, offs = eng.wire_encode_nack(np.array([(0, r) for r in rounds], dtype=NACK))
    LI = M.mcls("LeaderInbound")
    for i, r in enumerate(rounds):
        m = LI()
        m.ParseFromString(bytes(out[offs[i]: offs[i + 1]]))
        assert m.WhichOneof("request") == "nack" and m.nack.round == r
        assert bytes(out[offs[i]: offs[i + 1]]) == LI(nack=M.mcls("Nack")(round=r)).SerializeToString()


def test_other_protocols_refuse(eng):
    mp = Engine(1, 1, 3, slot_capacity=64, max_batch=64)
    for call in (lambda: mp.wire_encode_mencius_chosen_range(np.zeros(1, dtype=CHOSEN_RANGE)),
                 lambda: mp.wire_encode_mencius_phase2b_range(np.zeros(1, dtype=P2B_RANGE)),
                 lambda: mp.wire_decode_mencius_replica_inbound(np.zeros(16, dtype=np.uint8), np.array([0, 2], np.int32)),
                 lambda: mp.mencius_replica_inbound(np.zeros(1, dtype=MENCIUS_CHOSEN))):
        with pytest.raises(FpxError) as ei:
            call()
        assert ei.value.status == UNSUPPORTED
    mp.close()
    sharded = Engine(1, AG, PER, num_leaders=2, num_replicas=2, protocol=MENCIUS, num_leader_groups=LG,
                     slot_capacity=1 << 10, max_batch=1 << 10, shard_index=0, shard_count=2)
    with pytest.raises(FpxError) as ei:
        sharded.mencius_replica_inbound(np.zeros(1, dtype=MENCIUS_CHOSEN))
    assert ei.value.status == UNSUPPORTED
    sharded.close()


def random_batch(g, n):
    RI = M.mcls("ReplicaInbound")
    msgs = []
    for _ in range(n):
        if g.random() < 0.6:
            v = M.payload(g, int(g.integers(-1, 3)), int(g.integers(0, 40)))
            msgs.append(RI(chosen=M.mcls("Chosen")(slot=int(g.integers(0, 1 << 30)), command_batch_or_noop=v))
                        .SerializeToString())
        else:
            a = int(g.integers(0, 1 << 30))
            msgs.append(RI(chosen_noop_range=M.mcls("ChosenNoopRange")(slot_start_inclusive=a,
                                                                       slot_end_exclusive=a + int(g.integers(0, 99))))
                        .SerializeToString())
    return msgs


def test_random_mutations_match_the_oracle(eng):
    g = np.random.default_rng(11)
    msgs = random_batch(g, 600)
    buf, offs = O.pack(msgs)
    assert same_decode(eng, buf, offs) == 0
    statuses = set()
    for _ in range(300):
        b = buf.copy()
        for _ in range(int(g.integers(1, 4))):
            b[int(g.integers(0, offs[-1]))] = int(g.integers(0, 256))
        statuses.add(same_decode(eng, b, offs, base=int(g.integers(0, 1000))))
    assert statuses == {0, WIRE}


def dev(a):
    t = torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).copy()).cuda()
    return t


def test_dev_forms_equal_host_forms(eng):
    g = np.random.default_rng(3)
    msgs = random_batch(g, 1500)
    buf, offs = O.pack(msgs)
    n = len(msgs)
    kind, recs, vals = eng.wire_decode_mencius_replica_inbound(buf, offs, 5)
    d_buf, d_offs = dev(buf), dev(offs)
    d_kind = torch.zeros(n, dtype=torch.int32, device="cuda")
    d_recs = torch.zeros(n * 4, dtype=torch.int32, device="cuda")
    d_vals = torch.zeros(n * 2, dtype=torch.int32, device="cuda")
    eng.wire_decode_mencius_replica_inbound_dev(d_buf.data_ptr(), d_offs.data_ptr(), n, 5, d_kind.data_ptr(),
                                                d_recs.data_ptr(), d_vals.data_ptr())
    eng.sync()
    assert np.array_equal(d_kind.cpu().numpy(), kind)
    assert np.array_equal(d_recs.cpu().numpy(), recs.view(np.int32).ravel())
    assert np.array_equal(d_vals.cpu().numpy(), vals.ravel())
    for name, dt, rec in (("chosen_range", CHOSEN_RANGE, None), ("phase2b_range", P2B_RANGE, None)):
        r = np.zeros(3000, dtype=dt)
        for f in dt.names:
            r[f] = g.integers(-(1 << 31), 1 << 31, size=len(r), dtype=np.int64).astype(np.int32)
        if name == "phase2b_range":
            r["dst"] = (g.integers(0, LG * AG, size=len(r)) << 16) | g.integers(0, PER, size=len(r))
        out, offs2 = getattr(eng, f"wire_encode_mencius_{name}")(r)
        oout, ooffs = O.encode(name, r, AG)
        assert np.array_equal(out, oout) and np.array_equal(offs2, ooffs)
        d_out = torch.zeros(len(out) + 64, dtype=torch.uint8, device="cuda")
        d_o = torch.zeros(len(r) + 1, dtype=torch.int32, device="cuda")
        getattr(eng, f"wire_encode_mencius_{name}_dev")(dev(r).data_ptr(), len(r), d_out.data_ptr(), len(out) + 64,
                                                        d_o.data_ptr())
        eng.sync()
        assert np.array_equal(d_o.cpu().numpy(), offs2) and np.array_equal(d_out.cpu().numpy()[:len(out)], out)
        if name == "phase2b_range":      # decoding the bytes gives back the records
            kind2, back = eng.wire_decode_inbound(WIRE_MENCIUS_PROXYLEADER_INBOUND, out, offs2)
            ok = ((r["dst"] >> 16) // AG) == (((r["slot_start"] % LG) + LG) % LG)
            assert (kind2 == 5).all() and np.array_equal(back.view(np.int32).reshape(-1, 4)[ok], r.view(np.int32).reshape(-1, 4)[ok])
    # the mixed call's device form: same split and log as the host form on a twin engine
    twin = mencius(slot_capacity=1 << 14, max_batch=1 << 14)
    recs = mixed_batch(np.random.default_rng(9), 4000, 3, 1 << 14, overlaps=3, bad=False)
    split = eng.mencius_replica_inbound(recs)
    d_split = torch.zeros(1, dtype=torch.int32, device="cuda")
    twin.mencius_replica_inbound_dev(dev(recs).data_ptr(), len(recs), d_split.data_ptr())
    twin.sync()
    assert int(d_split.item()) == split
    assert np.array_equal(eng.snapshot_log(0, 1 << 14), twin.snapshot_log(0, 1 << 14))
    twin.close()
    eng.reset()


def mixed_batch(g, n, lg, cap, overlaps=20, retired=0, bad=True):
    """Chosens and about 1 % ranges interleaved: ranges that meet earlier Chosens and Chosens inside earlier ranges,
    duplicate Chosens, empty and one-slot ranges, slots below `retired`, and `overlaps` ranges that overlap an
    earlier range."""
    recs = np.zeros(n, dtype=MENCIUS_CHOSEN)
    slots = g.integers(0, cap - 1, size=n)
    recs["slot_start"] = slots
    recs["slot_end"] = slots + 1
    recs["value_id"] = np.arange(n)
    dup = g.random(n) < 0.05
    recs["slot_start"][dup] = recs["slot_start"][np.maximum(np.arange(n) - 7, 0)][dup]
    recs["slot_end"][dup] = recs["slot_start"][dup] + 1
    rng = np.nonzero(g.random(n) < 0.01)[0]
    for k, i in enumerate(rng):
        s = int(g.integers(0, cap - 400))
        if k % 5 == 0 and i > 10:      # starts at or just below an earlier Chosen: meets it
            s = max(0, int(recs["slot_start"][i - int(g.integers(1, 10))]) - lg * int(g.integers(0, 4)))
        length = int(g.choice([0, 1, lg, 2 * lg, 40, 300]))
        recs[i] = (s, min(cap, s + length), VALUE_NOOP, 0)
    if retired:
        few = g.choice(n, size=max(1, n // 200), replace=False)
        recs["slot_start"][few] = g.integers(0, retired, size=len(few))
        recs["slot_end"][few] = recs["slot_start"][few] + np.where(g.random(len(few)) < 0.5, 1, 5 * lg)
    multi = rng[(recs["slot_end"][rng] - recs["slot_start"][rng] + lg - 1) // lg >= 2]
    for i in g.choice(multi[multi > 0], size=min(overlaps, max(0, len(multi) - 1)), replace=False) if len(multi) > 1 else []:
        earlier = multi[multi < i]
        if len(earlier):
            j = int(g.choice(earlier))
            recs[i] = (recs["slot_start"][j] + lg, recs["slot_end"][j] + lg, VALUE_NOOP, 0)
    if bad:
        recs["slot_start"][int(g.integers(n // 4, n // 2))] = -3
    return recs


def check_mixed(eng, recs, rep, cap):
    start, calls = 0, 0
    while start < len(recs):
        rest = recs[start:]
        want = rep.split(rest)
        st, err = rep.apply(rest[:want])
        try:
            split = eng.mencius_replica_inbound(rest)
            est, eidx = 0, -1
        except FpxError as e:
            est, eidx = e.status, e.index
            split = None
        assert (est, eidx) == (st, err)
        if split is None:              # a bad slot: the status, and the split read from a clean rerun is not needed
            split = want
        assert split == want
        assert split > 0
        start += split
        calls += 1
    live = eng.snapshot_log(rep.retired, cap - rep.retired)
    assert np.array_equal(live, rep.log[rep.retired:])
    assert eng.chosen_watermark() == rep.watermark()
    return calls


@pytest.mark.parametrize("seed", [0, 1, 2])
@pytest.mark.parametrize("lg", [1, 3, 5])
def test_mixed_apply_against_the_per_message_oracle(seed, lg):
    cap = 1 << 21
    n = 1 << 20
    e = mencius(lg=lg, ag=1, slot_capacity=cap, max_batch=n, overflow_capacity=1 << 10)
    g = np.random.default_rng(100 * seed + lg)
    rep = O.Replica(lg, cap)
    # a prefix already chosen, half of it retired
    pre = np.zeros(4096, dtype=MENCIUS_CHOSEN)
    pre["slot_start"] = np.arange(4096); pre["slot_end"] = pre["slot_start"] + 1; pre["value_id"] = 7
    assert e.mencius_replica_inbound(pre) == 4096
    rep.apply(pre)
    e.chosen_watermark()
    e.retire_below(2048)
    rep.retire_below(2048)
    recs = mixed_batch(g, n, lg, cap, retired=2048)
    # the bad record is reported at its index by the call holding it; clear it afterwards so the rest runs on
    bad = int(np.nonzero(recs["slot_start"] < 0)[0][0])
    head = recs[:bad + 1]
    check_mixed(e, head, rep, cap)
    calls = check_mixed(e, recs[bad + 1:], rep, cap)
    assert calls > 1            # the overlapping ranges split the batch
    e.close()


def test_end_to_end_from_protobuf_bytes():
    """Phase2aNoopRange at the acceptors -> Phase2bNoopRange bytes -> the proxy leader's tally -> ChosenNoopRange
    bytes -> with Chosen bytes, the replica's decoder and its mixed call.  Every message equals what the runtime
    serialises for the reference's message, and the log the per-message oracle's."""
    lg, ag, cap = 3, 2, 1 << 12
    e = mencius(lg=lg, ag=ag, slot_capacity=cap, max_batch=1 << 12)
    PL, RI = M.mcls("ProxyLeaderInbound"), M.mcls("ReplicaInbound")
    ranges = [(1, 301, 0), (5, 98, 0), (12, 13, 0), (30, 30, 0)]      # start, end, round (leader group start % 3)
    e.mencius_arm_range(np.array([(s, t, r, -1) for s, t, r in ranges], dtype=P2A_RANGE))
    deliveries = []
    for s, t, r in ranges:
        for a in (0, 1):
            for agi in range(ag):
                deliveries.append((s, t, r, (((s % lg) * ag + agi) << 16) | a))
    out, nack = e.mencius_acceptor_noop_range(np.array(deliveries, dtype=P2A_RANGE))
    assert len(nack) == 0 and len(out) == len(deliveries)
    b, offs = e.wire_encode_mencius_phase2b_range(out)
    want = [PL(phase2b_noop_range=M.mcls("Phase2bNoopRange")(
        acceptor_group_index=int(d >> 16) % ag, acceptor_index=int(d & 0xffff), slot_start_inclusive=int(s),
        slot_end_exclusive=int(t), round=int(r))).SerializeToString() for d, s, t, r in out]
    assert [bytes(b[offs[i]: offs[i + 1]]) for i in range(len(out))] == want
    kind, rec = e.wire_decode_inbound(WIRE_MENCIUS_PROXYLEADER_INBOUND, b, offs)
    assert (kind == 5).all()
    chosen = e.mencius_range_phase2b(rec.view(P2B_RANGE))
    assert len(chosen) == len(ranges)
    cb, coffs = e.wire_encode_mencius_chosen_range(chosen)
    cwant = [RI(chosen_noop_range=M.mcls("ChosenNoopRange")(slot_start_inclusive=int(s), slot_end_exclusive=int(t)))
             .SerializeToString() for s, t in chosen]
    assert [bytes(cb[coffs[i]: coffs[i + 1]]) for i in range(len(chosen))] == cwant
    g = np.random.default_rng(4)
    msgs = []
    for k in range(200):
        msgs.append(RI(chosen=M.mcls("Chosen")(slot=int(g.integers(0, 400)), command_batch_or_noop=M.payload(g, 1, 8)))
                    .SerializeToString())
        if k % 50 == 25:
            msgs.append(cwant[(k // 50) % len(cwant)])
    buf, moffs = O.pack(msgs)
    kind, recs, vals = e.wire_decode_mencius_replica_inbound(buf, moffs, 0)
    rep = O.Replica(lg, cap)
    assert e.mencius_replica_inbound(recs) == rep.split(recs) == len(recs)
    rep.apply(recs)
    assert np.array_equal(e.snapshot_log(0, cap), rep.log)
    assert e.chosen_watermark() == rep.watermark()
    e.close()


def test_codec_edges(eng):
    """A CTA whose span exceeds the 24 KB stage (decoded unstaged), encoders past tile_offsets_kernel's first chunk of
    4096 tiles, and an out_capacity one byte short."""
    g = np.random.default_rng(8)
    RI = M.mcls("ReplicaInbound")
    msgs = [RI(chosen=M.mcls("Chosen")(slot=i, command_batch_or_noop=M.payload(g, 1, 120))).SerializeToString()
            for i in range(512)]
    buf, offs = O.pack(msgs)
    assert offs[256] > 24 * 1024
    assert same_decode(eng, buf, offs) == 0
    bad = buf.copy(); bad[offs[300] + 1] = 0x7f          # a length past the message inside the unstaged CTA
    same_decode(eng, bad, offs)
    n = 4096 * 1024 + 1025
    r = np.zeros(n, dtype=CHOSEN_RANGE)
    r["slot_start"] = np.arange(n); r["slot_end"] = np.arange(n) + 300
    out, offs2 = eng.wire_encode_mencius_chosen_range(r)
    oout, ooffs = O.encode("chosen_range", r)
    assert np.array_equal(offs2, ooffs) and np.array_equal(out, oout)
    p = np.zeros(n, dtype=P2B_RANGE)
    p["dst"] = 1; p["slot_start"] = np.arange(n); p["slot_end"] = np.arange(n) + 9; p["round"] = 1 << 20
    out, offs2 = eng.wire_encode_mencius_phase2b_range(p)
    oout, ooffs = O.encode("phase2b_range", p, AG)
    assert np.array_equal(offs2, ooffs) and np.array_equal(out, oout)
    small = p[:5000]
    total = int(O.encode("phase2b_range", small, AG)[1][-1])
    buf_out = np.zeros(total + 256, dtype=np.uint8)
    o = np.zeros(len(small) + 1, dtype=np.int32)
    err = C.c_int64(-1)
    st = eng._L.fpx_wire_encode_mencius_phase2b_range(eng.h, np.ascontiguousarray(small).ctypes.data, len(small),
                                                      buf_out.ctypes.data, total - 1, o.ctypes.data, C.byref(err))
    assert (st, err.value) == (INVALID_ARG, 0) and not buf_out.any()
    out, _ = eng.wire_encode_mencius_phase2b_range(small)      # nothing latched
    assert len(out) == total
