"""GPU parity of compartmentalized Mencius' leader change from bytes (fpx_mencius_acceptor_phase1a_wire,
fpx_mencius_leader_phase1b_wire, fpx_wire_encode_mencius_phase2a) against the CPU oracle
(tests/wire_mencius_phase1_oracle.cc) and the protobuf runtime, and the change of one leader group's leader end to end
at 2^20 slots in flight."""
import numpy as np
import pytest

import wire_mencius_phase1_cases as W
import wire_mencius_phase1_oracle as O
from frankenpaxos_b200 import MENCIUS, VALUE_NOOP, WIRE_MENCIUS_ACCEPTOR_INBOUND, WIRE_MENCIUS_PROXYLEADER_INBOUND, \
    Engine, FpxError, dst

pytestmark = pytest.mark.gpu

LG, AG, F, PER = 3, 2, 1, 3           # the leader tests' config


def status_of(fn, *a, **kw):
    try:
        return 0, -1, fn(*a, **kw)
    except FpxError as e:
        return e.status, e.index, None


def mencius(f, lgroups, agroups, capacity=1 << 12, **kw):
    return Engine(f, agroups, 2 * f + 1, protocol=MENCIUS, num_leader_groups=lgroups, slot_capacity=capacity,
                  max_batch=kw.pop("max_batch", 1 << 12), **kw)


def same_leader(eng, leader_group, round_, cw, msgs, recover_slot=-1, base=0, cap=1 << 12, f=F, lgroups=LG, agroups=AG):
    buf, offs = O.pack(msgs)
    o = O.leader_phase1b(f, lgroups, agroups, 2 * f + 1, leader_group, round_, cw, buf, offs, recover_slot, base, cap)
    st, idx, got = status_of(eng.mencius_leader_phase1b_wire, leader_group, round_, cw, buf, offs, recover_slot, base,
                             cap)
    assert (st, idx) == (o[0], o[1])
    if st == 0:
        complete, max_slot, next_slot, recs, spans = got
        assert (complete, max_slot, next_slot) == (o[2], o[3], o[4])
        assert np.array_equal(recs.view(np.int32), o[5].view(np.int32)) and np.array_equal(spans, o[6])
    return o, buf, offs


@pytest.fixture(scope="module")
def eng():
    e = mencius(F, LG, AG)
    yield e
    e.close()


def test_golden_batches(eng):
    for case in W.GOLD["leader"]:
        msgs = [bytes.fromhex(m) for m in case["msgs"]]
        o, _, _ = same_leader(eng, case["leader_group"], case["round"], case["chosen_watermark"], msgs,
                              case["recover_slot"], 40)
        assert (o[0], o[1] if o[0] else o[2]) == (case["status"], case["index"])
    for case in W.GOLD["phase2a"]:
        payload = np.frombuffer(bytes.fromhex(case["payload_hex"]), np.uint8).copy()
        rec = np.zeros(1, O.P2A)
        rec["slot"], rec["round"], rec["dst"] = case["slot"], case["round"], 7
        rec["value_id"] = VALUE_NOOP if case["noop"] else 3
        out, offs = eng.wire_encode_mencius_phase2a(rec, payload, [[0, len(payload)]], 3)
        assert bytes(out) == bytes.fromhex(case["hex"]) and list(offs) == [0, len(out)]


@pytest.mark.parametrize("leader_group", [0, 1, 2])
def test_leader_random_and_mutated_batches(eng, leader_group):
    g = np.random.Generator(np.random.PCG64(70 + leader_group))
    a, voffs = W.arena(g, 64)
    seen = set()
    for _ in range(40):
        msgs = W.random_batch(g, LG, AG, PER, leader_group, 9, 300, int(g.integers(1, 14)), a, voffs)
        if g.random() < 0.3:
            msgs = [msgs[i] for i in g.permutation(len(msgs))]
        rec = int(g.choice([-1, leader_group + LG * int(g.integers(0, 400)), int(g.integers(0, 1200))]))
        o, _, _ = same_leader(eng, leader_group, 9, int(g.integers(0, 1000)), msgs, rec, int(g.integers(0, 1000)))
        seen.add(o[0])
    assert 0 in seen
    # 300 byte mutations: status and first index as the oracle's
    small = W.random_batch(g, LG, AG, PER, leader_group, 9, 40, 8, a, voffs, extra=False)
    small += [W.empty_phase1b(ag, c, 9) for ag in range(AG) for c in range(2)]
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
        same_leader(eng, leader_group, 9, 0, small[:i] + [bytes(raw)] + small[i + 1:], -1, 3)


def test_leader_refusals(eng):
    q = [W.empty_phase1b(ag, c, 4) for ag in range(AG) for c in (1, 2)]
    a, voffs = W.value_arena()
    other = O.encode_phase1b(0, 0, 4, [4], [1], [1], a, voffs)            # slot 4 belongs to leader group 1
    assert same_leader(eng, 0, 4, 0, [other] + q)[0][:2] == (-14, 4)
    assert same_leader(eng, 0, 4, 0, q, recover_slot=5)[0][:2] == (-14, 3)
    assert same_leader(eng, 0, 4, 0, [W.empty_phase1b(AG, 0, 4)] + q)[0][:2] == (-5, 0)
    assert same_leader(eng, 0, 4, 0, [W.empty_phase1b(0, PER, 4)] + q)[0][:2] == (-5, 0)
    assert same_leader(eng, 0, 4, 0, [W.empty_phase1b(0, 0, 5)] + q)[0][:2] == (-14, 0)
    # n_out = 0 with next_slot reported: no votes, a watermark past recover_slot
    o, _, _ = same_leader(eng, 2, 4, 30, q, recover_slot=26)
    assert o[0] == 0 and (o[3], o[4], len(o[5])) == (26, 29, 0)
    buf, offs = O.pack(q)
    for lg, cw, rec in [(-1, 0, -1), (LG, 0, -1), (0, -1, -1), (0, 0, -2)]:
        assert status_of(eng.mencius_leader_phase1b_wire, lg, 4, cw, buf, offs, rec)[0] == -1


def test_leader_device_form_and_capacity(eng):
    import torch
    dev = torch.device("cuda", 0)
    g = np.random.Generator(np.random.PCG64(31))
    a, voffs = W.arena(g, 32)
    msgs = W.random_batch(g, LG, AG, PER, 1, 9, 600, 10, a, voffs, extra=False)
    msgs += [W.empty_phase1b(ag, c, 9) for ag in range(AG) for c in range(PER)]
    buf, offs = O.pack(msgs)
    complete, max_slot, next_slot, recs, spans = eng.mencius_leader_phase1b_wire(1, 9, 5, buf, offs, 7, 50, 4096)
    assert complete >= 0 and len(recs) == (max_slot - 7) // LG + 1 and next_slot == max_slot + LG
    d_buf, d_offs = torch.from_numpy(buf).to(dev), torch.from_numpy(offs).to(dev)
    d_out, d_sp, d_res = (torch.zeros(s, dtype=torch.int32, device=dev) for s in ((4096, 4), (4096, 2), (4,)))
    torch.cuda.synchronize()
    eng.mencius_leader_phase1b_wire_dev(1, 9, 5, 7, d_buf.data_ptr(), len(buf), d_offs.data_ptr(), len(msgs), 50,
                                        d_out.data_ptr(), d_sp.data_ptr(), 4096, d_res.data_ptr())
    eng.sync()
    assert d_res.cpu().tolist() == [complete, max_slot, len(recs), next_slot]
    assert np.array_equal(d_out[:len(recs)].cpu().numpy().reshape(-1), recs.view(np.int32).reshape(-1))
    assert np.array_equal(d_sp[:len(recs)].cpu().numpy(), spans)
    # Phase2a bytes, host and device forms, against the oracle and the runtime
    hb, hoffs = eng.wire_encode_mencius_phase2a(recs, buf, spans, 50)
    ost, _, ob, ooffs = O.encode_phase2a(recs, buf, spans, 50)
    assert ost == 0 and bytes(hb) == bytes(ob) and np.array_equal(hoffs, ooffs)
    d_recs = torch.from_numpy(recs.view(np.int32).reshape(-1, 4).copy()).to(dev)
    d_bytes = torch.zeros(len(hb) + 64, dtype=torch.uint8, device=dev)
    d_o = torch.zeros(len(recs) + 1, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    eng.wire_encode_mencius_phase2a_dev(d_recs.data_ptr(), len(recs), d_buf.data_ptr(), len(buf), d_sp.data_ptr(),
                                        len(recs), 50, d_bytes.data_ptr(), len(d_bytes), d_o.data_ptr())
    eng.sync()
    assert np.array_equal(d_o.cpu().numpy(), hoffs) and bytes(d_bytes[:len(hb)].cpu().numpy()) == bytes(hb)
    kind, dec = eng.wire_decode_inbound(WIRE_MENCIUS_PROXYLEADER_INBOUND, hb, hoffs)
    assert (kind == 2).all() and np.array_equal(dec["a"], recs["slot"]) and np.array_equal(dec["b"], recs["round"])
    # one record short: refused at `complete`, nothing written
    assert status_of(eng.mencius_leader_phase1b_wire, 1, 9, 5, buf, offs, 7, 50, len(recs) - 1)[:2] == (-1, complete)


def test_encoder_against_runtime(eng):
    mk = W.runtime()
    g = np.random.Generator(np.random.PCG64(8))
    a, voffs = W.value_arena()
    recs = np.zeros(200, O.P2A)
    recs["slot"] = g.integers(-(1 << 31), 1 << 31, 200)
    recs["round"] = g.integers(-(1 << 31), 1 << 31, 200)
    k = g.integers(0, len(W.VALUES), 200)
    recs["value_id"] = np.where(g.random(200) < 0.3, VALUE_NOOP, 10 + np.arange(200))
    spans = np.stack([voffs[k], voffs[k + 1] - voffs[k]], 1).astype(np.int32)
    hb, hoffs = eng.wire_encode_mencius_phase2a(recs, a, spans, 10)
    for i, raw in enumerate(O.split(hb, hoffs)):
        m = mk.cls("ProxyLeaderInbound")()
        m.phase2a.slot, m.phase2a.round = int(recs["slot"][i]), int(recs["round"][i])
        m.phase2a.command_batch_or_noop.ParseFromString(
            O.NOOP_BYTES if recs["value_id"][i] == VALUE_NOOP else W.VALUES[k[i]])
        assert m.SerializeToString() == raw


def same_acceptor(e, o, rounds_cws, dests, arena, voffs, first_held=0, mk=None):
    buf, kind, recs = W.phase1a_batch(rounds_cws, dests)
    ost, oidx, ob, ooffs = o.phase1a_wire(first_held, buf, kind, recs, arena, voffs)
    st, idx, got = status_of(e.mencius_acceptor_phase1a_wire, buf, kind, recs, arena, voffs)
    assert (st, idx) == (ost, oidx)
    if st == 0:
        gb, goffs = got
        assert bytes(gb) == bytes(ob) and np.array_equal(goffs, ooffs)
        if mk is not None:
            for raw in O.split(gb, goffs):
                m = mk.cls("LeaderInbound")()
                m.ParseFromString(raw)
                assert m.SerializeToString() == raw
    for gr in range(o.lgroups * o.agroups):
        for c in range(o.per_group):
            assert e.snapshot_acceptor(gr, c)[0] == o.round(gr, c)
    return st, got


@pytest.mark.parametrize("shape", [(1, 1, 1), (1, 3, 2), (2, 3, 1), (2, 1, 2), (1, 3, 1), (2, 3, 2)])
def test_acceptor_against_oracle(shape):
    f, lgroups, agroups = shape
    g = np.random.Generator(np.random.PCG64(90 + f * 10 + lgroups * 3 + agroups))
    mk = W.runtime()
    a, voffs = W.value_arena()
    cap = 1 << 12
    with mencius(f, lgroups, agroups, cap) as e:
        o = O.Acceptors(f, lgroups, agroups)
        p2a, ranges = W.random_trace(g, f, lgroups, agroups, cap, 3000, 60, 5, len(W.VALUES))
        e.acceptor_phase2a(p2a)
        o.phase2a(p2a)
        e.mencius_acceptor_noop_range(ranges)
        o.noop_range(ranges, cap)
        keys = [(gr, c) for gr in range(lgroups * agroups) for c in range(2 * f + 1)]
        noop_above = False
        for rnd in range(10):
            picks = [keys[int(g.integers(0, len(keys)))] for _ in range(int(g.integers(1, 10)))]
            rc = [(int(g.integers(0, 4)) + rnd // 3 * 2, int(g.choice([0, cap // 3, cap // 2, cap + 50])))
                  for _ in picks]
            st, got = same_acceptor(e, o, rc, [int(dst(*k)) for k in picks], a, voffs, 0, mk)
            assert st == 0
            # noop-range votes above the acceptor's highest Phase2a vote are in its Phase1b
            for i, k in enumerate(picks):
                raw = bytes(got[0][got[1][i]: got[1][i + 1]])
                m = mk.cls("LeaderInbound")()
                m.ParseFromString(raw)
                if m.WhichOneof("request") != "phase1b":
                    continue
                top = e.snapshot_acceptor(*k)[1]
                noop_above |= any(x.slot > top and x.vote_value.WhichOneof("value") == "noop" for x in m.phase1b.info)
        assert noop_above
        # a malformed body and a non-member refuse the call; no round changes
        buf, kind, recs = W.phase1a_batch([(9, 0), (9, 0)], [0, 1])
        recs["d"][1] = 1
        assert status_of(e.mencius_acceptor_phase1a_wire, buf, kind, recs, a, voffs)[:2] == (-15, 1)
        assert same_acceptor(e, o, [(9, 0)], [int(dst(lgroups * agroups, 0))], a, voffs)[0] == -1


def test_acceptor_below_retired_base():
    with mencius(1, 3, 2, 1 << 10, max_batch=1 << 12) as e:
        o = O.Acceptors(1, 3, 2)
        a, voffs = W.value_arena()
        recs = np.zeros(240, O.P2A)
        recs["slot"] = np.arange(240); recs["round"] = 1; recs["value_id"] = 1
        grp = (recs["slot"] % 3) * 2 + (recs["slot"] // 3) % 2
        e.proxyleader_arm(recs)
        acc = np.repeat(recs, 3)
        acc["dst"] = dst(np.repeat(grp, 3), np.tile(np.arange(3), 240))
        p2b, _ = e.acceptor_phase2a(acc)
        o.phase2a(acc)
        e.replica_chosen(e.proxyleader_phase2b(p2b))
        assert e.chosen_watermark() == 240
        e.retire_below(128)
        d = [int(dst(1, 1))]
        assert same_acceptor(e, o, [(5, 3)], d, a, voffs, 128)[0] == -6          # SLOT_RANGE, nothing applied
        assert e.snapshot_acceptor(1, 1)[0] == 1
        assert same_acceptor(e, o, [(5, 128)], d, a, voffs, 128)[0] == 0
        assert same_acceptor(e, o, [(6, 150)], d, a, voffs, 128)[0] == 0


def test_unsupported():
    buf, offs = O.pack([W.empty_phase1b(0, 0, 1)])
    recs = np.zeros(1, O.P2A)
    with Engine(1, 1, 3, slot_capacity=1 << 10, max_batch=1 << 10) as e:           # MultiPaxos
        assert status_of(e.mencius_leader_phase1b_wire, 0, 1, 0, buf, offs)[0] == -11
        assert status_of(e.wire_encode_mencius_phase2a, recs, buf, [[0, 0]])[0] == -11
        rb, kind, rr = W.phase1a_batch([(1, 0)], [0])
        assert status_of(e.mencius_acceptor_phase1a_wire, rb, kind, rr, *W.value_arena())[0] == -11
    with mencius(1, 2, 1, 1 << 10, shard_count=2) as e:
        assert status_of(e.mencius_leader_phase1b_wire, 0, 1, 0, buf, offs)[0] == -11


def test_leader_change_end_to_end_2e20():
    """f = 2, LG = 3, AG = 2 (30 acceptors), 2^20 slots in flight, votes from Phase2a and noop ranges in every leader
    group.  Leader group 1 changes leader: runtime Phase1a bytes -> the acceptors' call -> the leader's call -> its
    Phase2a bytes decoded again -> arm -> acceptor -> tally -> replica.  The bytes, max_slot, next_slot, the Chosen
    stream and the log are the oracle's; the other groups' log entries are untouched."""
    g = np.random.Generator(np.random.PCG64(0))
    f, S = 2, 1 << 20
    a, voffs = W.arena(g, 4096)
    o = O.Acceptors(f, LG, AG)
    with mencius(f, LG, AG, S, max_batch=1 << 22, overflow_capacity=1 << 14) as e:
        # Phase2a votes of acceptors 0-2 on 90% of the lower three quarters, noop ranges over the top quarter
        votes = []
        for c in range(3):
            voted = np.nonzero(g.random(3 * S // 4) < 0.9)[0].astype(np.int32)
            p = np.zeros(len(voted), O.P2A)
            grp = (voted % LG) * AG + (voted // LG) % AG
            p["slot"], p["round"], p["dst"] = voted, g.integers(0, 7, len(voted)), dst(grp, c)
            p["value_id"] = np.where(g.random(len(voted)) < 0.05, VALUE_NOOP, g.integers(0, 4096, len(voted)))
            votes.append(p)
        p = np.concatenate(votes)
        e.acceptor_phase2a(p)
        o.phase2a(p)
        ranges = []
        for start in range(3 * S // 4, S - 4095, 4095):          # 3 * S / 4 and 4095 are multiples of LG
            for lg in range(LG):
                for ag in range(AG):
                    for c in (0, 1):
                        ranges.append((start + lg, start + 4032, 6, int(dst(lg * AG + ag, c))))
        ranges = np.array(ranges, O.P2A_RANGE)
        e.mencius_acceptor_noop_range(ranges)
        o.noop_range(ranges, S)
        before = e.snapshot_log(0, S)
        # Phase1a{round 7 + 1 = 8 (leader 2 of group 1), chosen_watermark 0} to acceptors 0-2 of both acceptor groups
        mk = W.runtime()
        raw = mk.cls("AcceptorInbound")(phase1a=mk.cls("Phase1a")(round=8, chosen_watermark=0)).SerializeToString()
        req, roffs = O.pack([raw] * (AG * 3))
        kind, recs1a = e.wire_decode_inbound(WIRE_MENCIUS_ACCEPTOR_INBOUND, req, roffs)
        recs1a = recs1a.copy()
        recs1a["a"] = dst(1 * AG + np.repeat(np.arange(AG), 3), np.tile(np.arange(3), AG))
        ost, _, ob, _ = o.phase1a_wire(0, req, kind, recs1a, a, voffs)
        p1b, p1offs = e.mencius_acceptor_phase1a_wire(req, kind, recs1a, a, voffs)
        assert ost == 0 and bytes(p1b) == bytes(ob)
        msgs = O.split(p1b, p1offs)
        # the acceptors' round-6 noop votes lie above their highest Phase2a vote
        assert e.snapshot_acceptor(2, 0)[1] < 3 * S // 4
        o2, buf, offs = same_leader(e, 1, 8, 0, msgs, -1, 0, S, f=f)
        complete, max_slot, next_slot, recs, spans = o2[2], o2[3], o2[4], o2[5], o2[6]
        assert complete == AG * 3 - 1 and max_slot % LG == 1 and next_slot == max_slot + LG
        assert max_slot > 3 * S // 4 and len(recs) == (max_slot - 1) // LG + 1
        p2a, poffs = e.wire_encode_mencius_phase2a(recs, buf, spans, 0)
        ost, _, ob, _ = O.encode_phase2a(recs, buf, spans, 0)
        assert ost == 0 and bytes(p2a) == bytes(ob)
        kind, dec = e.wire_decode_inbound(WIRE_MENCIUS_PROXYLEADER_INBOUND, p2a, poffs)
        assert (kind == 2).all() and np.array_equal(dec["a"], recs["slot"]) and np.array_equal(dec["b"], recs["round"])
        e.proxyleader_arm(recs)
        acc = np.repeat(recs, 3)
        grp = 1 * AG + (acc["slot"] // LG) % AG
        acc["dst"] = dst(grp, np.tile(np.arange(3), len(recs)))
        p2b, nack = e.acceptor_phase2a(acc)
        assert len(nack) == 0 and len(p2b) == len(acc)
        chosen = e.proxyleader_phase2b(p2b)
        assert np.array_equal(np.sort(chosen["slot"]), recs["slot"])
        want = dict(zip(recs["slot"].tolist(), recs["value_id"].tolist()))
        assert all(want[s] == v for s, v in zip(chosen["slot"].tolist(), chosen["value_id"].tolist()))
        e.replica_chosen(chosen)
        after = e.snapshot_log(0, S)
        mine = np.zeros(S, bool)
        mine[recs["slot"]] = True
        assert np.array_equal(after[recs["slot"]], recs["value_id"])
        assert np.array_equal(after[~mine], before[~mine])
