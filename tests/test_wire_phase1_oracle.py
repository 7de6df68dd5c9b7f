"""CPU checks of the leader's Phase-1 wire path oracle (tests/wire_phase1_oracle.cc) against the golden vectors
written by the Python protobuf runtime (tests/golden/make_wire_phase1_golden.py) and against the runtime's parse of
random Phase1b batches."""
import numpy as np
import pytest

import wire_phase1_cases as W
import wire_phase1_oracle as O


@pytest.mark.parametrize("case", W.GOLD["decode"], ids=[c["name"] for c in W.GOLD["decode"]])
def test_golden_phase1b(case):
    msgs, round_ = W.golden_batch(case)
    buf, offs = O.pack(msgs)
    st, idx, complete, max_slot, recs, spans = O.leader_phase1b(W.F, W.GROUPS, W.PER_GROUP, 0, round_, 0, buf, offs, 40)
    est, ecomplete, emax, out = W.golden_expectation(case, buf, offs)
    assert st == est
    if st != 0:
        assert idx == 0
        return
    assert (complete, max_slot, len(recs)) == (ecomplete, emax, len(out))
    for k, (slot, val) in enumerate(out):
        assert recs[k]["slot"] == slot and recs[k]["round"] == round_ and recs[k]["dst"] == -1
        if val is None:
            assert recs[k]["value_id"] == O.VALUE_NOOP
        else:
            assert recs[k]["value_id"] == 40 + k
            assert bytes(buf[spans[k, 0]: spans[k, 0] + spans[k, 1]]) == val


@pytest.mark.parametrize("case", W.GOLD["phase2a"], ids=[str(i) for i in range(len(W.GOLD["phase2a"]))])
def test_golden_phase2a(case):
    payload = np.frombuffer(bytes.fromhex(case["payload_hex"]), np.uint8)
    rec = np.zeros(1, O.P2A)
    rec["slot"], rec["round"], rec["dst"] = case["slot"], case["round"], 7
    rec["value_id"] = O.VALUE_NOOP if case["noop"] else 3
    st, _, out, offs = O.encode_phase2a(rec, payload, [[0, len(payload)]], value_id_base=3)
    assert st == 0 and bytes(out) == bytes.fromhex(case["hex"]) and list(offs) == [0, len(out)]


def runtime():
    import importlib.util
    import os
    spec = importlib.util.spec_from_file_location("mk", os.path.join(W.HERE, "golden", "make_wire_phase1_golden.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    return mk


# canonical CommandBatchOrNoops, which the runtime re-serializes unchanged: Noop, an empty batch, one command
CMD_ID = b"\x0a\x01a\x10\x01\x18\x01"
CMD = b"\x0a" + bytes([len(CMD_ID)]) + CMD_ID + b"\x12\x02xy"
BATCH = b"\x0a" + bytes([len(CMD)]) + CMD
VALUES = [b"\x12\x00", b"\x0a\x00", b"\x0a" + bytes([len(BATCH)]) + BATCH]


def value_arena():
    a = np.frombuffer(b"".join(VALUES), np.uint8).copy()
    return a, np.concatenate([[0], np.cumsum([len(v) for v in VALUES])]).astype(np.int32)


def test_phase1b_encoder_matches_runtime():
    mk = runtime()
    g = np.random.Generator(np.random.PCG64(5))
    a, voffs = value_arena()
    for _ in range(40):
        n = int(g.integers(0, 12))
        slots = g.integers(-(1 << 31), 1 << 31, size=n).astype(np.int32)
        vr = g.integers(-(1 << 31), 1 << 31, size=n).astype(np.int32)
        vid = g.integers(0, len(VALUES), size=n).astype(np.int32)
        vid[g.random(n) < 0.3] = O.VALUE_NOOP
        raw = O.encode_phase1b(1, 2, -3, slots, vr, vid, a, voffs)
        m = mk.cls("LeaderInbound")()
        m.phase1b.group_index, m.phase1b.acceptor_index, m.phase1b.round = 1, 2, -3
        for s, r, v in zip(slots, vr, vid):
            i = m.phase1b.info.add()
            i.slot, i.vote_round = int(s), int(r)
            i.vote_value.ParseFromString(O.NOOP_BYTES if v == O.VALUE_NOOP else VALUES[v])
        assert m.SerializeToString() == raw


def python_leader(msgs, groups, per_group, f, flexible, round_, cw, base):
    """Leader.handlePhase1b over runtime-parsed Phase1bs (one message at a time), as the reference runs it."""
    mk = runtime()
    held = [dict() for _ in range(groups)]
    for i, raw in enumerate(msgs):
        m = mk.cls("LeaderInbound")()
        m.ParseFromString(raw)
        if m.WhichOneof("request") != "phase1b":
            continue
        p = m.phase1b
        if p.round != round_:
            if p.round > round_:
                return -14, i, None
            continue
        if not (0 <= p.group_index < groups and 0 <= p.acceptor_index < per_group):
            return -5, i, None
        held[p.group_index][p.acceptor_index] = p
        if flexible:
            done = any(len(h) == per_group for h in held)
        else:
            done = all(len(h) >= f + 1 for h in held)
        if not done:
            continue
        mx = max((max((x.slot for x in p1.info), default=-1) for h in held for p1 in h.values()))
        out = []
        for s in range(cw, mx + 1):
            best = None
            for a in sorted(held[s % groups]):
                x = next((x for x in held[s % groups][a].info if x.slot == s), None)
                if x is not None and (best is None or x.vote_round > best.vote_round):
                    best = x
            out.append((s, None if best is None else best.vote_value.SerializeToString()))
        return 0, i, (mx, out)
    return 0, -1, None


@pytest.mark.parametrize("shape", [(1, 3, 0), (2, 3, 0), (2, 3, 1)])
def test_random_batches_against_runtime(shape):
    groups, per_group, flexible = shape
    g = np.random.Generator(np.random.PCG64(100 + groups + flexible))
    for _ in range(30):
        a, voffs = value_arena()
        msgs = W.random_phase1b_batch(g, groups, per_group, 5, 40, int(g.integers(1, 10)), a, voffs)
        cw = int(g.integers(0, 20))
        buf, offs = O.pack(msgs)
        st, idx, complete, max_slot, recs, spans = O.leader_phase1b(1, groups, per_group, flexible, 5, cw, buf, offs, 9)
        est, ei, res = python_leader(msgs, groups, per_group, 1, flexible, 5, cw, 9)
        if est != 0:
            assert (st, idx) == (est, ei)
            continue
        assert st == 0 and complete == ei
        if res is None:
            assert len(recs) == 0
            continue
        assert max_slot == res[0] and len(recs) == len(res[1])
        for k, (slot, val) in enumerate(res[1]):
            assert recs[k]["slot"] == slot
            got = None if recs[k]["value_id"] == O.VALUE_NOOP else bytes(buf[spans[k, 0]: spans[k, 0] + spans[k, 1]])
            assert got == val
