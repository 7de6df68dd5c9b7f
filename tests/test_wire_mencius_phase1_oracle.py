"""CPU checks of compartmentalized Mencius' leader-change wire path oracle (tests/wire_mencius_phase1_oracle.cc)
against the golden vectors and the Python transcriptions over Google's protobuf runtime
(tests/golden/make_wire_mencius_phase1_golden.py)."""
import numpy as np
import pytest

import wire_mencius_phase1_cases as W
import wire_mencius_phase1_oracle as O

CFG = W.GOLD["config"]


def check_leader(msgs, lgroups, agroups, per_group, f, leader_group, round_, cw, recover_slot, base=9):
    """the oracle against the transcription over the runtime's parse"""
    buf, offs = O.pack(msgs)
    st, idx, complete, max_slot, next_slot, recs, spans = O.leader_phase1b(
        f, lgroups, agroups, per_group, leader_group, round_, cw, buf, offs, recover_slot, base, 1 << 14)
    est, ei, res = W.runtime().leader(msgs, f, lgroups, agroups, per_group, leader_group, round_, cw, recover_slot)
    if est != 0:
        assert (st, idx) == (est, ei)
        return st
    assert st == 0 and complete == ei
    if res is None:
        assert len(recs) == 0 and (max_slot, next_slot) == (-1, -1)
        return st
    assert (max_slot, next_slot) == res[:2] and len(recs) == len(res[2])
    for k, (slot, val) in enumerate(res[2]):
        assert (recs[k]["slot"], recs[k]["round"], recs[k]["dst"]) == (slot, round_, -1)
        got = None if recs[k]["value_id"] == O.VALUE_NOOP else bytes(buf[spans[k, 0]: spans[k, 0] + spans[k, 1]])
        assert got == val and (got is None or recs[k]["value_id"] == base + k)
    return st


@pytest.mark.parametrize("case", W.GOLD["leader"], ids=[c["name"] for c in W.GOLD["leader"]])
def test_golden_leader(case):
    msgs = [bytes.fromhex(m) for m in case["msgs"]]
    buf, offs = O.pack(msgs)
    st, idx, complete, max_slot, next_slot, recs, spans = O.leader_phase1b(
        CFG["f"], CFG["lgroups"], CFG["agroups"], CFG["per_group"], case["leader_group"], case["round"],
        case["chosen_watermark"], buf, offs, case["recover_slot"], 40)
    assert (st, idx) == (case["status"], case["index"] if case["status"] else idx)
    if st != 0:
        return
    assert complete == case["index"]
    if "records" not in case:
        assert len(recs) == 0
        return
    assert (max_slot, next_slot, len(recs)) == (case["max_slot"], case["next_slot"], len(case["records"]))
    for k, (slot, val) in enumerate(case["records"]):
        assert recs[k]["slot"] == slot and recs[k]["round"] == case["round"]
        if val is None:
            assert recs[k]["value_id"] == O.VALUE_NOOP
        else:
            assert recs[k]["value_id"] == 40 + k and bytes(buf[spans[k, 0]: spans[k, 0] + spans[k, 1]]).hex() == val


def test_golden_cases_cover_the_rules():
    names = {c["name"] for c in W.GOLD["leader"]}
    for want in ["empty phase1bs", "a nack parsed as field 7", "a recover member replacing a phase1b",
                 "two phase1b members merging", "a stale round is ignored", "a higher round",
                 "an info slot of another leader group", "a recover_slot beyond every info",
                 "a recover_slot of another group"]:
        assert want in names
    by = {c["name"]: c for c in W.GOLD["leader"]}
    assert by["empty phase1bs"]["next_slot"] == 1 and by["empty phase1bs"]["records"] == []
    assert by["a recover_slot of another group"]["status"] == -14
    assert by["a recover_slot beyond every info"]["records"][-1] == [19, None]


@pytest.mark.parametrize("case", W.GOLD["phase2a"], ids=[str(i) for i in range(len(W.GOLD["phase2a"]))])
def test_golden_phase2a(case):
    payload = np.frombuffer(bytes.fromhex(case["payload_hex"]), np.uint8)
    rec = np.zeros(1, O.P2A)
    rec["slot"], rec["round"], rec["dst"] = case["slot"], case["round"], 7
    rec["value_id"] = O.VALUE_NOOP if case["noop"] else 3
    st, _, out, offs = O.encode_phase2a(rec, payload, [[0, len(payload)]], value_id_base=3)
    assert st == 0 and bytes(out) == bytes.fromhex(case["hex"]) and list(offs) == [0, len(out)]


@pytest.mark.parametrize("leader_group", [0, 1, 2])
def test_random_batches_against_transcription(leader_group):
    g = np.random.Generator(np.random.PCG64(300 + leader_group))
    a, voffs = W.value_arena()
    seen = set()
    for _ in range(60):
        msgs = W.random_batch(g, 3, 2, 3, leader_group, 5, 30, int(g.integers(1, 14)), a, voffs)
        cw = int(g.integers(0, 60))
        rec = int(g.choice([-1, -1, leader_group + 3 * int(g.integers(0, 40)), int(g.integers(0, 120))]))
        seen.add(check_leader(msgs, 3, 2, 3, 1, leader_group, 5, cw, rec))
    assert 0 in seen and -14 in seen


def test_refused_arguments():
    buf, offs = O.pack([W.empty_phase1b(0, 0, 1)])
    for lg, cw, rec in [(-1, 0, -1), (3, 0, -1), (0, -1, -1), (0, 0, -2)]:
        assert O.leader_phase1b(1, 3, 2, 3, lg, 1, cw, buf, offs, rec)[0] == -1


def test_next_slot_past_int32():
    top = (1 << 31) - 1                      # 2^31 - 1 = 3 * 715827882 + 1: leader group 1's slot
    msgs = [W.empty_phase1b(ag, a, 1) for ag in range(2) for a in range(2)]
    buf, offs = O.pack(msgs)
    assert O.leader_phase1b(1, 3, 2, 3, 1, 1, top - 1, buf, offs, top)[:2] == (-6, 3)
    st, _, _, max_slot, next_slot, recs, _ = O.leader_phase1b(1, 3, 2, 3, 1, 1, top - 1, buf, offs, top - 3)
    assert st == 0 and (max_slot, next_slot, len(recs)) == (top - 3, top, 0)


def acceptor_states(p2a, ranges, f, lgroups, agroups):
    """the reference's acceptors after the trace: states[(group, acceptor)] = {slot: (vote_round, value_id)}, rounds"""
    per_group = 2 * f + 1
    states = {(gr, c): {} for gr in range(lgroups * agroups) for c in range(per_group)}
    rounds = {k: -1 for k in states}
    for r in p2a:
        k = (int(r["dst"]) >> 16, int(r["dst"]) & 0xffff)
        if r["round"] >= rounds[k]:
            rounds[k] = int(r["round"])
            states[k][int(r["slot"])] = (rounds[k], int(r["value_id"]))
    for r in ranges:
        k = (int(r["dst"]) >> 16, int(r["dst"]) & 0xffff)
        if r["round"] >= rounds[k]:
            rounds[k] = int(r["round"])
            s = int(r["slot_start"])
            while (s // lgroups) % agroups != k[0] % agroups:
                s += lgroups
            for slot in range(s, int(r["slot_end"]), lgroups * agroups):
                states[k][slot] = (rounds[k], O.VALUE_NOOP)
    return states, rounds


@pytest.mark.parametrize("shape", [(1, 1, 1), (1, 3, 2), (2, 3, 1)])
def test_acceptor_against_transcription(shape):
    f, lgroups, agroups = shape
    g = np.random.Generator(np.random.PCG64(400 + f * 10 + lgroups + agroups))
    mk = W.runtime()
    a, voffs = W.value_arena()
    values = W.VALUES
    o = O.Acceptors(f, lgroups, agroups)
    p2a, ranges = W.random_trace(g, f, lgroups, agroups, 600, 400, 12, 5, len(W.VALUES))
    o.phase2a(p2a)
    o.noop_range(ranges, 600)
    states, rounds = acceptor_states(p2a, ranges, f, lgroups, agroups)
    keys = sorted(states)
    for _ in range(6):
        picks = [keys[int(g.integers(0, len(keys)))] for _ in range(int(g.integers(1, 6)))]
        rc = [(int(g.integers(0, 8)), int(g.choice([0, 150, 300, 700]))) for _ in picks]
        buf, kind, recs = W.phase1a_batch(rc, [(k[0] << 16) | k[1] for k in picks])
        st, _, out, offs = o.phase1a_wire(0, buf, kind, recs, a, voffs)
        assert st == 0
        for i, (k, (r, cw)) in enumerate(zip(picks, rc)):
            m = mk.cls("AcceptorInbound")(phase1a=mk.cls("Phase1a")(round=r, chosen_watermark=cw))
            vals = {s: (vr, O.NOOP_BYTES if v == O.VALUE_NOOP else values[v]) for s, (vr, v) in states[k].items()}
            rounds[k], want = mk.acceptor(vals, rounds[k], k[0], k[1], agroups, m.phase1a.SerializeToString())
            assert bytes(out[offs[i]: offs[i + 1]]) == want
        for k in keys:
            assert o.round(*k) == rounds[k]
