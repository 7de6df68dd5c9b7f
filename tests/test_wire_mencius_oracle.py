"""CPU checks of the Compartmentalized Mencius wire oracle (tests/wire_mencius_oracle.cc): against the golden vectors
(Google's Python protobuf runtime over a Mencius.proto pool), against the runtime on random messages, and its
per-message replica and split rule against a plain restatement of Replica.handleChosen / handleChosenNoopRange."""
import json
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import wire_mencius_oracle as O  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "wire_mencius.json")
WIRE = -15


def cases(t):
    return [c for c in json.load(open(GOLDEN))["cases"] if c["type"] == t]


def test_golden_replica_inbound_decodes():
    cs = cases("chosen") + cases("chosen_noop_range")
    buf, offs = O.pack([bytes.fromhex(c["hex"]) for c in cs])
    st, err, kind, recs, vals = O.decode(buf, offs, value_id_base=100)
    assert st == 0 and err == -1
    for i, c in enumerate(cs):
        r = recs[i]
        if c["type"] == "chosen":
            assert kind[i] == 1
            assert (r["slot_start"], r["slot_end"], r["value_id"]) == (c["slot"], np.int32(np.uint32(c["slot"] + 1 & 0xffffffff)), 100 + i)
            assert bytes(buf[vals[i][0]: vals[i][0] + vals[i][1]]).hex() == c["value_hex"]
        else:
            assert kind[i] == 2 and tuple(vals[i]) == (0, 0)
            assert (r["slot_start"], r["slot_end"], r["value_id"]) == (c["start"], c["end"], O.VALUE_NOOP)


def test_golden_encoders():
    pr = cases("phase2b_noop_range")
    agroups = 1 << 14      # every acceptor_group_index of the vectors that fits 16 bits survives the packing
    keep = [c for c in pr if 0 <= c["acceptor_group_index"] < agroups and 0 <= c["acceptor_index"] < 0x10000]
    recs = np.array([((c["acceptor_group_index"] << 16) | c["acceptor_index"], c["start"], c["end"], c["round"])
                     for c in keep], dtype=O.P2B_RANGE)
    out, offs = O.encode("phase2b_range", recs, agroups)
    assert [m.hex() for m in O.split_messages(out, offs)] == [c["hex"] for c in keep]
    cr = cases("chosen_noop_range")
    out, offs = O.encode("chosen_range", np.array([(c["start"], c["end"]) for c in cr], dtype=O.CHOSEN_RANGE))
    assert [m.hex() for m in O.split_messages(out, offs)] == [c["hex"] for c in cr]
    nk = cases("nack")
    out, offs = O.encode("nack", np.array([(3, c["round"]) for c in nk], dtype=O.NACK))
    assert [m.hex() for m in O.split_messages(out, offs)] == [c["hex"] for c in nk]
    assert all(c["hex"].startswith("3a") for c in nk)          # LeaderInbound.nack = 7


def test_golden_robustness():
    for c in cases("robustness"):
        raw = bytes.fromhex(c["hex"])
        st, err, kind, recs, vals = O.decode(*O.pack([raw]))
        v = c["verdict"]
        name = c["name"]
        if "error" in v or not v["initialized"] or name == "command_batch_or_noop twice":
            # the runtime rejects it, `required` fails it, or (a second value) the codec refuses a merge
            assert st == WIRE and err == 0 and kind[0] == 0, name
            continue
        assert st == 0, name
        assert kind[0] == v["kind"], name
        if v["kind"] == 2:
            assert (recs[0]["slot_start"], recs[0]["slot_end"]) == (v["fields"]["slot_start_inclusive"],
                                                                    v["fields"]["slot_end_exclusive"]), name
        elif v["kind"] == 1:
            assert recs[0]["slot_start"] == v["fields"]["slot"], name
        else:
            assert (recs[0]["slot_start"], recs[0]["slot_end"], recs[0]["value_id"]) == (0, 0, O.VALUE_NOOP), name


def random_messages(g, n):
    import make_wire_mencius_golden as M
    RI = M.mcls("ReplicaInbound")
    msgs, exp = [], []
    for _ in range(n):
        if g.random() < 0.5:
            s = int(g.integers(-(1 << 31), 1 << 31))
            v = M.payload(g, int(g.integers(-1, 3)), int(g.integers(0, 50)))
            msgs.append(RI(chosen=M.mcls("Chosen")(slot=s, command_batch_or_noop=v)).SerializeToString())
            exp.append((1, s, v.SerializeToString()))
        else:
            a, b = (int(x) for x in g.integers(-(1 << 31), 1 << 31, size=2))
            msgs.append(RI(chosen_noop_range=M.mcls("ChosenNoopRange")(slot_start_inclusive=a,
                                                                       slot_end_exclusive=b)).SerializeToString())
            exp.append((2, a, b))
    return msgs, exp


def test_random_messages_against_the_runtime():
    g = np.random.default_rng(5)
    msgs, exp = random_messages(g, 400)
    buf, offs = O.pack(msgs)
    st, err, kind, recs, vals = O.decode(buf, offs)
    assert st == 0
    for i, e in enumerate(exp):
        assert kind[i] == e[0]
        assert recs[i]["slot_start"] == e[1]
        if e[0] == 1:
            assert bytes(buf[vals[i][0]: vals[i][0] + vals[i][1]]) == e[2]
        else:
            assert recs[i]["slot_end"] == e[2]


def restated(recs, lg, cap, log, retired=0):
    """Replica.handleChosen / handleChosenNoopRange, message by message."""
    for r in recs:
        s, e, v = int(r["slot_start"]), int(r["slot_end"]), int(r["value_id"])
        if s < 0 or e < s or e > cap:
            continue
        for slot in range(s, e, lg):
            if slot < retired or log[slot] != -1:
                break
            log[slot] = v


def restated_split(recs, lg, cap):
    ranges = []
    for i, r in enumerate(recs):
        s, e = int(r["slot_start"]), int(r["slot_end"])
        if s < 0 or e < s or e > cap or (e - s + lg - 1) // lg < 2:
            continue
        if len(ranges) == O.MAX_RANGE_BATCH:
            return i
        slots = set(range(s, e, lg))
        if any(slots & set(range(a, b, lg)) for a, b in ranges):
            return i
        ranges.append((s, e))
    return len(recs)


@pytest.mark.parametrize("lg", [1, 3, 5])
def test_replica_oracle_against_the_restatement(lg):
    g = np.random.default_rng(lg)
    cap = 2000
    for _ in range(30):
        n = int(g.integers(1, 60))
        recs = np.zeros(n, dtype=O.MENCIUS_CHOSEN)
        for i in range(n):
            s = int(g.integers(-2, cap))
            if g.random() < 0.6:
                recs[i] = (s, s + 1, i, 0)
            else:
                recs[i] = (s, s + int(g.integers(-2, 40)), O.VALUE_NOOP, 0)
        rep = O.Replica(lg, cap)
        split = rep.split(recs)
        assert split == restated_split(recs, lg, cap)
        rep.apply(recs[:split])
        log = np.full(cap, -1, dtype=np.int32)
        restated(recs[:split], lg, cap, log)
        assert np.array_equal(rep.log, log)
