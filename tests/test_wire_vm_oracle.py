"""The vanilla Mencius wire oracle (tests/wire_vm_oracle.cc) against tests/golden/wire_vanilla_mencius.json (bytes
written by Google's Python protobuf runtime from S/vanillamencius/VanillaMencius.proto's shapes) and against that
runtime on random messages."""
import importlib.util
import json
import os

import numpy as np
import pytest

import wire_vm_oracle as V

HERE = os.path.dirname(os.path.abspath(__file__))
CASES = json.load(open(os.path.join(HERE, "golden", "wire_vanilla_mencius.json")))["cases"]
N = 7                                                   # servers of the coordinator vectors


def of_type(t):
    return [c for c in CASES if c["type"] == t]


def golden_module():
    pytest.importorskip("google.protobuf")
    spec = importlib.util.spec_from_file_location("make_wire_vm_golden", os.path.join(HERE, "golden", "make_wire_vm_golden.py"))
    G = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(G)
    return G


def expected_decode(c):
    """(kind, (a, b, c, d) with value spans as hex, sender) of a golden case."""
    t = c["type"]
    if t == "phase2b":
        return 5, (0, c["server_index"], c["slot"], c["round"]), c["server_index"]
    if t == "skip":
        return 6, (c["server_index"], c["start"], c["stop"], 0), c["server_index"]
    if t == "phase2_nack":
        return 9, (c["slot"], c["round"], 0, 0), -1
    if t.startswith("phase2a"):
        return 4, (c["slot"], c["round"], c["value_hex"]), c["sending_server"]
    if t == "chosen":
        return 7, (c["slot"], c["is_revocation"], c["value_hex"]), -1
    if t == "client_request":
        return 1, (0, 0, c["value_hex"]), -1
    return {"phase1a": 2, "phase1b": 3, "phase1_nack": 8}[t], (0, 0, c["body_hex"]), -1


def decoded(buf, kind, rec, sender):
    """The decoder's output in expected_decode's form."""
    out = []
    for k, r, s in zip(kind, rec, sender):
        if k in (5, 6, 9):
            out.append((int(k), tuple(int(x) for x in r.tolist()), int(s)))
        else:
            out.append((int(k), (int(r["a"]), int(r["b"]), bytes(buf[r["c"]: r["c"] + r["d"]]).hex()), int(s)))
    return out


GOLDEN_TYPES = ["phase2b", "skip", "phase2_nack", "phase2a", "phase2a.coordinator", "chosen", "client_request",
                "phase1a", "phase1b", "phase1_nack"]


@pytest.mark.parametrize("t", GOLDEN_TYPES)
def test_decode_golden(t):
    cs = of_type(t)
    buf, offs = V.pack([bytes.fromhex(c["hex"]) for c in cs])
    st, err, kind, rec, sender = V.decode(buf, offs)
    assert (st, err) == (0, -1)
    assert decoded(buf, kind, rec, sender) == [expected_decode(c) for c in cs]


def test_client_request_span_is_the_coordinators_value():
    """The span of a ClientRequest is the encoding of CommandOrNoop().withCommand(command): the Phase2a encoder
    fed that span as the value reproduces the coordinator's Phase2a bytes."""
    reqs = of_type("client_request")
    buf, offs = V.pack([bytes.fromhex(c["hex"]) for c in reqs])
    st, _, kind, rec, _ = V.decode(buf, offs)
    assert st == 0 and (kind == 1).all()
    arena, voffs = V.pack([bytes(buf[r["c"]: r["c"] + r["d"]]) for r in rec])
    p2a = {c["value_hex"]: c for c in of_type("phase2a.coordinator")}
    recs = np.array([(p2a[c["value_hex"]]["slot"], p2a[c["value_hex"]]["round"], k, 0) for k, c in enumerate(reqs)],
                    dtype=V.P2A)
    st, _, out, eoffs = V.encode("phase2a", recs, arena, voffs, N)
    assert st == 0 and V.split(out, eoffs) == [bytes.fromhex(p2a[c["value_hex"]]["hex"]) for c in reqs]


def value_arena(cs):
    """(arena, offsets, value_id per case) with the Noop as VALUE_NOOP, like the engine's log holds it."""
    vals, ids = [], []
    for c in cs:
        if c["value_hex"] == "1200":
            ids.append(V.VALUE_NOOP)
        else:
            ids.append(len(vals)); vals.append(bytes.fromhex(c["value_hex"]))
    arena, voffs = V.pack(vals)
    return arena, voffs, ids


def test_encode_golden():
    cs = of_type("phase2b")
    st, _, out, offs = V.encode("replies", np.array([(0, c["server_index"], c["slot"], c["round"]) for c in cs], dtype=V.P2B))
    assert st == 0 and V.split(out, offs) == [bytes.fromhex(c["hex"]) for c in cs]
    cs = of_type("phase2_nack")
    st, _, out, offs = V.encode("replies", np.array([(1, 4, c["slot"], c["round"]) for c in cs], dtype=V.P2B))
    assert st == 0 and V.split(out, offs) == [bytes.fromhex(c["hex"]) for c in cs]
    cs = of_type("skip")
    st, _, out, offs = V.encode("skip", np.array([(c["server_index"], c["start"], c["stop"], 1) for c in cs], dtype=V.VM_SKIP))
    assert st == 0 and V.split(out, offs) == [bytes.fromhex(c["hex"]) for c in cs]
    cs = [c for c in of_type("chosen") if not c["is_revocation"]]
    arena, voffs, ids = value_arena(cs)
    assert V.VALUE_NOOP in ids
    st, _, out, offs = V.encode("chosen", np.array([(c["slot"], v) for c, v in zip(cs, ids)], dtype=V.CHOSEN), arena, voffs)
    assert st == 0 and V.split(out, offs) == [bytes.fromhex(c["hex"]) for c in cs]
    st, _, out, offs = V.encode("replies", np.array([(2, 1, c["slot"], v) for c, v in zip(cs, ids)], dtype=V.P2B), arena, voffs)
    assert st == 0 and V.split(out, offs) == [bytes.fromhex(c["hex"]) for c in cs]
    cs = of_type("phase2a.coordinator")
    arena, voffs, ids = value_arena(cs)
    st, _, out, offs = V.encode("phase2a", np.array([(c["slot"], c["round"], v, 3) for c, v in zip(cs, ids)], dtype=V.P2A),
                                arena, voffs, N)
    assert st == 0 and V.split(out, offs) == [bytes.fromhex(c["hex"]) for c in cs]


def test_encode_retired_reply_is_empty_and_bad_records_are_invalid_arg():
    arena, voffs = V.pack([b"\x0a\x00"])
    recs = np.array([(0, 1, 5, 0), (3, 1, 6, 0), (2, 1, 7, 0), (1, 1, 8, 2)], dtype=V.P2B)
    st, _, out, offs = V.encode("replies", recs, arena, voffs)
    assert st == 0 and [len(m) for m in V.split(out, offs)][1] == 0
    for bad, idx in ((np.array([(0, 1, 5, 0), (2, 1, 7, 1)], dtype=V.P2B), 1),       # value_id past the arena
                     (np.array([(4, 1, 5, 0)], dtype=V.P2B), 0),                       # no such reply kind
                     (np.array([(2, 1, 5, -5)], dtype=V.P2B), 0)):                     # negative, not the Noop
        assert V.encode("replies", bad, arena, voffs)[:2] == (-1, idx)
    assert V.encode("chosen", np.array([(1, 0), (2, 1)], dtype=V.CHOSEN), arena, voffs)[:2] == (-1, 1)


def test_robustness_agrees_with_the_protobuf_runtime():
    """The fixture's verdicts are Google's Python runtime's.  It does not enforce proto2 `required` on parse;
    scalapb's generated parser does ("Message missing required fields."), and so does the codec: a message the
    runtime leaves uninitialised is FPX_ERR_WIRE.  A second command_or_noop, which the runtime merges, is
    FPX_ERR_WIRE too (the value is one span of bytes)."""
    good = bytes.fromhex(of_type("phase2b")[2]["hex"])
    for c in of_type("robustness"):
        raw = bytes.fromhex(c["hex"])
        buf, offs = V.pack([good, raw, good])
        st, err, kind, rec, sender = V.decode(buf, offs)
        v = c["verdict"]
        if "error" in v or not v["initialized"] or c["name"] == "command_or_noop twice":
            assert (st, err) == (-15, 1), c["name"]
            continue
        assert st == 0 and kind[1] == v["kind"], c["name"]
        f = v.get("fields", {})
        if v["kind"] == 5:
            assert rec[1].tolist() == (0, f["server_index"], f["slot"], f["round"]) and sender[1] == f["server_index"]
        if v["kind"] == 7:
            assert (rec[1]["a"], rec[1]["b"]) == (f["slot"], int(f["isRevocation"])), c["name"]


def test_oracle_against_the_protobuf_runtime_on_random_messages():
    """Random messages serialised by Google's Python runtime (the same descriptors as the golden generator) decode
    to their fields, and the oracle's encoders reproduce the runtime's bytes."""
    G = golden_module()
    g = np.random.Generator(np.random.PCG64(2027))
    SI = G.vcls("ServerInbound")

    def r32():
        return int(g.integers(-(1 << 31), 1 << 31) >> int(g.integers(0, 32)))
    msgs, exp = [], []
    for _ in range(600):
        k = int(g.integers(0, 6))
        a, b, c = r32(), r32(), r32()
        if k == 0:
            m = SI(phase2b=G.vcls("Phase2b")(server_index=a, slot=b, round=c)); e = (5, (0, a, b, c), a)
        elif k == 1:
            m = SI(skip=G.vcls("Skip")(server_index=a, start_slot_inclusive=b, stop_slot_exclusive=c)); e = (6, (a, b, c, 0), a)
        elif k == 2:
            m = SI(phase2_nack=G.vcls("Phase2Nack")(slot=a, round=b)); e = (9, (a, b, 0, 0), -1)
        elif k == 3:
            v = G.vvalue(g, int(g.integers(-1, 150)))
            m = SI(phase2a=G.vcls("Phase2a")(sending_server=a, slot=b, round=c, command_or_noop=v))
            e = (4, (b, c, v.SerializeToString().hex()), a)
        elif k == 4:
            v = G.vvalue(g, int(g.integers(-1, 150)))
            rev = bool(g.integers(0, 2))
            m = SI(chosen=G.vcls("Chosen")(slot=a, command_or_noop=v, isRevocation=rev))
            e = (7, (a, int(rev), v.SerializeToString().hex()), -1)
        else:
            cmd = G.vcommand(g, int(g.integers(0, 150)))
            m = SI(client_request=G.vcls("ClientRequest")(command=cmd))
            e = (1, (0, 0, G.vcls("CommandOrNoop")(command=cmd).SerializeToString().hex()), -1)
        msgs.append(m.SerializeToString()); exp.append(e)
    buf, offs = V.pack(msgs)
    st, err, kind, rec, sender = V.decode(buf, offs)
    assert (st, err) == (0, -1) and decoded(buf, kind, rec, sender) == exp
    # encoders: replies (all kinds), Chosen, Phase2a, Skip
    vals = [G.vvalue(g, int(g.integers(0, 200))) for _ in range(50)]
    arena, voffs = V.pack([v.SerializeToString() for v in vals])
    noop = G.vvalue(g, -1)
    reps, want = np.zeros(800, dtype=V.P2B), []
    for i in range(len(reps)):
        k, a, b, c = int(g.integers(0, 4)), r32(), r32(), r32()
        vid = V.VALUE_NOOP if g.integers(0, 5) == 0 else int(g.integers(0, len(vals)))
        reps[i] = (k, a, b, c if k != 2 else vid)
        val = noop if vid == V.VALUE_NOOP else vals[max(vid, 0)]
        want.append([SI(phase2b=G.vcls("Phase2b")(server_index=a, slot=b, round=c)),
                     SI(phase2_nack=G.vcls("Phase2Nack")(slot=b, round=c)),
                     SI(chosen=G.vcls("Chosen")(slot=b, command_or_noop=val, isRevocation=False)), None][k])
    st, _, out, eoffs = V.encode("replies", reps, arena, voffs)
    assert st == 0 and V.split(out, eoffs) == [b"" if m is None else m.SerializeToString() for m in want]
    p2a = np.zeros(300, dtype=V.P2A)
    p2a["slot"] = g.integers(0, 1 << 31, size=len(p2a)) >> g.integers(0, 31, size=len(p2a))
    p2a["round"] = [r32() for _ in range(len(p2a))]
    p2a["value_id"] = np.where(g.integers(0, 4, size=len(p2a)) == 0, V.VALUE_NOOP, g.integers(0, len(vals), size=len(p2a)))
    st, _, out, eoffs = V.encode("phase2a", p2a, arena, voffs, N)
    assert st == 0 and V.split(out, eoffs) == [
        SI(phase2a=G.vcls("Phase2a")(sending_server=int(r["slot"]) % N, slot=int(r["slot"]), round=int(r["round"]),
                                     command_or_noop=noop if r["value_id"] == V.VALUE_NOOP else vals[r["value_id"]])).SerializeToString()
        for r in p2a]
    ch = p2a[["slot", "value_id"]].astype(V.CHOSEN)
    st, _, out, eoffs = V.encode("chosen", ch, arena, voffs)
    assert st == 0 and V.split(out, eoffs) == [
        SI(chosen=G.vcls("Chosen")(slot=int(r["slot"]), isRevocation=False,
                                   command_or_noop=noop if r["value_id"] == V.VALUE_NOOP else vals[r["value_id"]])).SerializeToString()
        for r in ch]
    sk = np.array([(r32(), r32(), r32(), 1) for _ in range(300)], dtype=V.VM_SKIP)
    st, _, out, eoffs = V.encode("skip", sk)
    assert st == 0 and V.split(out, eoffs) == [
        SI(skip=G.vcls("Skip")(server_index=int(r["server"]), start_slot_inclusive=int(r["slot_start"]),
                               stop_slot_exclusive=int(r["slot_stop"]))).SerializeToString() for r in sk]
