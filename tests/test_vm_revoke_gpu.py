"""Vanilla Mencius revocation, the servers' side, on the GPU against tests/vm_revoke_model.py and Google's protobuf
runtime: fpx_vm_phase1a_wire (Server.handlePhase1a from ServerInbound bytes), fpx_vm_choose (choose with
isRevocation), reply kind 4 of fpx_vm_phase2a and its bytes, and fpx_vm_entries."""
import importlib.util
import os

import numpy as np
import pytest

from frankenpaxos_b200 import (P2A, P2B, VALUE_NOOP, VANILLA_MENCIUS, Engine, FpxError)
import wire_vm_oracle as V
from vm_revoke_model import Server

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ERR_WIRE = -15   # include/fpx.h FPX_ERR_WIRE
CAP = 1 << 11


@pytest.fixture(scope="module")
def G():
    pytest.importorskip("google.protobuf")
    spec = importlib.util.spec_from_file_location("make_wire_vm_golden", os.path.join(HERE, "golden", "make_wire_vm_golden.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def arena_of(G, g, k):
    """k random CommandOrNoop values: their bytes packed, offsets, and the protobuf objects"""
    vals = [G.vvalue(g, int(g.integers(0, 40))) for _ in range(k)]
    arena, offs = V.pack([v.SerializeToString() for v in vals])
    return arena, offs, vals


def cmd_or_noop(G, vals, v):
    if v == VALUE_NOOP:
        c = G.vcls("CommandOrNoop")()
        c.noop.SetInParent()
        return c
    return vals[v]


def expected_reply(G, vals, server, reply):
    si = G.vcls("ServerInbound")()
    if reply[0] == "nack":
        _, start, stop, rnd = reply
        si.phase1_nack.start_slot_inclusive, si.phase1_nack.stop_slot_exclusive, si.phase1_nack.round = start, stop, rnd
        return si.SerializeToString()
    _, rnd, start, stop, infos = reply
    p = si.phase1b
    p.server_index, p.round, p.start_slot_inclusive, p.stop_slot_exclusive = server, rnd, start, stop
    for slot, kind, a, b in infos:
        info = p.info.add()
        info.slot = slot
        if kind == "pending":
            info.pending_slot_info.vote_round = a
            info.pending_slot_info.vote_value.CopyFrom(cmd_or_noop(G, vals, b))
        else:
            info.chosen_slot_info.value.CopyFrom(cmd_or_noop(G, vals, a))
            info.chosen_slot_info.is_revocation = bool(b)
    return si.SerializeToString()


def phase1a_bytes(G, round_, start, stop):
    si = G.vcls("ServerInbound")()
    si.phase1a.round, si.phase1a.start_slot_inclusive, si.phase1a.stop_slot_exclusive = round_, start, stop
    return si.SerializeToString()


def run_phase1a(eng, G, msgs, servers, next_slot):
    """msgs: ServerInbound bytes; servers[i]: the receiving server.  Returns the decoded rows and the batch."""
    buf, offs = V.pack(msgs)
    kind, rec, _ = eng.wire_decode_vm_server_inbound(buf, offs)
    rec = rec.copy()
    rec["a"] = servers
    return kind, rec, buf


def check_entries(eng, model, n, upto):
    for s in range(n):
        got = eng.vm_entries(s, 0, upto)
        want = np.array([model[s].entry_row(x) for x in range(upto)], dtype=np.int32)
        bad = np.nonzero((got != want).any(axis=1))[0]
        assert len(bad) == 0, (s, int(bad[0]), got[bad[0]].tolist(), want[bad[0]].tolist())


@pytest.mark.parametrize("n", [3, 7])
@pytest.mark.parametrize("seed", [0, 1])
def test_random_traces_agree_with_the_model(G, n, seed):
    g = np.random.default_rng(seed * 10 + n)
    f = (n - 1) // 2
    arena, voffs, vals = arena_of(G, g, 64)
    span = 64 * n                                   # the slots the trace touches
    eng = Engine(f, 1, n, slot_capacity=CAP, max_batch=1 << 12, protocol=VANILLA_MENCIUS)
    model = [Server(s, n) for s in range(n)]
    next_slot = np.array([span + s for s in range(n)], dtype=np.int32)
    for s in range(n):
        model[s].next_slot = int(next_slot[s])
    chosen_value = [VALUE_NOOP if g.random() < 0.2 else int(g.integers(0, len(vals))) for _ in range(span)]
    for step in range(6):
        # Phase2a: one per (slot, server) per call, rounds 0 .. 3n
        cells = {(int(g.integers(0, span)), int(g.integers(0, n))) for _ in range(3 * span // 2)}
        p2a = np.zeros(len(cells), dtype=P2A)
        for k, (slot, s) in enumerate(sorted(cells, key=lambda c: g.random())):
            rnd = 0 if g.random() < 0.5 else int(g.integers(0, 3 * n))
            v = VALUE_NOOP if g.random() < 0.1 else int(g.integers(0, len(vals)))
            p2a[k] = (slot, rnd, v, s)
        rep = eng.vm_phase2a(p2a)
        for k, r in enumerate(p2a):
            want = model[r["dst"]].phase2a(int(r["slot"]), int(r["round"]), int(r["value_id"]))
            kind, w = int(rep[k]["group"]), int(rep[k]["round"])
            if want[0] == "chosen":
                assert (kind, w) == (4 if want[2] else 2, want[1])
            else:
                assert (kind, w) == ((0, want[1]) if want[0] == "phase2b" else (1, want[1]))
        # Chosen, some of them revocations
        ch = []
        for _ in range(span // 8):
            slot, s, rev = int(g.integers(0, span)), int(g.integers(0, n)), int(g.random() < 0.5)
            v = chosen_value[slot]                  # one value per slot, as safety guarantees
            ch.append((rev, s, slot, v))
            model[s].choose(slot, v, rev)
        eng.vm_choose(np.array(ch, dtype=P2B))
        # Phase1a: a few revocations, one CTA per server walks them in order
        msgs, servers = [], []
        for _ in range(int(g.integers(1, 3 * n))):
            revoked = int(g.integers(0, n))
            start = revoked + n * int(g.integers(0, span // n))
            stop = start + int(g.integers(-2, span // 2))
            msgs.append(phase1a_bytes(G, int(g.integers(0, 4 * n)), start, max(stop, 0)))
            servers.append(int(g.integers(0, n)))
        pos = int(g.integers(0, len(msgs) + 1))     # another member: a zero-length reply
        msgs.insert(pos, G.vcls("ServerInbound")(phase2b=G.vcls("Phase2b")(server_index=0, slot=1, round=0)).SerializeToString())
        servers.insert(pos, 0)
        kind, rec, buf = run_phase1a(eng, G, msgs, servers, next_slot)
        replies, skips = eng.vm_phase1a_wire(buf, kind, rec, next_slot, arena, voffs)
        for i, m in enumerate(msgs):
            if kind[i] != 2:
                assert replies[i] == b""
                continue
            si = G.vcls("ServerInbound")(); si.ParseFromString(m)
            want, skip = model[servers[i]].phase1a(si.phase1a.round, si.phase1a.start_slot_inclusive,
                                                   si.phase1a.stop_slot_exclusive)
            assert replies[i] == expected_reply(G, vals, servers[i], want), (step, i, want)
            if skip is not None:
                assert (skips[i]["slot_start"], skips[i]["slot_stop"]) == skip
            else:
                assert skips[i]["slot_start"] == skips[i]["slot_stop"]
        assert next_slot.tolist() == [model[s].next_slot for s in range(n)]
        check_entries(eng, model, n, span + 2 * n + span // 2 + 2)
    eng.close()


def test_self_revocation_fills_and_reports_the_skip(G):
    n = 3
    eng = Engine(1, 1, n, slot_capacity=CAP, max_batch=1 << 12, protocol=VANILLA_MENCIUS)
    model = [Server(s, n, next_slot=4 if s == 1 else s) for s in range(n)]
    eng.vm_phase2a(np.array([(1, 0, VALUE_NOOP, 1)], dtype=P2A)); model[1].phase2a(1, 0, VALUE_NOOP)
    next_slot = np.array([0, 4, 2], dtype=np.int32)
    kind, rec, buf = run_phase1a(eng, G, [phase1a_bytes(G, 4, 1, 11)], [1], next_slot)
    replies, skips = eng.vm_phase1a_wire(buf, kind, rec, next_slot)
    want, skip = model[1].phase1a(4, 1, 11)
    assert replies[0] == expected_reply(G, [], 1, want)
    assert tuple(skips[0]) == (1, 4, 11, 1) and next_slot.tolist() == [0, 13, 2]
    check_entries(eng, model, n, 16)
    eng.close()


def test_revocation_chosen_reply_bytes(G):
    n = 3
    eng = Engine(1, 1, n, slot_capacity=CAP, max_batch=1 << 12, protocol=VANILLA_MENCIUS)
    arena, voffs, vals = arena_of(G, np.random.default_rng(5), 2)
    eng.vm_choose(np.array([(1, 0, 7, 1), (0, 0, 8, VALUE_NOOP)], dtype=P2B))
    rep = eng.vm_phase2a(np.array([(7, 0, 0, 0), (8, 0, 0, 0)], dtype=P2A))
    assert rep["group"].tolist() == [4, 2] and rep["round"].tolist() == [1, VALUE_NOOP]
    out = V.split(*eng.wire_encode_vm_replies(rep, arena, voffs))
    C = G.vcls("ServerInbound")
    want = [C(chosen=G.vcls("Chosen")(slot=7, command_or_noop=vals[1], isRevocation=True)).SerializeToString(),
            C(chosen=G.vcls("Chosen")(slot=8, command_or_noop=cmd_or_noop(G, vals, VALUE_NOOP),
                                      isRevocation=False)).SerializeToString()]
    assert out == want
    eng.close()


def test_refusals_change_nothing(G):
    n = 3
    eng = Engine(1, 1, n, slot_capacity=CAP, max_batch=1 << 12, protocol=VANILLA_MENCIUS)
    eng.vm_phase2a(np.array([(0, 0, 1, 1), (3, 0, 2, 1)], dtype=P2A))
    before = [eng.vm_entries(s, 0, 16).copy() for s in range(n)]
    next_slot = np.array([0, 1, 2], dtype=np.int32)
    good = phase1a_bytes(G, 5, 0, 6)
    cases = [
        ([good, phase1a_bytes(G, 5, 0, CAP + 3)], [1, 1], -6, 1),            # beyond the window
        ([good, phase1a_bytes(G, 5, -3, 6)], [1, 1], -6, 1),                 # start < 0
        ([good, good], [1, 7], -1, 1),                                       # no such server
    ]
    for msgs, servers, status, idx in cases:
        kind, rec, buf = run_phase1a(eng, G, msgs, servers, next_slot)
        with pytest.raises(FpxError) as ex:
            eng.vm_phase1a_wire(buf, kind, rec, next_slot)
        assert (ex.value.status, ex.value.index) == (status, idx)
    # a truncated body: FPX_ERR_WIRE
    kind, rec, buf = run_phase1a(eng, G, [good, good], [1, 1], next_slot)
    rec = rec.copy(); rec[1]["d"] -= 1
    with pytest.raises(FpxError) as ex:
        eng.vm_phase1a_wire(buf, kind, rec, next_slot)
    assert (ex.value.status, ex.value.index) == (ERR_WIRE, 1)
    # a next_slot that is not its server's: FPX_ERR_INVALID_ARG
    kind, rec, buf = run_phase1a(eng, G, [phase1a_bytes(G, 5, 1, 7)], [1], next_slot)
    with pytest.raises(FpxError) as ex:
        eng.vm_phase1a_wire(buf, kind, rec, np.array([0, 2, 2], dtype=np.int32))
    assert ex.value.status == -1
    for s in range(n):
        assert np.array_equal(eng.vm_entries(s, 0, 16), before[s])
    eng.close()


def test_raised_entries_survive_the_batch_tag_wrap(G):
    n = 3
    eng = Engine(1, 1, n, slot_capacity=CAP, max_batch=1 << 12, protocol=VANILLA_MENCIUS)
    model = [Server(s, n) for s in range(n)]
    eng.vm_phase2a(np.array([(0, 0, 3, 2)], dtype=P2A)); model[2].phase2a(0, 0, 3)
    next_slot = np.array([0, 1, 2], dtype=np.int32)
    kind, rec, buf = run_phase1a(eng, G, [phase1a_bytes(G, 4, 0, 9)], [2], next_slot)
    eng.vm_phase1a_wire(buf, kind, rec, next_slot, *V.pack([b"\x0a\x00"] * 4))
    model[2].phase1a(4, 0, 9)
    eng.set_counters(vm_tag=0xffffffff - 2)
    for k in range(5):                              # across the wrap: lower rounds are nacked, the raise stays
        rep = eng.vm_phase2a(np.array([(0, 0, 1, 2), (3, 0, 1, 2)], dtype=P2A))
        assert rep["group"].tolist() == [1, 1]
    assert eng.counters()["vm_tag"] < 10
    check_entries(eng, model, n, 12)
    eng.close()


def test_other_engines_are_unsupported():
    e = Engine(1, 1, 3, slot_capacity=1 << 10, max_batch=1 << 10)
    with pytest.raises(FpxError) as ex:
        e.vm_entries(0, 0, 1)
    assert ex.value.status == -11
    e.close()


# --------------------------------------------------------------------------- golden vectors
def golden():
    import json
    with open(os.path.join(HERE, "golden", "wire_vm_revoke.json")) as f:
        return json.load(f)


@pytest.mark.parametrize("name", [c["name"] for c in golden()["cases"]])
def test_golden(name):
    d = golden()
    c = next(c for c in d["cases"] if c["name"] == name)
    n = d["n"]
    arena, voffs = V.pack([bytes.fromhex(h) for h in d["values_hex"]])
    eng = Engine(1, 1, n, slot_capacity=CAP, max_batch=1 << 12, protocol=VANILLA_MENCIUS)
    # one Phase2a per (slot, server) per call: deliver the setup records one call each
    for r in c["setup_phase2a"]:
        eng.vm_phase2a(np.array([tuple(r)], dtype=P2A))
    if c["setup_chosen"]:
        eng.vm_choose(np.array([tuple(r) for r in c["setup_chosen"]], dtype=P2B))
    msgs = [bytes.fromhex(m) for _, m in c["batch"]]
    buf, offs = V.pack(msgs)
    kind, rec, _ = eng.wire_decode_vm_server_inbound(buf, offs)
    rec = rec.copy(); rec["a"] = [s for s, _ in c["batch"]]
    next_slot = np.array(c["next_slot"], dtype=np.int32)
    replies, skips = eng.vm_phase1a_wire(buf, kind, rec, next_slot, arena, voffs)
    assert [r.hex() for r in replies] == c["replies"]
    for i, sk in enumerate(c["skips"]):
        if sk is not None:
            assert [int(skips[i]["slot_start"]), int(skips[i]["slot_stop"])] == sk
        else:
            assert skips[i]["slot_start"] == skips[i]["slot_stop"]
    assert next_slot.tolist() == c["next_slot_after"]
    for s in range(n):
        assert eng.vm_entries(s, 0, d["slots"]).tolist() == c["entries"][s], s
    eng.close()


# --------------------------------------------------------------------------- output capacity, device forms, retire
def revoke_setup(G, n=3):
    eng = Engine(1, 1, n, slot_capacity=CAP, max_batch=1 << 12, protocol=VANILLA_MENCIUS)
    arena, voffs, vals = arena_of(G, np.random.default_rng(9), 8)
    eng.vm_phase2a(np.array([(s, s % 4, s % 8, 1) for s in range(0, 60, 3)], dtype=P2A))
    eng.vm_choose(np.array([(1, 1, 9, 2), (0, 1, 12, VALUE_NOOP)], dtype=P2B))
    msgs = [phase1a_bytes(G, 5, 0, 60), phase1a_bytes(G, 2, 0, 30), phase1a_bytes(G, 6, 3, 40)]
    return eng, arena, voffs, vals, msgs, [1, 2, 1]


def test_output_one_short_of_capacity(G):
    a, arena, voffs, _, msgs, servers = revoke_setup(G)
    b, *_ = revoke_setup(G)
    kind, rec, buf = run_phase1a(a, G, msgs, servers, None)
    ns = np.array([0, 1, 2], dtype=np.int32)
    replies, _ = a.vm_phase1a_wire(buf, kind, rec, ns.copy(), arena, voffs)
    need = sum(len(r) for r in replies)
    with pytest.raises(FpxError) as ex:
        b.vm_phase1a_wire(buf, kind, rec, ns.copy(), arena, voffs, out_capacity=need - 1)
    assert ex.value.status == -1
    c, *_ = revoke_setup(G)
    assert c.vm_phase1a_wire(buf, kind, rec, ns.copy(), arena, voffs, out_capacity=need)[0] == replies
    for e in (a, b, c):
        e.close()


def test_device_forms_equal_host_forms(G):
    import torch
    dev = torch.device("cuda", 0)
    a, arena, voffs, _, msgs, servers = revoke_setup(G)
    b, *_ = revoke_setup(G)
    kind, rec, buf = run_phase1a(a, G, msgs, servers, None)
    ns = np.array([0, 1, 2], dtype=np.int32)
    replies, skips = a.vm_phase1a_wire(buf, kind, rec, ns, arena, voffs)
    n, cap = len(msgs), 1 << 16

    def dev_of(x):
        return torch.from_numpy(np.ascontiguousarray(x).view(np.uint8).reshape(-1).copy()).to(dev)
    d_buf, d_kind, d_rec, d_arena = dev_of(np.frombuffer(bytes(buf) + b"\0", np.uint8)), dev_of(kind), dev_of(rec), \
        dev_of(np.frombuffer(bytes(arena) + b"\0", np.uint8))
    d_voffs, d_ns = dev_of(voffs), dev_of(np.array([0, 1, 2], dtype=np.int32))
    d_out = torch.zeros(cap, dtype=torch.uint8, device=dev)
    d_offs = torch.zeros(n + 1, dtype=torch.int32, device=dev)
    d_skips = torch.zeros((n, 4), dtype=torch.int32, device=dev)
    b.vm_phase1a_wire_dev(d_buf.data_ptr(), len(buf), d_kind.data_ptr(), d_rec.data_ptr(), n, d_arena.data_ptr(),
                          d_voffs.data_ptr(), len(voffs) - 1, d_ns.data_ptr(), d_out.data_ptr(), cap,
                          d_offs.data_ptr(), d_skips.data_ptr())
    torch.cuda.synchronize()
    out, offs = d_out.cpu().numpy(), d_offs.cpu().numpy()
    assert [out[offs[i]:offs[i + 1]].tobytes() for i in range(n)] == replies
    assert np.array_equal(d_skips.cpu().numpy().reshape(-1), skips.view(np.int32).reshape(-1))
    assert d_ns.cpu().numpy().view(np.int32).tolist() == ns.tolist()
    # fpx_vm_choose_dev
    ch = np.array([(1, 0, 30, 3), (0, 2, 33, VALUE_NOOP), (1, 2, 33, VALUE_NOOP)], dtype=P2B)
    a.vm_choose(ch)
    b.vm_choose_dev(dev_of(ch).data_ptr(), len(ch))
    torch.cuda.synchronize()
    for s in range(3):
        assert np.array_equal(a.vm_entries(s, 0, 64), b.vm_entries(s, 0, 64))
    a.close(); b.close()


def test_revocation_across_retire_below(G):
    from frankenpaxos_b200 import CHOSEN
    n = 3
    eng = Engine(1, 1, n, slot_capacity=CAP, max_batch=1 << 12, protocol=VANILLA_MENCIUS)
    next_slot = np.array([0, 1, 2], dtype=np.int32)
    kind, rec, buf = run_phase1a(eng, G, [phase1a_bytes(G, 4, 0, 30)], [1], None)
    eng.vm_phase1a_wire(buf, kind, rec, next_slot)
    assert eng.vm_entries(1, 0, 30)[::3, 0].tolist() == [1] * 10          # voteless, raised
    eng.replica_chosen(np.array([(s, VALUE_NOOP) for s in range(12)], dtype=CHOSEN))
    assert eng.chosen_watermark() >= 12             # the scan publishes the executed prefix retire_below checks
    eng.retire_below(12)
    # a range that reaches a retired slot is refused and changes nothing
    before = eng.vm_entries(1, 12, 30).copy()
    kind, rec, buf = run_phase1a(eng, G, [phase1a_bytes(G, 5, 12, 30), phase1a_bytes(G, 5, 9, 30)], [1, 1], None)
    with pytest.raises(FpxError) as ex:
        eng.vm_phase1a_wire(buf, kind, rec, next_slot)
    assert (ex.value.status, ex.value.index) == (-6, 1)
    assert np.array_equal(eng.vm_entries(1, 12, 30), before)
    with pytest.raises(FpxError):
        eng.vm_entries(1, 0, 12)
    # the recycled ring positions serve slots one window ahead: no raise leaks into them
    assert eng.vm_entries(1, CAP, 12)[:, 0].tolist() == [0] * 12
    kind, rec, buf = run_phase1a(eng, G, [phase1a_bytes(G, 3, CAP, CAP + 12)], [1], None)
    replies, _ = eng.vm_phase1a_wire(buf, kind, rec, next_slot)
    assert replies[0] == expected_reply(G, [], 1, ("phase1b", 3, CAP, CAP + 12, []))
    eng.close()


# --------------------------------------------------------------------------- cfg5 scale
@pytest.mark.parametrize("suspected", [False, True])
def test_cfg5_scale_revocation_of_server_3(G, suspected):
    """n = 7, 2^20 slots; server 3 stops (or is only suspected and keeps a round-0 Phase 2 in flight).  The f + 1
    survivors 0, 1, 2, 4 answer a Phase1a over 2^17 of server 3's slots; their replies and entries equal the model's."""
    n, f, cap = 7, 3, 1 << 20
    g = np.random.default_rng(3 + suspected)
    arena, voffs, vals = arena_of(G, g, 32)
    eng = Engine(f, 1, n, slot_capacity=cap, max_batch=1 << 20, protocol=VANILLA_MENCIUS)
    survivors = [0, 1, 2, 4]
    model = {s: Server(s, n) for s in survivors + [3]}
    walked = 1 << 17
    start, stop = 3, 3 + n * walked
    slots = np.arange(start, stop, n)
    # server 3's Phase2as reached some survivors before it stopped
    p2a = []
    for s in survivors:
        hit = slots[g.random(len(slots)) < 0.3]
        v = g.integers(0, len(vals), size=len(hit))
        p2a.append(np.rec.fromarrays([hit, np.zeros(len(hit)), v, np.full(len(hit), s)], dtype=P2A))
    p2a = np.concatenate(p2a).view(P2A)
    eng.vm_phase2a(p2a)
    for r in p2a:
        model[int(r["dst"])].phase2a(int(r["slot"]), 0, int(r["value_id"]))
    rnd = n + 1                                     # a revocation round of server 1
    msgs = [phase1a_bytes(G, rnd, start, stop)] * len(survivors)
    next_slot = np.arange(n, dtype=np.int32) + n * (stop // n + 1)
    for s in survivors:
        model[s].next_slot = int(next_slot[s])
    kind, rec, buf = run_phase1a(eng, G, msgs, survivors, None)
    replies, _ = eng.vm_phase1a_wire(buf, kind, rec, next_slot, arena, voffs)
    for i, s in enumerate(survivors):
        want, _ = model[s].phase1a(rnd, start, stop)
        assert replies[i] == expected_reply(G, vals, s, want), s
    if suspected:
        # server 3 was alive: its round-0 Phase2as arrive after the raise and are nacked; the votes stay intact
        late = slots[g.random(len(slots)) < 0.2]
        lp = np.rec.fromarrays([late, np.zeros(len(late)), np.full(len(late), 5), np.full(len(late), 0)], dtype=P2A)
        rep = eng.vm_phase2a(lp.view(P2A))
        assert set(rep["group"].tolist()) == {1} and set(rep["round"].tolist()) == {rnd}
        for r in lp:
            model[0].phase2a(int(r["slot"]), 0, 5)
    for s in survivors:
        got = eng.vm_entries(s, start, stop - start)[::n]
        want = np.array([model[s].entry_row(int(x)) for x in slots], dtype=np.int32)
        assert np.array_equal(got, want), s
    eng.close()
