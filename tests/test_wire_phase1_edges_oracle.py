"""CPU checks of the Phase 1 edge builders (tests/wire_phase1_edges.py): the protobuf runtime parses every built
message to the fields it claims, each claimed header sits where the builder says relative to the walk's window, the
padded varints decode to their values, and the leaders' CPU oracles agree with the reference's fill-in over the
runtime's parse on these batches.  The mirrored kernel constants are read back from the CUDA sources."""
import os
import re

import numpy as np
import pytest

import wire_mencius_phase1_cases as MW
import wire_mencius_phase1_oracle as MO
import wire_phase1_edges as E
import wire_phase1_oracle as O
from test_wire_phase1_oracle import runtime

CSRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "frankenpaxos_b200", "csrc")


def src(name):
    return open(os.path.join(CSRC, name)).read()


def const(text, name):
    m = re.search(r"constexpr\s+(?:int|int32_t|uint32_t)\s+" + name + r"\s*=\s*([^;]+);", text)
    assert m, name
    return m.group(1)


def test_constants_match_the_kernels():
    p1, vm, wire, scan, inc = (src(n) for n in ("fpx_wire_phase1.cuh", "fpx_vm_revoke.cuh", "fpx_wire.cuh",
                                                "fpx_scan.cuh", "fpx_engine_wire_phase1.inc"))
    assert eval(const(p1, "kP1Window")) == E.P1_WINDOW
    assert int(const(p1, "kP1Threads")) == E.P1_THREADS
    assert int(const(p1, "kP1MinInfo")) == E.P1_MIN_INFO
    assert int(const(p1, "kP1aTile")) == E.P1A_TILE
    assert int(const(vm, "kVmP1aThreads")) == E.VM_P1A_THREADS
    assert re.search(r"wend - p < (\d+)\)", p1).group(1) == str(E.HEADER_MAX)
    per, thr = int(const(wire, "kWireEncPer")), int(const(wire, "kWireEncThreads"))
    assert const(wire, "kWireEncTile").replace(" ", "") == "kWireEncPer*kWireEncThreads" and per * thr == E.ENC_TILE
    assert re.search(r"base < m; base \+= 1024 \* 4\)", scan) and E.SCAN_CHUNK == 1024 * 4
    assert re.search(r"const dim3 grid\((\d+), \(unsigned\)std::min\(n, (\d+)\)\);", inc).groups() == \
        (str(E.PARSE_CTAS), str(E.GRID_Y))
    assert re.search(r"kP1Threads, (\d+)\)\), kP1Threads", inc).group(1) == str(E.EMIT_CTAS)
    assert len(re.findall(r"n > (\d+) \|\|", inc)) == 2 and set(re.findall(r"n > (\d+) \|\|", inc)) == {str(E.P1A_MAX_N)}
    # tiles of the acceptor's scan: the live window's slots of one residue, plus one
    assert "(e->g.local_slots / stride + 1 + kP1aTile - 1) / kP1aTile" in inc
    hdr = open(os.path.join(CSRC, "..", "..", "include", "fpx.h")).read()
    for name in ("INVALID_ARG", "BAD_ACCEPTOR", "SLOT_RANGE", "CHECK_FAILED", "WIRE"):
        assert int(re.search(r"FPX_ERR_" + name + r" = (-\d+)", hdr).group(1)) == getattr(E, "ERR_" + name)


def runtime_parse(mk):
    """parse(raw) for E.python_fill_in over the protobuf runtime `mk` (MultiPaxos or Mencius LeaderInbound)"""
    def parse(raw):
        m = mk.cls("LeaderInbound")()
        try:
            m.ParseFromString(raw)
        except Exception:
            return "bad", 0, 0, 0, []
        if not m.IsInitialized():         # Java's parseFrom checks required fields
            return "bad", 0, 0, 0, []
        if m.WhichOneof("request") != "phase1b":
            return 0, 0, 0, 0, []
        p = m.phase1b
        return 1, p.group_index, p.acceptor_index, p.round, [(x.slot, x.vote_round, x.vote_value.SerializeToString())
                                                             for x in p.info]
    return parse


def mp_parse(mk):
    return runtime_parse(mk)


def mencius_parse():
    return runtime_parse(MW.runtime())


def split(buf, offs):
    return [bytes(buf[offs[i]: offs[i + 1]]) for i in range(len(offs) - 1)]


def mp_agrees(buf, offs, cw, round_=9, f=1, groups=1, per_group=3, parse=None):
    """fpo_leader_phase1b against the fill-in over the runtime's parse -> the oracle's status"""
    st, idx, complete, max_slot, recs, spans = O.leader_phase1b(f, groups, per_group, 0, round_, cw, buf, offs, 40,
                                                                1 << 16)
    est, ei, res = E.python_fill_in(split(buf, offs), parse, groups, per_group, f, round_, cw)
    if est != 0:
        assert (st, idx) == (est, ei)
        return st
    assert st == 0 and complete == ei
    if res is None:
        assert len(recs) == 0
        return st
    assert max_slot == res[0] and len(recs) == len(res[2])
    for k, (slot, val) in enumerate(res[2]):
        assert recs[k]["slot"] == slot
        got = None if recs[k]["value_id"] == O.VALUE_NOOP else bytes(buf[spans[k, 0]: spans[k, 0] + spans[k, 1]])
        assert got == val, k
    return st


@pytest.mark.parametrize("target", ["info", "scalar", "member"])
@pytest.mark.parametrize("d", E.WINDOW_DISTANCES)
def test_window_edge_builders(d, target):
    mk = runtime()
    parse = mp_parse(mk)
    g = np.random.default_rng(d + 50)
    for tag_w, len_w in [(1, 0), (5, 10), (10, 10)]:
        for lead in (0, 33):
            buf, offs, m, pos, head, infos = E.window_batch(d, target, tag_w, len_w or None, lead, g)
            assert offs[-1] % 16 == 7
            lo = int(offs[m])
            assert pos - ((lo & ~15) + E.P1_WINDOW) == -d                      # where the claimed header sits
            assert buf[pos: pos + len(head)].tobytes() == head
            t, p = E.read_varint(head, 0)
            assert t == {"info": 0x22, "scalar": 0x18, "member": 0x0a}[target] and p == tag_w
            v, p = E.read_varint(head, p)
            assert p == len(head) and (len_w == 0 or len(head) == tag_w + len_w)
            if target == "scalar":
                assert v == 9
            if tag_w > 5:                 # beyond the runtime's tag limit: the oracle alone (Java takes ten bytes)
                continue
            kind, grp, acc, rnd, got = parse(bytes(buf[lo: offs[m + 1]]))
            assert (kind, grp, acc, rnd) == (1, 0, 0, 9) and got == infos
            assert mp_agrees(buf, offs, 0, parse=parse) == 0


@pytest.mark.parametrize("case", sorted(E.oneof_cases()))
def test_oneof_cases(case):
    mk = runtime()
    parse = mp_parse(mk)
    msg, want = E.oneof_cases()[case]
    kind, grp, acc, rnd, infos = parse(msg)
    if want == "bad":
        assert kind == "bad"
    elif want is None:
        assert kind == 0
    else:
        assert kind == 1 and (grp, acc, rnd, infos) == want[:3] + ([(s, r, v) for s, r, v in want[3]],)
    buf, offs = E.oneof_batch(msg)
    assert mp_agrees(buf, offs, 0, parse=parse) == (E.ERR_WIRE if want == "bad" else 0)
    # the Mencius leader: nack is member 7
    mparse = mencius_parse()
    msg, want = E.oneof_cases(nack=7)[case]
    assert (mparse(msg)[0] == "bad") == (want == "bad")
    buf, offs = E.oneof_batch(msg)
    mencius_agrees(buf, offs, 0, 0, -1, mparse, lgroups=1, agroups=1)


def mencius_agrees(buf, offs, leader_group, cw, recover_slot, parse, f=1, lgroups=3, agroups=2, round_=9):
    st, idx, complete, max_slot, next_slot, recs, spans = MO.leader_phase1b(
        f, lgroups, agroups, 2 * f + 1, leader_group, round_, cw, buf, offs, recover_slot, 40, 1 << 16)
    est, ei, res = E.python_fill_in(split(buf, offs), parse, agroups, 2 * f + 1, f, round_, cw, lgroups, leader_group,
                                    recover_slot)
    if est != 0:
        assert (st, idx) == (est, ei)
        return st
    assert st == 0 and complete == ei
    if res is None:
        assert len(recs) == 0
        return st
    assert (max_slot, next_slot, len(recs)) == (res[0], res[1], len(res[2]))
    for k, (slot, val) in enumerate(res[2]):
        assert recs[k]["slot"] == slot
        got = None if recs[k]["value_id"] == O.VALUE_NOOP else bytes(buf[spans[k, 0]: spans[k, 0] + spans[k, 1]])
        assert got == val, k
    return st


def test_tight_batches_take_every_offset():
    mk = runtime()
    parse = mp_parse(mk)
    seen = set()
    for lead in range(16):
        g = np.random.default_rng(lead)
        buf, offs = E.tight_batch(lead, g)
        seen |= {int(o) % E.P1_MIN_INFO for o in offs[:-1]}
        for i in range(len(offs) - 1):
            raw = bytes(buf[offs[i]: offs[i + 1]])
            kind, _, _, _, infos = parse(raw)
            assert kind == 1
            # nothing but the scalars and 8-byte infos: the most infos a message of this size can hold
            assert len(raw) - E.width_of(len(raw)) - 1 - 6 == E.P1_MIN_INFO * len(infos)
        assert mp_agrees(buf, offs, 0, f=2, per_group=5, parse=parse) == 0
    assert seen == set(range(E.P1_MIN_INFO))


@pytest.mark.parametrize("case", sorted(E.mp_slot_cases()))
def test_mp_slot_cases(case):
    msgs, cw = E.mp_slot_cases()[case]
    buf, offs = O.pack(msgs)
    for raw in msgs:                      # ten-byte varints for negative slots, as the runtime writes them
        m = runtime().cls("LeaderInbound")()
        m.ParseFromString(raw)
        assert m.SerializeToString() == raw
    assert mp_agrees(buf, offs, cw, parse=mp_parse(runtime())) == 0


@pytest.mark.parametrize("case", sorted(E.mencius_slot_cases()))
def test_mencius_slot_cases(case):
    lg, cw, rec, msgs = E.mencius_slot_cases()[case]
    buf, offs = O.pack(msgs)
    st = mencius_agrees(buf, offs, lg, cw, rec, mencius_parse())
    assert st == E.MENCIUS_SLOT_STATUS.get(case, 0)


def test_cross_group_votes_are_not_read():
    """safeValue reads phase1bs(slot % numAcceptorGroups) only: group 1's higher votes on group 0's slots count
    toward max_slot and nothing else"""
    msgs = E.cross_group_mp()
    buf, offs = O.pack(msgs)
    assert mp_agrees(buf, offs, 0, groups=2, parse=mp_parse(runtime())) == 0
    st, _, complete, max_slot, recs, spans = O.leader_phase1b(1, 2, 3, 0, 9, 0, buf, offs, 40, 64)
    assert (complete, max_slot, len(recs)) == (3, 6, 7) and recs["value_id"][6] == O.VALUE_NOOP
    assert all(bytes(buf[spans[k, 0]: spans[k, 0] + spans[k, 1]]) == E.VALUES[1] for k in (0, 2, 4))


def test_padded_varints():
    for v in (0, 1, 127, 128, 16383, 1 << 21, E.INT_MAX, (1 << 64) - 1):
        for w in range(len(E.venc(v)), 11):
            b = E.pvenc(v, w)
            assert len(b) == w and E.read_varint(b, 0) == (v, w)


def test_body_length_solvers():
    for body in E.BODY_EDGES:
        vlen = E.phase1b_value_len(body, 0, 0, 5, 0, 1)
        ib = E.info_body(0, 1, bytes(vlen))
        assert len(E.scalars(0, 0, 5) + E.field(4, ib)) == body
        assert E.vm_phase1b_value_len(body, 1, 5, 0, 3, 0, 1) is not None
