"""GPU wire codec of EPaxos (fpx_epaxos_wire_decode / _pack): the golden vectors, the CPU oracle
(tests/wire_ep_oracle.cc) on random and mutated messages, the device forms against the host forms, a failing
decode refusing the calls queued behind it, and BASELINE cfg4 rounds from protobuf bytes through the handlers."""
import json
import os

import numpy as np
import pytest
import torch

from frankenpaxos_b200 import FpxError
from frankenpaxos_b200 import traces as T
from frankenpaxos_b200.epaxos import (CALL_ACCEPT, CALL_ACCEPTOK, CALL_COMMIT, CALL_PREACCEPT, CALL_PREACCEPTOK,
                                      CALL_PREPARE, EpaxosReplica)
from epaxos_recovery_traces import CALLS, Trace
import wire_ep_oracle as W

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
CASES = json.load(open(os.path.join(HERE, "golden", "wire_epaxos.json")))["cases"]
DEV = torch.device("cuda", 0)


@pytest.fixture(scope="module")
def G():
    return W.golden_module()


def decode_both(eng, raws, n, base=0):
    """(GPU (status, err, kind, rows, values), oracle's)"""
    buf, offs = W.pack(raws)
    try:
        kind, rows, values = eng.wire_decode(buf, offs, base)
        gpu = (0, -1, kind, rows, values)
    except FpxError as e:
        gpu = (e.status, e.index, None, None, None)
    return gpu, W.decode(buf, offs, n, base)


def test_golden_decode():
    eng = EpaxosReplica(1, 0, 64, max_batch=1 << 10)
    raws = [bytes.fromhex(c["hex"]) for c in CASES]
    ok = [r for r, c in zip(raws, CASES) if c["status"] == W.OK]
    (st, _, kind, rows, values), (ost, _, okind, orows, ovalues) = decode_both(eng, ok, 3, 5)
    assert st == ost == 0
    assert np.array_equal(kind, okind) and np.array_equal(rows, orows) and np.array_equal(values, ovalues)
    for c in CASES:                                       # one at a time: every status, and the handle recovers
        (st, err, *_), (ost, oerr, *_) = decode_both(eng, [bytes.fromhex(c["hex"])], 3)
        assert (st, err) == (ost, oerr) == (c["status"], -1 if c["status"] == 0 else 0), c.get("name", c["type"])
    eng.close()


@pytest.mark.parametrize("f", [1, 2, 3])
def test_random_and_mutated_batches_match_the_oracle(G, f):
    n = 2 * f + 1
    eng = EpaxosReplica(f, 0, 64, max_batch=1 << 10)
    g = np.random.Generator(np.random.PCG64(100 + f))
    msgs = [W.random_message(G, g, n).SerializeToString() for _ in range(3000)]
    buf, offs = W.pack(msgs)
    kind, rows, values = eng.wire_decode(buf, offs, 11)
    st, _, okind, orows, ovalues = W.decode(buf, offs, n, 11)
    assert st == 0
    assert np.array_equal(kind, okind) and np.array_equal(rows, orows) and np.array_equal(values, ovalues)
    for trial in range(20):
        mm = list(msgs[:800])
        for j in g.choice(len(mm), size=int(g.integers(1, 6)), replace=False):
            mm[j] = W.mutate(mm[j], g)
        (gst, gerr, *_), (ost, oerr, *_) = decode_both(eng, mm, n)
        assert (gst, gerr) == (ost, oerr), trial
    eng.close()


def dev_i32(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.int32)).to(DEV)


def test_device_forms_equal_host_forms(G):
    f, n = 2, 5
    eng = EpaxosReplica(f, 0, 64, max_batch=1 << 12)
    g = np.random.Generator(np.random.PCG64(5))
    msgs = [W.random_message(G, g, n).SerializeToString() for _ in range(2000)]
    buf, offs = W.pack(msgs)
    kind, rows, values = eng.wire_decode(buf, offs, 40)
    m = len(msgs)
    d_buf, d_offs = torch.from_numpy(buf).to(DEV), dev_i32(offs)
    d_kind = torch.empty(m, dtype=torch.int32, device=DEV)
    d_rows = torch.empty((m, 12 + n), dtype=torch.int32, device=DEV)
    d_values = torch.empty((m, 2), dtype=torch.int32, device=DEV)
    eng.wire_decode_dev(d_buf.data_ptr(), d_offs.data_ptr(), m, 40, d_kind.data_ptr(), d_rows.data_ptr(),
                        d_values.data_ptr())
    eng.sync()
    assert np.array_equal(d_kind.cpu().numpy(), kind) and np.array_equal(d_rows.cpu().numpy(), rows)
    assert np.array_equal(d_values.cpu().numpy(), values)
    idx = np.nonzero(kind == 3)[0]                        # a run of PreAcceptOks from its first one
    first, count = int(idx[0]), 1
    while first + count < m and kind[first + count] == 3:
        count += 1
    host = eng.wire_pack(CALL_PREACCEPTOK, kind, rows, first, count)
    d_out = torch.empty((count, 6 + n), dtype=torch.int32, device=DEV)
    eng.wire_pack_dev(CALL_PREACCEPTOK, d_kind.data_ptr(), d_rows.data_ptr(), first, count, 0, d_out.data_ptr())
    eng.sync()
    assert np.array_equal(d_out.cpu().numpy(), host)
    assert np.array_equal(host, W.pack_rows(CALL_PREACCEPTOK, kind, rows, first, count, n)[2])
    eng.close()


def test_pack_errors_are_the_batchs_indices(G):
    eng = EpaxosReplica(1, 0, 64, max_batch=1 << 10)
    c = next(c for c in CASES if c["type"] == "pre_accept.overflow_packed")
    pa = next(c for c in CASES if c["type"] == "pre_accept")
    buf, offs = W.pack([bytes.fromhex(pa["hex"]), bytes.fromhex(pa["hex"]), bytes.fromhex(c["hex"])])
    kind, rows, _ = eng.wire_decode(buf, offs)
    with pytest.raises(FpxError) as ei:
        eng.wire_pack(CALL_PREACCEPT, kind, rows, 1, 2)
    assert (ei.value.status, ei.value.index) == (W.UNSUPPORTED, 2)
    with pytest.raises(FpxError) as ei:
        eng.wire_pack(CALL_ACCEPT, kind, rows, 0, 3)
    assert (ei.value.status, ei.value.index) == (W.INVALID_ARG, 0)
    with pytest.raises(FpxError) as ei:
        eng.wire_pack(0, kind, rows, 0, 1)                # lead takes no decoded rows
    assert ei.value.status == W.INVALID_ARG
    assert eng.wire_pack(CALL_PREACCEPT, kind, rows, 0, 2).shape == (2, 12)
    eng.close()


def test_failed_decode_refuses_the_calls_queued_behind_it(G):
    f, n, N = 1, 3, 600
    lead, pa, _ = T.epaxos_cfg4(3, f=f, n_instances=N, me=0)
    eng = EpaxosReplica(f, 0, N // n + 2, max_batch=1 << 12)
    eng.lead(lead)
    raws = W.preaccept_messages(G, pa, n)
    bad = 17
    raws[bad] = raws[bad][:-3]                            # truncated
    buf, offs = W.pack(raws)
    m = len(raws)
    d_buf, d_offs = torch.from_numpy(buf).to(DEV), dev_i32(offs)
    d_kind = torch.empty(m, dtype=torch.int32, device=DEV)
    d_rows = torch.empty((m, 12 + n), dtype=torch.int32, device=DEV)
    d_values = torch.empty((m, 2), dtype=torch.int32, device=DEV)
    d_in = dev_i32(pa)
    d_reply = torch.zeros((m, 4 + n), dtype=torch.int32, device=DEV)
    probe = [tuple(r) for r in pa[:, :2][::37].tolist()]
    before = [eng.entry(*p) for p in probe]
    eng.wire_decode_dev(d_buf.data_ptr(), d_offs.data_ptr(), m, 0, d_kind.data_ptr(), d_rows.data_ptr(),
                        d_values.data_ptr())
    eng.preaccept_dev(d_in.data_ptr(), m, d_reply.data_ptr())
    with pytest.raises(FpxError) as ei:
        eng.sync()
    assert (ei.value.status, ei.value.index) == (W.WIRE, bad)
    after = [eng.entry(*p) for p in probe]
    for (a, la, ba), (b, lb, bb) in zip(before, after):
        assert np.array_equal(a, b) and la == lb and np.array_equal(ba, bb)
    assert not d_reply.any()
    # collected: the same handler call now applies
    eng.preaccept_dev(d_in.data_ptr(), m, d_reply.data_ptr())
    eng.sync()
    ref = EpaxosReplica(f, 0, N // n + 2, max_batch=1 << 12)
    ref.lead(lead)
    assert np.array_equal(d_reply.cpu().numpy(), ref.preaccept(pa))
    eng.close(); ref.close()


def wire_round(G, eng, raws, call, n, base, local_deps=None):
    """bytes -> decode_dev -> pack_dev on the handle's stream; returns the packed rows (device)"""
    buf, offs = W.pack(raws)
    m = len(raws)
    d_buf, d_offs = torch.from_numpy(buf).to(DEV), dev_i32(offs)
    d_kind = torch.empty(m, dtype=torch.int32, device=DEV)
    d_rows = torch.empty((m, 12 + n), dtype=torch.int32, device=DEV)
    d_values = torch.empty((m, 2), dtype=torch.int32, device=DEV)
    width = {CALL_PREACCEPT: 6 + 2 * n, CALL_PREACCEPTOK: 6 + n, CALL_ACCEPT: 6 + n, CALL_ACCEPTOK: 6}[call]
    d_out = torch.empty((m, width), dtype=torch.int32, device=DEV)
    d_ld = dev_i32(local_deps) if local_deps is not None else None
    eng.wire_decode_dev(d_buf.data_ptr(), d_offs.data_ptr(), m, base, d_kind.data_ptr(), d_rows.data_ptr(),
                        d_values.data_ptr())
    eng.wire_pack_dev(call, d_kind.data_ptr(), d_rows.data_ptr(), 0, m, 0 if d_ld is None else d_ld.data_ptr(),
                      d_out.data_ptr())
    return d_out, (d_buf, d_offs, d_kind, d_rows, d_values, d_ld)


def cfg4_from_bytes(G, seed, f, N):
    n = 2 * f + 1
    lead, pa, ok = T.epaxos_cfg4(seed, f=f, n_instances=N, me=0)
    pa = pa.copy()
    base = 1 << 20
    pa[:, 4] = base + np.arange(len(pa))                  # the value ids the decoder hands out: base + index
    wire = EpaxosReplica(f, 0, N // n + 2, max_batch=max(len(pa), len(ok)))
    direct = EpaxosReplica(f, 0, N // n + 2, max_batch=max(len(pa), len(ok)))
    wire.lead(lead); direct.lead(lead)
    # PreAccepts: decoded, packed with the conflict index's answers, handled on the device
    d_in, keep = wire_round(G, wire, W.preaccept_messages(G, pa, n), CALL_PREACCEPT, n, base, pa[:, 6:6 + n])
    d_reply = torch.empty((len(pa), 4 + n), dtype=torch.int32, device=DEV)
    wire.preaccept_dev(d_in.data_ptr(), len(pa), d_reply.data_ptr())
    wire.sync()
    assert np.array_equal(d_in.cpu().numpy(), pa)
    assert np.array_equal(d_reply.cpu().numpy(), direct.preaccept(pa))
    # PreAcceptOks answering this replica's instances
    d_in2, keep2 = wire_round(G, wire, W.preacceptok_messages(G, ok, n), CALL_PREACCEPTOK, n, 0)
    d_ev = torch.empty((len(ok), 2 + n), dtype=torch.int32, device=DEV)
    wire.preacceptok_dev(d_in2.data_ptr(), len(ok), d_ev.data_ptr())
    wire.sync()
    assert np.array_equal(d_in2.cpu().numpy(), ok)
    assert np.array_equal(d_ev.cpu().numpy(), direct.preacceptok(ok))
    # the replies and events back to bytes, on the device, against the runtime's serialisation of the same messages
    arena, voffs = W.value_arena(base + len(pa) + 1)
    d_arena, d_voffs = torch.from_numpy(arena).to(DEV), dev_i32(voffs)
    value = {(int(r[0]), int(r[1])): int(r[4]) for r in np.concatenate([lead[:, :5], pa[:, :5]])}
    cmd_value = lambda rep, num: value[(rep, num)]      # noqa: E731

    def encode_dev(handle, call, d_in, d_rows, m):
        cap = m * (128 + 14 * n) + 16
        d_out = torch.empty(cap, dtype=torch.uint8, device=DEV)
        d_offs = torch.empty(m + 1, dtype=torch.int32, device=DEV)
        handle.wire_encode_dev(call, d_in.data_ptr(), d_rows.data_ptr(), m, d_arena.data_ptr(), d_voffs.data_ptr(),
                               len(voffs) - 1, d_out.data_ptr(), cap, d_offs.data_ptr())
        handle.sync()
        offs = d_offs.cpu().numpy()
        return W.split(d_out[:int(offs[-1])].cpu().numpy(), offs)

    assert encode_dev(wire, CALL_PREACCEPT, d_in, d_reply, len(pa)) == \
        W.expected_encode(G, CALL_PREACCEPT, pa, d_reply.cpu().numpy(), n, 0, cmd_value)
    events = d_ev.cpu().numpy()
    accepts = encode_dev(wire, CALL_PREACCEPTOK, d_in2, d_ev, len(ok))
    assert accepts == W.expected_encode(G, CALL_PREACCEPTOK, ok, events, n, 0, cmd_value)
    # the slow path: Accept to f other replicas, their AcceptOks back, the Commits out
    slow = [i for i in range(len(ok)) if events[i, 0] == 2]
    if slow:
        acc_bytes = [accepts[i] for i in slow]
        acc_rows = np.concatenate([ok[slow, :4], [[value[(int(r[0]), int(r[1]))]] for r in ok[slow]],
                                   events[slow, 1:2], events[slow, 2:]], axis=1).astype(np.int32)
        oks, ok_rows = [], []
        for q in range(1, f + 1):
            peer = EpaxosReplica(f, q, N // n + 2, max_batch=len(slow))
            d_acc, keep3 = wire_round(G, peer, acc_bytes, CALL_ACCEPT, n, base)
            d_rep = torch.empty((len(slow), 4 + n), dtype=torch.int32, device=DEV)
            peer.accept_dev(d_acc.data_ptr(), len(slow), d_rep.data_ptr())
            peer.sync()
            got = d_acc.cpu().numpy()
            assert np.array_equal(got[:, [0, 1, 2, 3, 5]], acc_rows[:, [0, 1, 2, 3, 5]])
            assert np.array_equal(got[:, 6:], acc_rows[:, 6:])
            rep = d_rep.cpu().numpy()
            b = encode_dev(peer, CALL_ACCEPT, d_acc, d_rep, len(slow))
            assert b == W.expected_encode(G, CALL_ACCEPT, got, rep, n, q, lambda *a: 0)
            oks += [x for x, r in zip(b, rep) if r[0] == 1]
            ok_rows += [[r0[0], r0[1], r[1], r[2], q, 0] for r0, r in zip(got, rep) if r[0] == 1]
            peer.close()
        ok_rows = np.array(ok_rows, dtype=np.int32).reshape(-1, 6)
        d_aok, keep4 = wire_round(G, wire, oks, CALL_ACCEPTOK, n, 0)
        d_ev2 = torch.empty((len(oks), 2 + n), dtype=torch.int32, device=DEV)
        wire.acceptok_dev(d_aok.data_ptr(), len(oks), d_ev2.data_ptr())
        wire.sync()
        assert np.array_equal(d_aok.cpu().numpy(), ok_rows)
        ev2 = d_ev2.cpu().numpy()
        assert np.array_equal(ev2, direct.acceptok(ok_rows))
        assert encode_dev(wire, CALL_ACCEPTOK, d_aok, d_ev2, len(oks)) == \
            W.expected_encode(G, CALL_ACCEPTOK, ok_rows, ev2, n, 0, cmd_value)
    g = np.random.Generator(np.random.PCG64(seed))
    for r in np.concatenate([pa[:, :2], ok[:, :2]])[g.choice(len(pa) + len(ok), size=200)]:
        a, b = wire.entry(int(r[0]), int(r[1])), direct.entry(int(r[0]), int(r[1]))
        assert np.array_equal(a[0], b[0]) and a[1] == b[1] and np.array_equal(a[2], b[2])
    wire.close(); direct.close()


@pytest.mark.parametrize("seed", [0, 1, 2])
@pytest.mark.parametrize("f", [1, 2, 3])
def test_cfg4_round_from_bytes(G, seed, f):
    cfg4_from_bytes(G, seed, f, 6000)


def test_cfg4_round_from_bytes_at_scale(G):
    cfg4_from_bytes(G, 0, 2, 1 << 20)


def test_prepare_rows_from_bytes(G):
    """Prepare messages decode and pack to the rows fpx_epaxos_prepare takes"""
    f, n = 2, 5
    eng = EpaxosReplica(f, 1, 64, max_batch=1 << 10)
    rows = np.array([[r % n, r, 3 + r, (r + 1) % n] for r in range(40)], dtype=np.int32)
    raws = []
    for r in rows.tolist():
        m = G.RI(); m.prepare.instance.replica_index, m.prepare.instance.instance_number = r[:2]
        m.prepare.ballot.ordering, m.prepare.ballot.replica_index = r[2:]
        raws.append(m.SerializeToString())
    buf, offs = W.pack(raws)
    kind, drows, _ = eng.wire_decode(buf, offs)
    packed = eng.wire_pack(CALL_PREPARE, kind, drows)
    assert np.array_equal(packed, rows)
    ref = EpaxosReplica(f, 1, 64, max_batch=1 << 10)
    assert np.array_equal(eng.prepare(packed), ref.prepare(rows))
    eng.close(); ref.close()


def test_commit_rows_from_bytes(G):
    f, n = 1, 3
    eng = EpaxosReplica(f, 0, 64, max_batch=1 << 10)
    m = G.RI(); c = m.commit
    c.instance.replica_index, c.instance.instance_number = 2, 9
    c.command_or_noop.noop.SetInParent(); c.sequence_number = 4
    c.dependencies.CopyFrom(G.depset([1, 0, 9]))
    buf, offs = W.pack([m.SerializeToString()])
    kind, rows, _ = eng.wire_decode(buf, offs)
    packed = eng.wire_pack(CALL_COMMIT, kind, rows)
    assert packed.tolist() == [[2, 9, W.VALUE_NOOP, 4, 1, 0, 9]]
    eng.commit(packed)
    e, _, _ = eng.entry(2, 9)
    assert e[0] == 4 and e[5] == W.VALUE_NOOP and e[6] == 4 and e[7:].tolist() == [1, 0, 9]
    eng.close()


# a mixed recovery trace (every handler call) through the codec: each inbound batch is serialised by the runtime,
# decoded and packed on the device, and applied to a handle; the same packed rows go to a second handle directly.
# Each call's outputs are encoded and compared with the runtime's serialisation of what the reference sends.
IN_CALLS = {"preaccept": CALL_PREACCEPT, "accept": CALL_ACCEPT, "preacceptok": CALL_PREACCEPTOK,
            "acceptok": CALL_ACCEPTOK, "commit": CALL_COMMIT, "nack": 6, "prepare": CALL_PREPARE, "prepareok": 9}
SENDS = {"lead": 0, "preaccept": 1, "accept": 2, "preacceptok": 3, "acceptok": 4, "prepare_phase": 7, "prepare": 8,
         "slow_path_timer": 10}


@pytest.mark.parametrize("f", [1, 2])
def test_recovery_trace_through_the_codec(G, f):
    n = 2 * f + 1
    index, per, steps = 1, 6, 200
    wire, direct = EpaxosReplica(f, index, per, 1 << 12), EpaxosReplica(f, index, per, 1 << 12)
    trace = Trace(f, index, per, 77 + f, direct, max_batch=10)
    arena, voffs = W.value_arena(1 << 16)
    seen = set()
    for step in range(steps):
        call, rows = trace.step()
        rows = np.asarray(rows, dtype=np.int32)
        if call in IN_CALLS:
            c = IN_CALLS[call]
            base = 1000 + 10 * step
            buf, offs = W.pack([W.inbound_message(G, c, r, n) for r in rows])
            kind, drows, _ = wire.wire_decode(buf, offs, base)
            packed = wire.wire_pack(c, kind, drows,
                                    local_deps=rows[:, 6:6 + n] if c == CALL_PREACCEPT else None)
            vcol = {CALL_PREACCEPT: 4, CALL_ACCEPT: 4, CALL_COMMIT: 2, 9: 8}.get(c)
            same = np.ones(packed.shape[1], dtype=bool)
            if vcol is not None:
                same[vcol] = False
                noop = rows[:, vcol] == W.VALUE_NOOP
                want = np.where(noop, W.VALUE_NOOP, base + np.arange(len(rows)))
                if c == 9:
                    want = np.where(rows[:, 7] == 0, 0, want)
                assert np.array_equal(packed[:, vcol], want), call
                # the shim's arena maps value id base + i to the bytes of message i, which carry the trace's value:
                # hand the handlers the trace's ids, so a re-delivered response repeats its content (E2)
                packed[:, vcol] = rows[:, vcol]
            assert np.array_equal(packed[:, same], rows[:, same]), call
            rows = packed
        fn = getattr(direct, call)
        out_d = fn(rows)
        out_w = getattr(wire, call)(rows)
        if out_d is not None:
            assert np.array_equal(out_w, out_d), call
        trace.observe(call, rows, out_d)
        if call in SENDS:
            seen.add(call)
            got, offs = wire.wire_encode(SENDS[call], rows, out_w, arena, voffs)
            cmd_value = lambda rep, num: int(direct.entry(rep, num)[0][5])   # noqa: E731
            assert W.split(got, offs) == W.expected_encode(G, SENDS[call], rows, out_d, n, index, cmd_value), call
        for r in rows[:8]:
            a, b = wire.entry(int(r[0]), int(r[1])), direct.entry(int(r[0]), int(r[1]))
            assert np.array_equal(a[0], b[0]) and a[1] == b[1] and np.array_equal(a[2], b[2])
    assert {"prepare", "prepare_phase", "preaccept", "accept"} <= seen
    wire.close(); direct.close()


def test_encode_refuses_calls_that_send_nothing_and_bad_values():
    eng = EpaxosReplica(1, 0, 8, max_batch=64)
    for call in (CALL_COMMIT, 6, 9):
        with pytest.raises(FpxError) as ei:
            eng.wire_encode(call, np.zeros((1, 4), np.int32))
        assert ei.value.status == W.INVALID_ARG
    lead = np.array([[0, 1, 0, 0, 5, 1, 0, 0, 0, 0, 0], [0, 2, 0, 0, 99, 1, 0, 0, 0, 0, 0]], np.int32)
    arena, voffs = W.value_arena(10)
    with pytest.raises(FpxError) as ei:
        eng.wire_encode(0, lead, None, arena, voffs)
    assert (ei.value.status, ei.value.index) == (W.INVALID_ARG, 1)
    eng.close()
