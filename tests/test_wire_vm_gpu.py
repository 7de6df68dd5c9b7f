"""GPU wire codec of vanilla Mencius (fpx_wire_*_vm_*): the golden vectors, the CPU oracle (tests/wire_vm_oracle.cc),
the device forms against the host forms, and BASELINE cfg5 end to end from protobuf bytes through fpx_vm_step_dev
back to protobuf bytes."""
import importlib.util
import json
import os

import numpy as np
import pytest

from frankenpaxos_b200 import (CHOSEN, P2A, P2B, VALUE_NOOP, VANILLA_MENCIUS, VM_SKIP, WIRE_REC, Engine, FpxError)
from frankenpaxos_b200 import traces as T
import wire_vm_oracle as V

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
CASES = json.load(open(os.path.join(HERE, "golden", "wire_vanilla_mencius.json")))["cases"]
F, N = 3, 7


def of_type(t):
    return [c for c in CASES if c["type"] == t]


@pytest.fixture(scope="module")
def eng():
    e = Engine(F, 1, N, slot_capacity=1 << 12, max_batch=1 << 12, protocol=VANILLA_MENCIUS)
    yield e
    e.close()


def same_decode(eng, msgs):
    """Engine and oracle agree: status, first offending index, and (on success) every output."""
    buf, offs = V.pack(msgs)
    st, err, okind, orec, osender = V.decode(buf, offs)
    try:
        kind, rec, sender = eng.wire_decode_vm_server_inbound(buf, offs)
        est, eidx = 0, -1
    except FpxError as e:
        est, eidx = e.status, e.index
    assert (est, eidx) == (st, err)
    if st == 0:
        assert np.array_equal(kind, okind) and np.array_equal(sender, osender)
        assert np.array_equal(rec.view(np.int32), orec.view(np.int32))
    return st


def value_arena(cs):
    vals, ids = [], []
    for c in cs:
        if c["value_hex"] == "1200":
            ids.append(VALUE_NOOP)
        else:
            ids.append(len(vals)); vals.append(bytes.fromhex(c["value_hex"]))
    arena, voffs = V.pack(vals)
    return arena, voffs, ids


def test_decode_golden(eng):
    for t in ("phase2b", "skip", "phase2_nack", "phase2a", "phase2a.coordinator", "chosen", "client_request", "phase1a",
              "phase1b", "phase1_nack"):
        assert same_decode(eng, [bytes.fromhex(c["hex"]) for c in of_type(t)]) == 0, t
    # all kinds in one batch, in the staged and the unstaged span path (a large value pushes the CTA's span past
    # the shared-memory stage)
    msgs = [bytes.fromhex(c["hex"]) for c in CASES if c["type"] != "robustness"]
    assert same_decode(eng, msgs) == 0
    big = bytes.fromhex(of_type("client_request")[-1]["hex"])
    assert same_decode(eng, msgs + [big] * 200 + msgs) == 0


def test_decode_robustness_cases(eng):
    good = bytes.fromhex(of_type("phase2b")[3]["hex"])
    for c in of_type("robustness"):
        st = same_decode(eng, [good, bytes.fromhex(c["hex"]), good])
        v = c["verdict"]
        assert (st == -15) == ("error" in v or not v["initialized"] or c["name"] == "command_or_noop twice"), c["name"]


def test_encode_golden(eng):
    cs = of_type("phase2b")
    out, offs = eng.wire_encode_vm_replies(np.array([(0, c["server_index"], c["slot"], c["round"]) for c in cs], dtype=P2B))
    assert V.split(out, offs) == [bytes.fromhex(c["hex"]) for c in cs]
    cs = of_type("phase2_nack")
    out, offs = eng.wire_encode_vm_replies(np.array([(1, 2, c["slot"], c["round"]) for c in cs], dtype=P2B))
    assert V.split(out, offs) == [bytes.fromhex(c["hex"]) for c in cs]
    cs = of_type("skip")
    out, offs = eng.wire_encode_vm_skip(np.array([(c["server_index"], c["start"], c["stop"], 0) for c in cs], dtype=VM_SKIP))
    assert V.split(out, offs) == [bytes.fromhex(c["hex"]) for c in cs]
    cs = [c for c in of_type("chosen") if not c["is_revocation"]]
    arena, voffs, ids = value_arena(cs)
    out, offs = eng.wire_encode_vm_chosen(np.array([(c["slot"], v) for c, v in zip(cs, ids)], dtype=CHOSEN), arena, voffs)
    assert V.split(out, offs) == [bytes.fromhex(c["hex"]) for c in cs]
    reps = np.array([(2, 5, c["slot"], v) for c, v in zip(cs, ids)] + [(3, 5, 9, 0)], dtype=P2B)
    out, offs = eng.wire_encode_vm_replies(reps, arena, voffs)
    assert V.split(out, offs) == [bytes.fromhex(c["hex"]) for c in cs] + [b""]      # kind 3: zero-length
    cs = of_type("phase2a.coordinator")
    arena, voffs, ids = value_arena(cs)
    out, offs = eng.wire_encode_vm_phase2a(np.array([(c["slot"], c["round"], v, 0) for c, v in zip(cs, ids)], dtype=P2A),
                                           arena, voffs)
    assert V.split(out, offs) == [bytes.fromhex(c["hex"]) for c in cs]
    with pytest.raises(FpxError) as ei:
        eng.wire_encode_vm_chosen(np.array([(1, 0), (2, len(voffs) - 1)], dtype=CHOSEN), arena, voffs)
    assert (ei.value.status, ei.value.index) == (-1, 1)
    with pytest.raises(FpxError) as ei:
        eng.wire_encode_vm_replies(np.array([(0, 1, 2, 3), (0, 1, 2, 3), (7, 1, 2, 3)], dtype=P2B))
    assert (ei.value.status, ei.value.index) == (-1, 2)


def rand_i32(g, n):
    return (g.integers(-(1 << 31), 1 << 31, size=n) >> g.integers(0, 32, size=n)).astype(np.int32)


def random_values(g, k, max_len):
    vals = [bytes(g.integers(0, 256, size=int(g.integers(0, max_len)), dtype=np.uint8)) for _ in range(k)]
    return V.pack(vals)


@pytest.mark.parametrize("n", [1, 1023, 1025, 70001])
def test_encoders_agree_with_the_oracle(eng, n):
    g = np.random.Generator(np.random.PCG64(n))
    arena, voffs = random_values(g, 300, 400)
    vid = np.where(g.integers(0, 5, size=n) == 0, VALUE_NOOP, g.integers(0, 300, size=n)).astype(np.int32)
    reps = np.zeros(n, dtype=P2B)
    reps["group"] = g.integers(0, 4, size=n); reps["acceptor"] = rand_i32(g, n); reps["slot"] = rand_i32(g, n)
    reps["round"] = np.where(reps["group"] == 2, vid, rand_i32(g, n))
    ch = np.zeros(n, dtype=CHOSEN); ch["slot"] = rand_i32(g, n); ch["value_id"] = vid
    p2a = np.zeros(n, dtype=P2A); p2a["slot"] = rand_i32(g, n); p2a["round"] = rand_i32(g, n); p2a["value_id"] = vid
    sk = np.zeros(n, dtype=VM_SKIP)
    for f in ("server", "slot_start", "slot_stop"):
        sk[f] = rand_i32(g, n)
    for what, fn, recs, extra in (("replies", eng.wire_encode_vm_replies, reps, (arena, voffs)),
                                  ("chosen", eng.wire_encode_vm_chosen, ch, (arena, voffs)),
                                  ("phase2a", eng.wire_encode_vm_phase2a, p2a, (arena, voffs)),
                                  ("skip", eng.wire_encode_vm_skip, sk, ())):
        out, offs = fn(recs, *extra)
        st, _, oout, ooffs = V.encode(what, recs, *extra, servers=N)
        assert st == 0 and np.array_equal(offs, ooffs) and np.array_equal(out, oout), what
    # round trip through the decoder
    out, offs = eng.wire_encode_vm_skip(sk)
    kind, rec, sender = eng.wire_decode_vm_server_inbound(out, offs)
    assert (kind == 6).all() and np.array_equal(sender, sk["server"])
    assert np.array_equal(rec.view(np.int32).reshape(-1, 4)[:, :3], sk.view(np.int32).reshape(-1, 4)[:, :3])


def test_malformed_random_mutations_agree_with_oracle(eng):
    """Truncate, flip and extend bytes of valid messages of every kind: engine and oracle agree on the status and
    the first offending index."""
    g = np.random.Generator(np.random.PCG64(78))
    msgs = [bytes.fromhex(c["hex"]) for c in CASES if c["type"] != "robustness"]
    bad = 0
    for trial in range(80):
        ms = [msgs[int(k)] for k in g.integers(0, len(msgs), size=300)]
        for _ in range(int(g.integers(1, 4))):
            k = int(g.integers(0, len(ms)))
            m = bytearray(ms[k])
            op = g.integers(0, 3)
            if op == 0 and len(m) > 1: m = m[: int(g.integers(1, len(m)))]
            elif op == 1: m[int(g.integers(0, len(m)))] ^= 1 << int(g.integers(0, 8))
            else: m += bytes(g.integers(0, 256, size=int(g.integers(1, 4)), dtype=np.uint8))
            ms[k] = bytes(m)
        bad += same_decode(eng, ms) != 0
    assert bad > 20


def test_other_protocols_are_unsupported():
    e = Engine(1, 1, 3, slot_capacity=64, max_batch=64)
    with pytest.raises(FpxError) as ei:
        e.wire_decode_vm_server_inbound(np.zeros(2, dtype=np.uint8), np.array([0, 2], dtype=np.int32))
    assert ei.value.status == -11
    for fn in (e.wire_encode_vm_replies, e.wire_encode_vm_skip):
        with pytest.raises(FpxError) as ei:
            fn(np.zeros(1, dtype=P2B if fn == e.wire_encode_vm_replies else VM_SKIP))
        assert ei.value.status == -11
    e.close()


# --------------------------------------------------------------------------- device forms
def _torch():
    import torch
    return torch, torch.device("cuda", 0)


def to_dev(x):
    torch, dev = _torch()
    return torch.from_numpy(np.ascontiguousarray(x).view(np.uint8).reshape(-1).copy()).to(dev)


def from_dev(t, dtype, n):
    return t.cpu().numpy().view(dtype)[:n]


def test_device_forms_equal_host_forms(eng):
    torch, dev = _torch()
    g = np.random.Generator(np.random.PCG64(31))
    msgs = [bytes.fromhex(c["hex"]) for c in CASES if c["type"] != "robustness"] * 30
    msgs = [msgs[int(k)] for k in g.permutation(len(msgs))]
    buf, offs = V.pack(msgs)
    kind, rec, sender = eng.wire_decode_vm_server_inbound(buf, offs)
    n = len(msgs)
    d_kind = torch.zeros(n, dtype=torch.int32, device=dev); d_rec = torch.zeros((n, 4), dtype=torch.int32, device=dev)
    d_sender = torch.zeros(n, dtype=torch.int32, device=dev)
    d_buf, d_offs = to_dev(buf), to_dev(offs)
    eng.wire_decode_vm_server_inbound_dev(d_buf.data_ptr(), d_offs.data_ptr(), n, d_kind.data_ptr(), d_rec.data_ptr(),
                                          d_sender.data_ptr())
    eng.sync()
    assert np.array_equal(d_kind.cpu().numpy(), kind) and np.array_equal(d_sender.cpu().numpy(), sender)
    assert np.array_equal(d_rec.cpu().numpy().reshape(-1), rec.view(np.int32).reshape(-1))
    # the encoders
    m = 5000
    arena, voffs = random_values(g, 200, 300)
    vid = np.where(g.integers(0, 5, size=m) == 0, VALUE_NOOP, g.integers(0, 200, size=m)).astype(np.int32)
    reps = np.zeros(m, dtype=P2B); reps["group"] = g.integers(0, 4, size=m); reps["acceptor"] = g.integers(0, N, size=m)
    reps["slot"] = rand_i32(g, m); reps["round"] = np.where(reps["group"] == 2, vid, rand_i32(g, m))
    ch = np.zeros(m, dtype=CHOSEN); ch["slot"] = rand_i32(g, m); ch["value_id"] = vid
    p2a = np.zeros(m, dtype=P2A); p2a["slot"] = rand_i32(g, m); p2a["round"] = rand_i32(g, m); p2a["value_id"] = vid
    sk = np.zeros(m, dtype=VM_SKIP)
    for f in ("server", "slot_start", "slot_stop"):
        sk[f] = rand_i32(g, m)
    d_arena, d_voffs = to_dev(arena), to_dev(voffs)
    nv = len(voffs) - 1
    for host, devf, recs, valued in ((eng.wire_encode_vm_replies, eng.wire_encode_vm_replies_dev, reps, True),
                                     (eng.wire_encode_vm_chosen, eng.wire_encode_vm_chosen_dev, ch, True),
                                     (eng.wire_encode_vm_phase2a, eng.wire_encode_vm_phase2a_dev, p2a, True),
                                     (eng.wire_encode_vm_skip, eng.wire_encode_vm_skip_dev, sk, False)):
        out, hoffs = host(recs, arena, voffs) if valued else host(recs)
        cap = len(out) + 64
        d_out = torch.zeros(cap, dtype=torch.uint8, device=dev)
        d_o = torch.zeros(m + 1, dtype=torch.int32, device=dev)
        d_in = to_dev(recs)
        if valued:
            devf(d_in.data_ptr(), m, d_arena.data_ptr(), d_voffs.data_ptr(), nv, d_out.data_ptr(), cap, d_o.data_ptr())
        else:
            devf(d_in.data_ptr(), m, d_out.data_ptr(), cap, d_o.data_ptr())
        eng.sync()
        assert np.array_equal(d_o.cpu().numpy(), hoffs)
        assert np.array_equal(d_out.cpu().numpy()[: len(out)], out)
    # the device form reports a bad value id at fpx_sync, with its index
    bad = ch.copy(); bad["value_id"][777] = nv
    d_in = to_dev(bad)
    cap = len(eng.wire_encode_vm_chosen(ch, arena, voffs)[0]) + 64
    d_out = torch.zeros(cap, dtype=torch.uint8, device=dev)
    eng.wire_encode_vm_chosen_dev(d_in.data_ptr(), m, d_arena.data_ptr(), d_voffs.data_ptr(), nv, d_out.data_ptr(),
                                  cap, d_o.data_ptr())
    r = eng.sync(check=False)
    assert (r.status, r.err_index) == (-1, 777)


# --------------------------------------------------------------------------- BASELINE cfg5 end to end
def golden_module():
    pytest.importorskip("google.protobuf")
    spec = importlib.util.spec_from_file_location("make_wire_vm_golden", os.path.join(HERE, "golden", "make_wire_vm_golden.py"))
    G = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(G)
    return G


def gather(buf, start, length):
    """Rows buf[start[i] : start[i] + length] (one length for all rows)."""
    return np.lib.stride_tricks.sliding_window_view(buf, length)[start]


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_cfg5_end_to_end_from_and_to_protobuf_bytes(seed):
    """traces.vanilla_cfg5 (f = 3, 7 servers, 2^20 slots) as ServerInbound bytes serialised by the protobuf runtime:
    ClientRequests, the coordinators' Phase2as and the Phase2bs, in one batch.  Decoded on the device, the records
    are the ones the vm tests feed directly; fpx_vm_step_dev on them gives the outputs and final state the direct
    records give; the replies, the Chosen broadcast and the Phase2a broadcast encoded on the device are byte for
    byte what the reference's handlers send (SerializeToString of Phase2b(serverIndex = index, slot, round)
    :1077-1081, Chosen(slot, phase2.value, false) :1127-1135, Phase2a(index, nextSlot, 0, value) :806-815)."""
    torch, dev = _torch()
    G = golden_module()
    SI, CR, P2a, P2b, Ch = (G.vcls(k) for k in ("ServerInbound", "ClientRequest", "Phase2a", "Phase2b", "Chosen"))
    Cmd, CId, CoN = G.vcls("Command"), G.vcls("CommandId"), G.vcls("CommandOrNoop")
    S = 1 << 20
    req, p, b = T.vanilla_cfg5(seed, F, S)
    assert np.array_equal(req["slot"], np.arange(S))
    # one command per slot, all of one length (client_id always a 5-byte varint) so spans compare as rows
    cmds = [Cmd(command_id=CId(client_address=b"node-7", client_pseudonym=seed, client_id=(1 << 28) | s),
                command=s.to_bytes(4, "little") * 2) for s in range(S)]
    values = [CoN(command=c).SerializeToString() for c in cmds]
    L = len(values[0])
    assert all(len(v) == L for v in values[:: 4099])
    vals = np.frombuffer(b"".join(values), dtype=np.uint8).reshape(S, L)
    req_bytes = [SI(client_request=CR(command=c)).SerializeToString() for c in cmds]
    p2a_by_slot = [SI(phase2a=P2a(sending_server=s % N, slot=s, round=0, command_or_noop=CoN(command=cmds[s]))).SerializeToString()
                   for s in range(S)]
    # the servers' Phase2b replies, in the order of the Phase2as they answer; the Phase2b batch is their permutation
    replies = [SI(phase2b=P2b(server_index=int(d), slot=int(s), round=0)).SerializeToString()
               for d, s in zip(p["dst"].tolist(), p["slot"].tolist())]
    key_p = p["slot"].astype(np.int64) * N + p["dst"]
    key_b = b["slot"].astype(np.int64) * N + b["acceptor"]
    pos_p = np.argsort(key_p)
    b_from_p = pos_p[np.searchsorted(key_p[pos_p], key_b)]
    assert np.array_equal(key_p[b_from_p], key_b)
    msgs = req_bytes + [p2a_by_slot[s] for s in p["slot"].tolist()] + [replies[i] for i in b_from_p.tolist()]
    n_req, n_p, n_b = len(req), len(p), len(b)
    n = len(msgs)
    buf, offs = V.pack(msgs)
    del msgs

    # decode on the device
    d_buf, d_offs = to_dev(buf), to_dev(offs)
    d_kind = torch.zeros(n, dtype=torch.int32, device=dev)
    d_rec = torch.zeros((n, 4), dtype=torch.int32, device=dev)
    d_sender = torch.zeros(n, dtype=torch.int32, device=dev)
    cfg, _ = T.config_by_name("cfg5")
    A = Engine(slot_capacity=S, max_batch=(N - 1) * S, protocol=VANILLA_MENCIUS, **cfg)
    B = Engine(slot_capacity=S, max_batch=(N - 1) * S, protocol=VANILLA_MENCIUS, **cfg)
    A.wire_decode_vm_server_inbound_dev(d_buf.data_ptr(), d_offs.data_ptr(), n, d_kind.data_ptr(), d_rec.data_ptr(),
                                        d_sender.data_ptr())
    A.sync()
    kind, rec, sender = d_kind.cpu().numpy(), d_rec.cpu().numpy().view(WIRE_REC).reshape(-1), d_sender.cpu().numpy()
    r_req, r_p, r_b = rec[:n_req], rec[n_req: n_req + n_p], rec[n_req + n_p:]
    assert (kind[:n_req] == 1).all() and (kind[n_req: n_req + n_p] == 4).all() and (kind[n_req + n_p:] == 5).all()
    assert (sender[:n_req] == -1).all()
    assert np.array_equal(sender[n_req: n_req + n_p], p["slot"] % N)          # the coordinator owns the slot
    assert np.array_equal(sender[n_req + n_p:], b["acceptor"])
    # the records the vm tests feed, except value_id = the index of the message whose span holds the value
    assert np.array_equal(r_p["a"], p["slot"]) and np.array_equal(r_p["b"], p["round"])
    assert np.array_equal(r_b.view(np.int32).reshape(-1, 4), b.view(np.int32).reshape(-1, 4))
    assert (r_req["d"] == L).all() and (r_p["d"] == L).all()
    assert np.array_equal(gather(buf, r_req["c"], L), vals)                      # the ClientRequest span = CommandOrNoop
    assert np.array_equal(gather(buf, r_p["c"], L), vals[p["slot"]])
    a_req = req.copy(); a_req["value_id"] = np.arange(n_req)
    a_p = p.copy(); a_p["value_id"] = n_req + np.arange(n_p)
    a_b = r_b.view(P2B)
    # the arena: message k's value span (empty for a Phase2b), so value_id k is message k's value
    has = np.zeros(n, dtype=bool); has[: n_req + n_p] = True
    lens = np.where(has, rec["d"], 0).astype(np.int64)
    voffs = np.zeros(n + 1, dtype=np.int32); voffs[1:] = np.cumsum(lens)
    arena = gather(buf, rec["c"][has], L).reshape(-1)
    assert len(arena) == voffs[-1]
    # to the trace's value ids: what engine B holds where engine A holds message k's value
    to_trace = np.full(n, -1, dtype=np.int64); to_trace[:n_req] = req["value_id"]; to_trace[n_req: n_req + n_p] = p["value_id"]

    # one step of the co-located servers on both engines
    def step(E, rq, pp, bb):
        d_rq, d_pp, d_bb = to_dev(rq), to_dev(pp), to_dev(bb)
        d_rep = torch.zeros((n_p, 4), dtype=torch.int32, device=dev)
        d_ch = torch.zeros((n_b, 2), dtype=torch.int32, device=dev)
        d_wm = torch.zeros(1, dtype=torch.int32, device=dev)
        E.vm_step_dev(d_rq.data_ptr(), len(rq), d_pp.data_ptr(), len(pp), d_rep.data_ptr(), d_bb.data_ptr(), len(bb),
                      d_ch.data_ptr(), d_wm.data_ptr())
        r = E.sync()
        return r, d_rep, d_ch[: r.n_chosen]
    ra, d_rep, d_ch = step(A, a_req, a_p, a_b)
    rb, d_rep_b, d_ch_b = step(B, req, p, b)
    assert (ra.status, ra.n_chosen, ra.watermark) == (rb.status, rb.n_chosen, rb.watermark) == (0, S, S)
    rep_a = d_rep.cpu().numpy().view(P2B).reshape(-1)
    assert np.array_equal(rep_a, d_rep_b.cpu().numpy().view(P2B).reshape(-1)) and (rep_a["group"] == 0).all()
    ch_a, ch_b = d_ch.cpu().numpy().view(CHOSEN).reshape(-1), d_ch_b.cpu().numpy().view(CHOSEN).reshape(-1)
    assert np.array_equal(ch_a["slot"], ch_b["slot"]) and np.array_equal(to_trace[ch_a["value_id"]], ch_b["value_id"])
    la, lb = A.snapshot_log(0, S), B.snapshot_log(0, S)
    assert np.array_equal(np.where(la >= 0, to_trace[np.maximum(la, 0)], la), lb)
    for s in range(N):
        xa, xb = A.snapshot_acceptor(0, s, 0, S), B.snapshot_acceptor(0, s, 0, S)
        assert xa[:2] == xb[:2] and np.array_equal(xa[2], xb[2])
        assert np.array_equal(np.where(xa[2] >= 0, to_trace[np.maximum(xa[3], 0)], xb[3]), xb[3])

    # encode on the device: the replies, the Chosen broadcast, the coordinators' Phase2a broadcast
    d_arena, d_voffs = to_dev(arena), to_dev(voffs)

    def encode(fn, d_in, m, cap):
        d_out = torch.zeros(cap, dtype=torch.uint8, device=dev)
        d_o = torch.zeros(m + 1, dtype=torch.int32, device=dev)
        fn(d_in.data_ptr(), m, d_arena.data_ptr(), d_voffs.data_ptr(), n, d_out.data_ptr(), cap, d_o.data_ptr())
        A.sync()
        o = d_o.cpu().numpy()
        return d_out[: o[-1]].cpu().numpy().tobytes(), o

    def check(got, want):
        out, o = got
        assert np.array_equal(np.diff(o), [len(w) for w in want])
        assert out == b"".join(want)
    check(encode(A.wire_encode_vm_replies_dev, d_rep, n_p, 16 * n_p), replies)
    check(encode(A.wire_encode_vm_chosen_dev, d_ch, S, (L + 32) * S),
          [SI(chosen=Ch(slot=int(s), command_or_noop=CoN(command=cmds[s]), isRevocation=False)).SerializeToString()
           for s in ch_a["slot"].tolist()])
    check(encode(A.wire_encode_vm_phase2a_dev, to_dev(a_req), n_req, (L + 32) * S), p2a_by_slot)
    A.close(); B.close()
