"""GPU parity of the MultiPaxos replica / read-path wire codec (fpx_wire_decode_replica_inbound,
fpx_wire_encode_max_slot_replies, fpx_reads_wire_*) against the golden vectors, the CPU oracle
(tests/wire_reads_oracle.cc), the Python protobuf runtime and the Scala transcription of the read path."""
import importlib.util
import json
import os
import zlib

import numpy as np
import pytest

import reads_oracle as RO
import reads_traces as RT
import wire_reads_oracle as O
from frankenpaxos_b200 import (MENCIUS, VANILLA_MENCIUS, WIRE_ACCEPTOR_INBOUND, Engine, FpxError, Reads, READS_CLIENT,
                               READS_READ_BATCHER)
from frankenpaxos_b200 import traces as T
from scala_transcription_reads import ReadQuorumTally, ReplicaReads

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = json.load(open(os.path.join(HERE, "golden", "wire_multipaxos_reads.json")))
CASES, KEY_CAP = GOLD["cases"], GOLD["key_capacity"]


def golden_module():
    pytest.importorskip("google.protobuf")
    spec = importlib.util.spec_from_file_location("make_wire_reads_golden",
                                                  os.path.join(HERE, "golden", "make_wire_reads_golden.py"))
    G = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(G)
    return G


@pytest.fixture(scope="module")
def eng():
    e = Engine(1, 2, 3, slot_capacity=1 << 10, max_batch=1 << 10)
    yield e
    e.close()


def status_of(fn, *a, **kw):
    try:
        return 0, -1, fn(*a, **kw)
    except FpxError as e:
        return e.status, e.index, None


def same_replica(eng, msgs, value_id_base=0, handle_base=0, cap=None):
    buf, offs = O.pack(msgs)
    o = O.decode_replica(buf, offs, value_id_base, handle_base, cap)
    st, idx, got = status_of(eng.wire_decode_replica_inbound, buf, offs, value_id_base, handle_base, cap)
    assert (st, idx) == (o[0], o[1])
    if st == 0:
        kind, chosen, cvals, reads, rcmds, split = got
        assert split == o[7]
        for x, y in zip((kind, chosen, cvals, reads, rcmds), o[2:7]):
            assert np.array_equal(np.asarray(x).view(np.int32), np.asarray(y).view(np.int32))
    return o


def same_reads(r, batcher, msgs):
    buf, offs = O.pack(msgs)
    o = O.decode_reads(buf, offs, batcher, r.key_capacity)
    st, idx, got = status_of(r.wire_decode, buf, offs)
    assert (st, idx) == (o[0], o[1])
    if st == 0:
        for x, y in zip(got, o[2:]):
            assert np.array_equal(np.asarray(x).view(np.int32), np.asarray(y).view(np.int32))
    return o


def test_golden_decodes_and_encodes(eng):
    rep = [c for c in CASES if c["inbound"] == "replica"]
    for c in rep:                                                   # one at a time: statuses and records
        o = same_replica(eng, [bytes.fromhex(c["hex"])])
        assert o[0] == c["expect"]["status"], c["name"]
    good = [bytes.fromhex(c["hex"]) for c in rep if c["expect"]["status"] == 0]
    same_replica(eng, good, value_id_base=100, handle_base=7)      # and as one batch
    for kind, inbound in ((READS_CLIENT, "client"), (READS_READ_BATCHER, "batcher")):
        with Reads(eng, kind, key_capacity=KEY_CAP) as r:
            for c in (c for c in CASES if c["inbound"] == inbound):
                o = same_reads(r, kind == READS_READ_BATCHER, [bytes.fromhex(c["hex"])])
                assert o[0] == c["expect"]["status"], c["name"]
                if o[0] == 0:
                    e = c["expect"]
                    assert tuple(int(x) for x in o[3][0].tolist()) == (e["key"], e["id"], e["voter"], e["slot"])
    for c in (c for c in CASES if c["inbound"] == "acceptor"):
        raw = bytes.fromhex(c["hex"])
        buf, offs = O.pack([raw])
        kind, rec = eng.wire_decode_inbound(WIRE_ACCEPTOR_INBOUND, buf, offs)
        rec["a"], rec["b"] = (c["group"] << 16) | c["acceptor"], c["max_voted_slot"]
        st, idx, got = status_of(eng.wire_encode_max_slot_replies, buf[:len(raw)], kind, rec)
        assert st == c["expect"]["status"], c["name"]
        if st == 0:
            assert bytes(got[0]).hex() == c["expect"]["reply_hex"], c["name"]
    for batcher in (0, 1):
        cs = [c for c in CASES if c["inbound"] == "read_request" and c["batcher"] == batcher]
        arena = b"".join(bytes.fromhex(c["arena_hex"]) for c in cs)
        voffs = np.concatenate([[0], np.cumsum([len(bytes.fromhex(c["arena_hex"])) for c in cs])]).astype(np.int32)
        recs = np.zeros(len(cs), O.READ_SLOT)
        recs["key"] = np.arange(len(cs)); recs["slot"] = [c["slot"] for c in cs]
        with Reads(eng, READS_READ_BATCHER if batcher else READS_CLIENT, key_capacity=KEY_CAP) as r:
            out, offs = r.wire_encode_read_requests(recs, np.frombuffer(arena, np.uint8), voffs)
        assert O.split(out, offs) == [bytes.fromhex(c["hex"]) for c in cs]


def mutate(g, raw):
    b = bytearray(raw)
    for _ in range(int(g.integers(1, 4))):
        i = int(g.integers(0, len(b) + 1))
        if g.integers(0, 2) and i < len(b):
            b[i] = int(g.integers(0, 256))
        else:
            b.insert(i, int(g.integers(0, 256)))
    return bytes(b)


def test_random_and_mutated_batches_against_oracle(eng):
    G = golden_module()
    g = np.random.Generator(np.random.PCG64(11))
    for trial in range(40):
        msgs = [G.replica_message(g, int(g.integers(1, 8))).SerializeToString() for _ in range(int(g.integers(1, 700)))]
        if trial % 2:
            msgs = [mutate(g, m) if g.random() < 0.02 else m for m in msgs]
        same_replica(eng, msgs, int(g.integers(-5, 5)), int(g.integers(0, 1 << 30)))
    for kind in (READS_CLIENT, READS_READ_BATCHER):
        make = G.batcher_message if kind else G.client_message
        with Reads(eng, kind, key_capacity=KEY_CAP) as r:
            for trial in range(20):
                msgs = [make(g, int(g.integers(1, 5 if kind else 6))).SerializeToString() for _ in range(600)]
                if trial % 2:
                    msgs = [mutate(g, m) if g.random() < 0.02 else m for m in msgs]
                same_reads(r, kind == READS_READ_BATCHER, msgs)


def test_device_forms_match_host_forms(eng):
    import torch
    G = golden_module()
    g = np.random.Generator(np.random.PCG64(12))
    dev = torch.device("cuda", 0)
    msgs = [G.replica_message(g, int(g.integers(1, 8)), 3).SerializeToString() for _ in range(3000)]
    buf, offs = O.pack(msgs)
    host = eng.wire_decode_replica_inbound(buf, offs, 3, 9)
    n, cap = len(msgs), int(offs[-1])
    d_buf, d_offs = torch.from_numpy(buf).to(dev), torch.from_numpy(offs).to(dev)
    t = lambda *s: torch.zeros(s, dtype=torch.int32, device=dev)
    kind, ch, cv, rd, rc, cnt = t(n), t(n, 2), t(n, 2), t(cap, 2), t(cap, 2), t(3)
    torch.cuda.synchronize()
    eng.wire_decode_replica_inbound_dev(d_buf.data_ptr(), d_offs.data_ptr(), n, 3, 9, cap, kind.data_ptr(),
                                        ch.data_ptr(), cv.data_ptr(), rd.data_ptr(), rc.data_ptr(), cnt.data_ptr())
    eng.sync()
    nc, nr, split = cnt.cpu().tolist()
    assert split == host[5] and nc == len(host[1]) and nr == len(host[3])
    assert np.array_equal(kind.cpu().numpy(), host[0])
    for d, h, k in ((ch, host[1], nc), (cv, host[2], nc), (rd, host[3], nr), (rc, host[4], nr)):
        assert np.array_equal(d[:k].cpu().numpy().reshape(-1), np.asarray(h).view(np.int32).reshape(-1))
    with Reads(eng, READS_CLIENT, key_capacity=KEY_CAP) as r:
        cm = [G.client_message(g, int(g.integers(1, 6))).SerializeToString() for _ in range(2000)]
        cbuf, coffs = O.pack(cm)
        hk, ho, hs = r.wire_decode(cbuf, coffs)
        k2, o2, s2 = t(len(cm)), t(len(cm), 4), t(len(cm), 2)
        d_cbuf, d_coffs = torch.from_numpy(cbuf).to(dev), torch.from_numpy(coffs).to(dev)
        torch.cuda.synchronize()
        r.wire_decode_dev(d_cbuf.data_ptr(), d_coffs.data_ptr(), len(cm), k2.data_ptr(), o2.data_ptr(), s2.data_ptr())
        r.sync()
        assert np.array_equal(k2.cpu().numpy(), hk) and np.array_equal(o2.cpu().numpy().reshape(-1), ho.view(np.int32))
        assert np.array_equal(s2.cpu().numpy(), hs)
        # the read-request encoder on device pointers
        arena_parts = [G.arena_entry([G.command(g)]) for _ in range(500)]
        arena = np.frombuffer(b"".join(arena_parts), np.uint8).copy()
        voffs = np.concatenate([[0], np.cumsum([len(a) for a in arena_parts])]).astype(np.int32)
        recs = np.zeros(500, O.READ_SLOT)
        recs["key"] = g.permutation(500); recs["slot"] = g.integers(-1, 1 << 20, 500)
        hb, hoffs = r.wire_encode_read_requests(recs, arena, voffs)
        out = torch.zeros(len(hb) + 64, dtype=torch.uint8, device=dev)
        doffs = t(501)
        d_recs, d_arena = torch.from_numpy(recs.view(np.int32).reshape(-1, 4)).to(dev), torch.from_numpy(arena).to(dev)
        d_voffs = torch.from_numpy(voffs).to(dev)
        torch.cuda.synchronize()
        r.wire_encode_read_requests_dev(d_recs.data_ptr(), 500, d_arena.data_ptr(), d_voffs.data_ptr(), 500,
                                        out.data_ptr(), len(out), doffs.data_ptr())
        r.sync()
        assert np.array_equal(doffs.cpu().numpy(), hoffs) and bytes(out[:len(hb)].cpu().numpy()) == bytes(hb)


def test_non_monotone_offsets_with_split_inside_a_tile(eng):
    """Offsets that run backwards for one message, with overlapping messages around it and split inside the tile,
    staged in shared memory or read from global memory: FPX_ERR_WIRE at that message, as the oracle says."""
    for big in (False, True):
        buf, offs = O.overlapping_batch(big)
        o = O.decode_replica(buf, offs)
        assert (o[0], o[1]) == (-15, 1)
        for cap in (None, 1, 4):
            st, idx, _ = status_of(eng.wire_decode_replica_inbound, buf, offs, 0, 0, cap)
            assert (st, idx) == (-15, 1)


def test_reads_capacity_overflow(eng):
    G = golden_module()
    g = np.random.Generator(np.random.PCG64(13))
    msgs = [G.replica_message(g, 5, 64).SerializeToString() for _ in range(40)]
    for cap in (0, 63, 64, 1000, 2559):
        o = same_replica(eng, msgs, cap=cap)
        assert (o[0], o[1]) == (-8, cap // 64)
    assert same_replica(eng, msgs, cap=2560)[0] == 0


def test_unsupported_on_mencius_protocols():
    buf, offs = O.pack([b""])
    for proto, kw in ((MENCIUS, dict(num_leader_groups=1)), (VANILLA_MENCIUS, {})):
        with Engine(1, 1, 3, protocol=proto, slot_capacity=64, max_batch=64, **kw) as e:
            with pytest.raises(FpxError) as ei:
                e.wire_decode_replica_inbound(buf, offs)
            assert ei.value.status == -11
            with pytest.raises(FpxError) as ei:
                e.wire_encode_max_slot_replies(buf, np.zeros(1, np.int32), np.zeros(1, O.WIRE_REC))
            assert ei.value.status == -11


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_cfg2_chosen_stream_round_trip(seed):
    """fpx_step_dev's Chosen stream -> fpx_wire_encode_chosen -> the replica decode -> fpx_replica_chosen_dev on a
    second engine: the same watermark and log (value ids mapped back through the messages)."""
    import torch
    cfg, n_slots = T.config_by_name("cfg2")
    dev = torch.device("cuda", 0)
    a, p, b = T.workload(seed, cfg, n_slots)
    td = lambda x: torch.from_numpy(np.ascontiguousarray(x).view(np.int32).reshape(len(x), -1).copy()).to(dev)
    with Engine(slot_capacity=n_slots, max_batch=len(b), **cfg) as e1, \
            Engine(slot_capacity=n_slots, max_batch=n_slots, **cfg) as e2:
        da, dp, db = td(a), td(p), td(b)
        o1 = torch.zeros((len(dp), 4), dtype=torch.int32, device=dev)
        o2 = torch.zeros((len(dp), 2), dtype=torch.int32, device=dev)
        o3 = torch.zeros((len(db), 2), dtype=torch.int32, device=dev)
        wm = torch.zeros(1, dtype=torch.int32, device=dev)
        torch.cuda.synchronize()
        e1.step_dev(da.data_ptr(), len(da), dp.data_ptr(), len(dp), o1.data_ptr(), o2.data_ptr(), db.data_ptr(),
                    len(db), o3.data_ptr(), wm.data_ptr())
        s = e1.sync()
        chosen = o3[:s.n_chosen].cpu().numpy().reshape(-1).view(O.CHOSEN)
        assert len(chosen) == n_slots
        vmax = int(chosen["value_id"].max()) + 1
        lens = np.random.default_rng(seed).integers(2, 9, vmax)
        voffs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
        arena = np.random.default_rng(seed + 1).integers(0, 256, int(voffs[-1])).astype(np.uint8)
        wbuf, woffs = e1.wire_encode_chosen(chosen, arena, voffs)
        wbuf = np.concatenate([wbuf, np.zeros(16, np.uint8)])
        n = len(chosen)
        t = lambda *sh: torch.zeros(sh, dtype=torch.int32, device=dev)
        kind, ch, cv, cnt = t(n), t(n, 2), t(n, 2), t(3)
        d_wbuf, d_woffs = torch.from_numpy(wbuf).to(dev), torch.from_numpy(woffs).to(dev)
        torch.cuda.synchronize()
        e2.wire_decode_replica_inbound_dev(d_wbuf.data_ptr(), d_woffs.data_ptr(), n, 0, 0, 0, kind.data_ptr(),
                                           ch.data_ptr(), cv.data_ptr(), 0, 0, cnt.data_ptr())
        e2.replica_chosen_dev(ch.data_ptr(), n)
        s2 = e2.sync()
        assert cnt.cpu().tolist() == [n, 0, n]
        assert e2.chosen_watermark() == e1.chosen_watermark() == n_slots
        got = ch.cpu().numpy().reshape(-1).view(O.CHOSEN)
        assert np.array_equal(got["slot"], chosen["slot"]) and np.array_equal(got["value_id"], np.arange(n))
        spans = cv.cpu().numpy()
        vid = chosen["value_id"]
        for i in np.random.default_rng(seed).integers(0, n, 2000):   # the located value is the arena entry
            assert bytes(wbuf[spans[i, 0]: spans[i, 0] + spans[i, 1]]) == bytes(arena[voffs[vid[i]]: voffs[vid[i] + 1]])
        log1, log2 = e1.snapshot_log(0, n_slots), e2.snapshot_log(0, n_slots)
        order = np.argsort(chosen["slot"])
        assert np.array_equal(log1, vid[order]) and np.array_equal(vid[log2], log1)


SHAPES = {"1x5": dict(f=2, num_acceptor_groups=1, acceptors_per_group=5, flexible=False, num_leaders=3, num_replicas=3),
          "2x3": RT.SHAPES["groups2x3"], "grid2x3": RT.SHAPES["grid2x3"]}


@pytest.mark.parametrize("shape", sorted(SHAPES))
@pytest.mark.parametrize("kind", [READS_CLIENT, READS_READ_BATCHER])
def test_read_round_trip_bytes_to_bytes(shape, kind):
    """MaxSlotRequests (runtime bytes) -> AcceptorInbound decode -> MaxSlotReply encode (= what Acceptor.scala sends)
    -> shuffled -> Reads.wire_decode -> tally -> ReadRequest encode (= what Client / ReadBatcher send) -> replica
    decode -> fpx_reads_replica / advance, against the Scala transcription on the same trace."""
    G = golden_module()
    cfg = SHAPES[shape]
    g = np.random.default_rng(zlib.crc32(shape.encode()) + kind)
    groups, per = cfg["num_acceptor_groups"], cfg["acceptors_per_group"]
    batcher = kind == READS_READ_BATCHER
    n_reads, key_cap = 300, 512
    with Engine(slot_capacity=1 << 12, max_batch=1 << 14, **cfg) as eng, \
            Reads(eng, kind, key_capacity=key_cap, pending_capacity=1 << 14, max_batch=1 << 14) as r:
        tally = ReadQuorumTally(kind, cfg["f"], groups, per, cfg["flexible"])
        keys = g.choice(key_cap, n_reads, replace=False).astype(np.int32)
        ids = g.integers(-5, 1 << 20, n_reads).astype(np.int32)
        if batcher:
            keys = (ids % key_cap).astype(np.int32)
            ids = ids[np.unique(keys, return_index=True)[1]]; keys = (ids % key_cap).astype(np.int32)
        r.open(keys, ids)
        for k, i in zip(keys, ids):
            tally.read(int(k), int(i))
        cmds = {int(k): G.command(g, pseudo=int(k) if not batcher else None, cid=int(i)) for k, i in zip(keys, ids)}
        # every acceptor answers every read: the requests in AcceptorInbound bytes
        reqs, who = [], []
        for k, i in zip(keys, ids):
            for grp in range(groups):
                for acc in range(per):
                    m = G.cls("AcceptorInbound")()
                    if batcher:
                        m.batch_max_slot_request.read_batcher_index = 3; m.batch_max_slot_request.read_batcher_id = int(i)
                    else:
                        m.max_slot_request.command_id.CopyFrom(cmds[int(k)].command_id)
                    reqs.append(m.SerializeToString()); who.append((grp, acc))
        buf, offs = O.pack(reqs)
        akind, arec = eng.wire_decode_inbound(WIRE_ACCEPTOR_INBOUND, buf, offs)
        mvs = g.integers(-1, 1 << 12, len(reqs)).astype(np.int32)
        arec["a"] = [(gr << 16) | ac for gr, ac in who]; arec["b"] = mvs
        rbuf, roffs = eng.wire_encode_max_slot_replies(buf[:offs[-1]], akind, arec)
        replies = O.split(rbuf, roffs)
        want = [G.max_slot_reply_bytes(m, gr, ac, int(s)) for m, (gr, ac), s in zip(reqs, who, mvs)]
        assert replies == want
        perm = g.permutation(len(replies))
        replies = [replies[j] for j in perm]
        pbuf, poffs = O.pack(replies)
        dk, dout, _ = r.wire_decode(pbuf, poffs)
        assert (dk == 4).all()
        done = r.max_slot_replies(dout)
        expect = []
        for rec in dout:
            v = int(rec["voter"])
            s = tally.handle_max_slot_reply(int(rec["key"]), int(rec["id"]), v >> 16, v & 0xffff, int(rec["slot"]))
            if s is not None:
                expect.append((int(rec["key"]), int(rec["id"]), s, 0))
        RT.same_outputs([done], [np.array(expect, RO.READ_SLOT)], "tally")
        assert len(done) == len(keys)
        # the completed reads as the ReadRequest / ReadRequestBatch bytes
        order = {int(k): j for j, k in enumerate(keys)}
        batches = {int(k): [cmds[int(k)]] * (1 + int(k) % 3 if batcher else 1) for k in keys}
        parts = [G.arena_entry(batches[int(k)]) for k in keys]
        arena = np.frombuffer(b"".join(parts), np.uint8).copy()
        voffs = np.concatenate([[0], np.cumsum([len(p) for p in parts])]).astype(np.int32)
        recs = done.copy()
        recs["key"] = [order[int(k)] for k in done["key"]]
        qbuf, qoffs = r.wire_encode_read_requests(recs, arena, voffs)
        sent = O.split(qbuf, qoffs)
        assert sent == [G.read_request_bytes(batcher, int(d["slot"]), batches[int(d["key"])]) for d in done]
        # the replica: decode, defer or answer, then release as the log executes
        xbuf, xoffs = O.pack(sent)
        _, _, _, reads, _, split = eng.wire_decode_replica_inbound(xbuf, xoffs)
        assert split == len(sent)
        rr = ReplicaReads()
        outs = [r.replica(reads)]
        want_out = [np.array([x + (0,) for x in (rr.handle_read(int(q["slot"]), int(q["handle"])) for q in reads)
                              if x is not None], RO.READ_REPLY)]
        for W in (1 << 10, 1 << 12, (1 << 12) + groups):
            outs.append(r.advance(W))
            want_out.append(np.array([x + (0,) for x in rr.execute_log(W)], RO.READ_REPLY))
        RT.same_outputs(outs, want_out, "replica")


def mixed_batch(g, n, n_slots):
    """ReplicaInbound bytes in alternating runs of reads (all six members, empty messages between) and Chosen (every
    slot once, shuffled), hand-built; and per message what it carries: ("c", slot) or ("r", slot, commands)."""
    cmd = bytes.fromhex("0a0a0a0461626364100118021203787978")       # Command{CommandId{abcd, 1, 2}, xyx}
    cf = b"\x12" + bytes([len(cmd)]) + cmd
    ev = b"\x0a" + bytes([len(cmd)]) + cmd

    def vi(v):
        v &= (1 << 64) - 1
        out = b""
        while v >= 0x80:
            out += bytes([(v & 0x7f) | 0x80]); v >>= 7
        return out + bytes([v])

    def fld(f, body):
        return vi(f << 3 | 2) + vi(len(body)) + body
    slots = g.permutation(n_slots)
    msgs, desc, si = [], [], 0
    while len(msgs) < n or si < n_slots:
        for _ in range(int(g.integers(1, max(2, n // 16)))):          # a run of reads
            k = int(g.choice(8, p=[0.05, 0, 0.55, 0.15, 0.15, 0.04, 0.03, 0.03]))
            s = int(g.integers(-1, n_slots + 8))
            if k in (2, 3):
                msgs.append(fld(k, b"\x08" + vi(s) + cf)); desc.append(("r", s, 1))
            elif k == 4:
                msgs.append(fld(4, ev)); desc.append(("r", -1, 1))
            elif k in (5, 6):
                c = int(g.choice([0, 1, 64]))
                msgs.append(fld(k, b"\x08" + vi(s) + cf * c)); desc.append(("r", s, c))
            elif k == 7:
                c = int(g.choice([0, 2, 64]))
                msgs.append(fld(7, ev * c)); desc.append(("r", -1, c))
            else:
                msgs.append(b""); desc.append(("e",))
        run = n_slots - si if len(msgs) >= n else int(g.integers(0, max(1, n_slots // 8)))
        for s in slots[si: si + run]:                                   # a run of Chosen
            msgs.append(fld(1, b"\x08" + vi(int(s)) + b"\x12\x02\x12\x00")); desc.append(("c", int(s)))
        si += len(slots[si: si + run])
    return msgs, desc


@pytest.mark.parametrize("n", [3000, 1 << 20])
def test_mixed_batches_split_loop(n):
    """Chosen and reads interleaved, processed by looping on `split`: the replies equal handling the messages one at
    a time in delivery order (the transcription), the log's watermark the first hole."""
    g = np.random.default_rng(n)
    n_slots = max(4096, n // 4)
    msgs, desc = mixed_batch(g, n, n_slots)
    buf, offs = O.pack(msgs)
    with Engine(1, 1, 3, slot_capacity=n_slots, max_batch=1 << 20) as eng, \
            Reads(eng, READS_CLIENT, key_capacity=1, pending_capacity=1 << 22, max_batch=1 << 22) as r:
        got, start, handle, calls = [], 0, 0, 0
        while start < len(msgs):
            o = offs[start:] - offs[start]
            kind, chosen, _, reads, _, split = eng.wire_decode_replica_inbound(buf[offs[start]:], o, 0, handle)
            assert split > 0
            got.append(r.replica(reads))
            eng.replica_chosen(chosen)
            got.append(r.advance(eng.chosen_watermark()))
            handle += len(reads); start += split; calls += 1
        # one message at a time, in delivery order
        rr, imm, handle, W = ReplicaReads(), [], 0, 0
        chosen_set = np.zeros(n_slots + 1, bool)
        for d in desc:
            if d[0] == "r":
                for _ in range(d[2]):
                    x = rr.handle_read(d[1], handle)
                    handle += 1
                    if x is not None:
                        imm.append(x + (0,))
            elif d[0] == "c":
                chosen_set[d[1]] = True
                while chosen_set[W]:
                    W += 1
                imm.extend(x + (0,) for x in rr.execute_log(W))
        flat = np.concatenate([np.asarray(x).view(np.int32).reshape(-1) for x in got])
        assert np.array_equal(flat, np.array(imm, RO.READ_REPLY).view(np.int32).reshape(-1))
        assert eng.chosen_watermark() == W == n_slots and calls > 1
