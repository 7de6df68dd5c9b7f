"""The MultiPaxos replica / read-path wire oracle (tests/wire_reads_oracle.cc) against
tests/golden/wire_multipaxos_reads.json (bytes and verdicts of Google's Python protobuf runtime over
MultiPaxos.proto's shapes), against that runtime on random messages, and under byte mutations."""
import importlib.util
import json
import os

import numpy as np
import pytest

import wire_reads_oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = json.load(open(os.path.join(HERE, "golden", "wire_multipaxos_reads.json")))
CASES, KEY_CAP = GOLD["cases"], GOLD["key_capacity"]


def of(inbound):
    return [c for c in CASES if c["inbound"] == inbound]


def golden_module():
    pytest.importorskip("google.protobuf")
    spec = importlib.util.spec_from_file_location("make_wire_reads_golden",
                                                  os.path.join(HERE, "golden", "make_wire_reads_golden.py"))
    G = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(G)
    return G


def replica_view(raw_msgs, res):
    """Per message of a decode that refused nothing and has no split: {status, kind, slot, value_hex, commands}."""
    st, idx, kind, chosen, cvals, reads, rcmds, split = res
    buf = b"".join(raw_msgs)
    offs = np.concatenate([[0], np.cumsum([len(m) for m in raw_msgs])])
    out, ci, ri = [], 0, 0
    for i, k in enumerate(kind):
        if k == 0:
            out.append({"status": 0, "kind": 0})
        elif k == 1:
            o, ln = cvals[ci]
            out.append({"status": 0, "kind": 1, "slot": int(chosen[ci]["slot"]), "value_hex": buf[o:o + ln].hex()})
            assert chosen[ci]["value_id"] == i
            ci += 1
        else:
            lo, hi = offs[i], offs[i + 1]
            cmds, slot = [], -1 if k in (4, 7) else None
            while ri < len(reads) and lo <= rcmds[ri][0] < hi:
                o, ln = rcmds[ri]
                cmds.append(buf[o:o + ln])
                slot = int(reads[ri]["slot"]); assert reads[ri]["handle"] == ri
                ri += 1
            out.append({"status": 0, "kind": int(k), "slot": slot, "commands": cmds})
    return out


def canonical_commands(G, cmds):
    """Command bytes as the runtime re-serialises them."""
    out = []
    for c in cmds:
        m = G.cls("Command")(); m.ParseFromString(c); out.append(m.SerializeToString().hex())
    return out


def test_golden_replica_one_at_a_time():
    G = golden_module()
    for c in of("replica"):
        raw = bytes.fromhex(c["hex"])
        buf, offs = O.pack([raw])
        res = O.decode_replica(buf, offs)
        e = c["expect"]
        assert res[0] == e["status"], c["name"]
        if e["status"]:
            assert res[1] == 0, c["name"]
            continue
        (got,) = replica_view([raw], res)
        assert got["kind"] == e["kind"], c["name"]
        if e["kind"] == 1:
            assert (got["slot"], got["value_hex"]) == (e["slot"], e["value_hex"]), c["name"]
        elif e["kind"]:
            assert canonical_commands(G, got["commands"]) == e["commands"], c["name"]
            if e["commands"]:
                assert got["slot"] == e["slot"], c["name"]


def test_golden_deviations_are_documented_refusals():
    dev = [c for c in CASES if c.get("deviation")]
    assert len(dev) >= 3 and all(c["runtime"]["status"] == 0 for c in dev)
    # and the mutation test's detector knows them, and nothing the codec accepts
    assert all(documented_deviation(bytes.fromhex(c["hex"]), "replica") for c in dev)
    assert not any(documented_deviation(bytes.fromhex(c["hex"]), c["inbound"]) for c in CASES
                   if c["inbound"] in ("replica", "client", "batcher") and c["expect"]["status"] == 0)


def test_golden_reads_inbounds():
    for inbound, batcher in (("client", False), ("batcher", True)):
        for c in of(inbound):
            buf, offs = O.pack([bytes.fromhex(c["hex"])])
            st, idx, kind, out, spans = O.decode_reads(buf, offs, batcher, KEY_CAP)
            e = c["expect"]
            assert st == e["status"], c["name"]
            if st:
                continue
            assert int(kind[0]) == e["kind"], c["name"]
            assert tuple(int(x) for x in out[0].tolist()) == (e["key"], e["id"], e["voter"], e["slot"]), c["name"]


def test_golden_encoders():
    for c in of("acceptor"):
        raw = bytes.fromhex(c["hex"])
        # the request's member and body, as fpx_wire_decode_inbound(FPX_WIRE_ACCEPTOR_INBOUND) writes them
        assert raw[0] & 7 == 2 and raw[1] < 0x80
        kind = raw[0] >> 3
        rec = np.array([((c["group"] << 16) | c["acceptor"], c["max_voted_slot"], 2, raw[1])], O.WIRE_REC)
        buf, _ = O.pack([raw])
        st, idx, out, offs = O.encode_max_slot_replies(buf, [kind], rec, 2, 3)
        assert st == c["expect"]["status"], c["name"]
        if st == 0:
            assert bytes(out).hex() == c["expect"]["reply_hex"], c["name"]
    for c in of("read_request"):
        arena = bytes.fromhex(c["arena_hex"])
        rec = np.array([(0, 7, c["slot"], 0)], O.READ_SLOT)
        st, idx, out, offs = O.encode_read_requests(rec, c["batcher"], np.frombuffer(arena, np.uint8), [0, len(arena)])
        assert st == 0 and bytes(out).hex() == c["hex"], c["name"]


def test_random_replica_batches_against_runtime():
    G = golden_module()
    g = np.random.Generator(np.random.PCG64(5))
    for trial in range(20):
        msgs = [G.replica_message(g, int(g.integers(1, 8))).SerializeToString() for _ in range(int(g.integers(1, 60)))]
        # reads only, then Chosen only: no split inside
        msgs.sort(key=lambda m: m[0] == 0x0a)
        buf, offs = O.pack(msgs)
        res = O.decode_replica(buf, offs, handle_base=0)
        assert res[0] == 0 and res[7] == len(msgs)
        for raw, got in zip(msgs, replica_view(msgs, res)):
            e = G.expect_replica(raw)
            assert got["kind"] == e["kind"]
            if e["kind"] == 1:
                assert (got["slot"], got["value_hex"]) == (e["slot"], e["value_hex"])
            else:
                assert canonical_commands(G, got["commands"]) == e["commands"]


def test_split_rule():
    G = golden_module()
    g = np.random.Generator(np.random.PCG64(6))
    for trial in range(50):
        kinds = g.integers(0, 8, size=int(g.integers(1, 40)))
        msgs = [G.replica_message(g, int(k)).SerializeToString() if k else b"" for k in kinds]
        buf, offs = O.pack(msgs)
        res = O.decode_replica(buf, offs)
        c0 = next((i for i, k in enumerate(kinds) if k == 1), None)
        want = next((i for i, k in enumerate(kinds) if c0 is not None and i > c0 and k >= 2), len(kinds))
        assert res[0] == 0 and res[7] == want
        assert len(res[3]) == int((kinds[:want] == 1).sum())


def test_random_reads_inbounds_against_runtime():
    G = golden_module()
    g = np.random.Generator(np.random.PCG64(7))
    for batcher in (False, True):
        make = G.batcher_message if batcher else G.client_message
        msgs = [make(g, int(g.integers(1, 5 if batcher else 6))).SerializeToString() for _ in range(300)]
        buf, offs = O.pack(msgs)
        st, idx, kind, out, spans = O.decode_reads(buf, offs, batcher, KEY_CAP)
        assert st == 0
        for i, raw in enumerate(msgs):
            e = G.expect_reads(raw, batcher, KEY_CAP)
            assert (int(kind[i]), *(int(x) for x in out[i].tolist())) == \
                (e["kind"], e["key"], e["id"], e["voter"], e["slot"])


def mutate(g, raw):
    b = bytearray(raw)
    for _ in range(int(g.integers(1, 4))):
        op = int(g.integers(0, 3))
        if op == 0 and b:
            b[int(g.integers(0, len(b)))] = int(g.integers(0, 256))
        elif op == 1 and b:
            i = int(g.integers(0, len(b)))
            del b[i:i + int(g.integers(1, 4))]
        else:
            b.insert(int(g.integers(0, len(b) + 1)), int(g.integers(0, 256)))
    return bytes(b)


def _fields(b):
    """(field, wire type, payload) of one message level; wire types 3 / 4 are yielded and end the walk."""
    p = 0

    def varint():
        nonlocal p
        v, k = 0, 0
        while True:
            c = b[p]; p += 1
            v |= (c & 0x7f) << (7 * k); k += 1
            if not c & 0x80:
                return v
    while p < len(b):
        t = varint()
        f, wt = t >> 3, t & 7
        if wt in (3, 4):
            yield f, wt, None
            return
        if wt == 0:
            yield f, wt, varint()
        elif wt in (1, 5):
            n = 8 if wt == 1 else 4
            yield f, wt, b[p:p + n]; p += n
        else:
            n = varint()
            yield f, wt, b[p:p + n]; p += n


def _has_group(b, nested=()):
    """A group wire type at this level, or in the length-delimited fields `nested` = ((field, sub-nested), ...)."""
    sub = dict(nested)
    for f, wt, v in _fields(b):
        if wt in (3, 4):
            return True
        if wt == 2 and f in sub and _has_group(v, sub[f]):
            return True
    return False


def documented_deviation(raw, inbound):
    """The bytes hold one of the codec's documented refusals that the runtime accepts, at a level the codec parses:
    a group wire type, a second Command in a singular read member, a second value in a Chosen (DESIGN section 7)."""
    members = 7 if inbound == "replica" else 5 if inbound == "client" else 4
    run, which = [], 0
    for f, wt, v in _fields(raw):
        if wt in (3, 4):
            return True
        if wt == 2 and f <= members:
            if f != which:
                which, run = f, []
            run.append(v)
    CID = ((1, ()),)
    if inbound == "replica":
        cf = 1 if which in (4, 7) else 2
        seen = 0
        for body in run:
            for f, wt, v in _fields(body):
                if wt in (3, 4):
                    return True
                if wt == 2 and f == (2 if which == 1 else cf):
                    seen += 1
                    if which != 1 and _has_group(v, ((1, ()),)):
                        return True
        return which in (1, 2, 3, 4) and seen > 1
    if which != 4:
        return False
    return any(_has_group(body, CID if inbound == "client" else ()) for body in run)


def test_mutations_never_accept_what_the_runtime_rejects():
    """A mutated message the oracle accepts parses in the runtime to the same records; one the runtime rejects
    the oracle rejects; one the runtime accepts the oracle accepts unless it holds a documented deviation."""
    G = golden_module()
    g = np.random.Generator(np.random.PCG64(8))
    accepted = refused = 0
    for trial in range(3000):
        raw = mutate(g, G.replica_message(g, int(g.integers(1, 8)), int(g.integers(0, 3))).SerializeToString())
        buf, offs = O.pack([raw])
        res = O.decode_replica(buf, offs)
        e = G.expect_replica(raw)
        if e["status"]:
            assert res[0] != 0, raw.hex()
            continue
        if res[0]:
            assert documented_deviation(raw, "replica"), raw.hex()
            refused += 1
            continue
        accepted += 1
        (got,) = replica_view([raw], res)
        assert got["kind"] == e["kind"], raw.hex()
        if e["kind"] == 1:
            assert (got["slot"], got["value_hex"]) == (e["slot"], e["value_hex"])
        elif e["kind"]:
            assert canonical_commands(G, got["commands"]) == e["commands"]
    assert accepted > 100 and refused < accepted
    for batcher in (False, True):
        make = G.batcher_message if batcher else G.client_message
        for trial in range(1000):
            raw = mutate(g, make(g, 4).SerializeToString())
            buf, offs = O.pack([raw])
            st, idx, kind, out, spans = O.decode_reads(buf, offs, batcher, KEY_CAP)
            e = G.expect_reads(raw, batcher, KEY_CAP)
            if st == 0 and kind[0] != 4:
                continue                  # the other members are not parsed: the host reads them from their span
            if e["status"]:
                assert st != 0, raw.hex()
            elif st == 0:
                assert (int(kind[0]), *(int(x) for x in out[0].tolist())) == \
                    (e["kind"], e["key"], e["id"], e["voter"], e["slot"]), raw.hex()
            else:
                assert documented_deviation(raw, "batcher" if batcher else "client"), raw.hex()


def test_overflow_is_reported_at_the_first_message_that_does_not_fit():
    G = golden_module()
    g = np.random.Generator(np.random.PCG64(9))
    msgs = [G.replica_message(g, 5, 3).SerializeToString() for _ in range(10)]
    buf, offs = O.pack(msgs)
    res = O.decode_replica(buf, offs, reads_capacity=10)
    assert (res[0], res[1]) == (-8, 3)


def test_non_monotone_offsets_are_refused_in_their_tile():
    """A message whose offsets run backwards is FPX_ERR_WIRE at its index, while the messages around it, which
    overlap each other, are read where the codec reads them (inside the tile's span)."""
    for big in (False, True):
        buf, offs = O.overlapping_batch(big)
        res = O.decode_replica(buf, offs)
        assert (res[0], res[1]) == (-15, 1)
        assert list(res[2]) == [2, 0, 1, 2] and res[7] == 3
