"""Golden wire vectors for Compartmentalized Mencius' noop ranges and replica: tests/golden/wire_mencius.json.

Built the way make_wire_golden.py builds its Mencius vectors: the reference serialises with scalapb over
protobuf-java (every *Serializer is ProtoSerializer, shared/src/main/scala/frankenpaxos/ProtoSerializer.scala:3-11),
neither of which runs here, so the bytes come from an INDEPENDENT implementation of the same published format,
Google's Python protobuf runtime, with the message shapes transcribed from
shared/src/main/scala/frankenpaxos/mencius/Mencius.proto.  Its vectors stay in a file of their own.

    python tests/golden/make_wire_mencius_golden.py      # rewrites tests/golden/wire_mencius.json
"""
import json
import os

import numpy as np
from google.protobuf import descriptor_pb2, descriptor_pool, message_factory

F = descriptor_pb2.FieldDescriptorProto
# int32 values around every varint length boundary, negative ones included (10-byte varints)
EDGE = [0, 1, 127, 128, 255, 300, 16383, 16384, (1 << 21) - 1, 1 << 21, (1 << 28) - 1, 1 << 28, (1 << 31) - 1, -1,
        -(1 << 31)]
MPKG = "frankenpaxos.mencius"


def build_mencius_pool():
    """S/mencius/Mencius.proto: Noop :49-52, CommandId :54-62, Command :64-70, CommandBatch :72-77, CommandBatchOrNoop
    :79-88, Phase2bNoopRange :178-187, Chosen :189-195, ChosenNoopRange :197-203, Nack :266-271, LeaderInbound
    :322-337 (only nack = 7 and the member at 6 are transcribed), ProxyLeaderInbound :339-350 (phase2b_noop_range = 5
    and the members before it as opaque bodies), ReplicaInbound :363-371."""
    fdp = descriptor_pb2.FileDescriptorProto()
    fdp.name = "Mencius.proto"; fdp.package = MPKG; fdp.syntax = "proto2"

    def msg(name, fields, oneof=None):
        m = fdp.message_type.add(); m.name = name
        if oneof:
            m.oneof_decl.add().name = oneof
        for (fname, num, ftype, label, tname) in fields:
            f = m.field.add(); f.name = fname; f.number = num; f.type = ftype; f.label = label
            if tname:
                f.type_name = f".{MPKG}.{tname}"
            if oneof:
                f.oneof_index = 0

    REQ, OPT, REP = F.LABEL_REQUIRED, F.LABEL_OPTIONAL, F.LABEL_REPEATED
    I32, BYT, MSG = F.TYPE_INT32, F.TYPE_BYTES, F.TYPE_MESSAGE
    msg("Noop", [])
    msg("CommandId", [("client_address", 1, BYT, REQ, None), ("client_pseudonym", 2, I32, REQ, None),
                      ("client_id", 3, I32, REQ, None)])
    msg("Command", [("command_id", 1, MSG, REQ, "CommandId"), ("command", 2, BYT, REQ, None)])
    msg("CommandBatch", [("command", 1, MSG, REP, "Command")])
    msg("CommandBatchOrNoop", [("command_batch", 1, MSG, OPT, "CommandBatch"), ("noop", 2, MSG, OPT, "Noop")], "value")
    msg("Phase2bNoopRange", [("acceptor_group_index", 1, I32, REQ, None), ("acceptor_index", 2, I32, REQ, None),
                             ("slot_start_inclusive", 3, I32, REQ, None), ("slot_end_exclusive", 4, I32, REQ, None),
                             ("round", 5, I32, REQ, None)])
    msg("Chosen", [("slot", 1, I32, REQ, None), ("command_batch_or_noop", 2, MSG, REQ, "CommandBatchOrNoop")])
    msg("ChosenNoopRange", [("slot_start_inclusive", 1, I32, REQ, None), ("slot_end_exclusive", 2, I32, REQ, None)])
    msg("Nack", [("round", 1, I32, REQ, None)])
    msg("LeaderInfoRequestBatcher", [])
    msg("LeaderInbound", [("leader_info_request_batcher", 6, MSG, OPT, "LeaderInfoRequestBatcher"),
                          ("nack", 7, MSG, OPT, "Nack")], "request")
    msg("ProxyLeaderInbound", [("phase2b_noop_range", 5, MSG, OPT, "Phase2bNoopRange")], "request")
    msg("ReplicaInbound", [("chosen", 1, MSG, OPT, "Chosen"), ("chosen_noop_range", 2, MSG, OPT, "ChosenNoopRange")],
        "request")
    pool = descriptor_pool.DescriptorPool()
    pool.Add(fdp)
    return pool


POOL = build_mencius_pool()


def mcls(name):
    return message_factory.GetMessageClass(POOL.FindMessageTypeByName(f"{MPKG}.{name}"))


def payload(g, n_cmds, cmd_len):
    """A CommandBatchOrNoop: n_cmds < 0 -> Noop."""
    v = mcls("CommandBatchOrNoop")()
    if n_cmds < 0:
        v.noop.SetInParent()
        return v
    v.command_batch.SetInParent()
    for _ in range(n_cmds):
        c = v.command_batch.command.add()
        c.command_id.client_address = bytes(g.integers(0, 256, size=6, dtype=np.uint8))
        c.command_id.client_pseudonym = int(g.integers(0, 1 << 20))
        c.command_id.client_id = int(g.integers(0, 1 << 30))
        c.command = bytes(g.integers(0, 256, size=cmd_len, dtype=np.uint8))
    return v


def mencius_cases():
    g = np.random.Generator(np.random.PCG64(20261018))
    RI, PL, LI = mcls("ReplicaInbound"), mcls("ProxyLeaderInbound"), mcls("LeaderInbound")
    cases = []

    def add(t, m, **fields):
        cases.append(dict(type=t, hex=m.SerializeToString().hex(), **fields))
    E = len(EDGE)
    for k in range(E):
        a, b, c, d, e = EDGE[k], EDGE[(k + 2) % E], EDGE[(k + 5) % E], EDGE[(k + 7) % E], EDGE[(k + 11) % E]
        add("chosen_noop_range", RI(chosen_noop_range=mcls("ChosenNoopRange")(slot_start_inclusive=a, slot_end_exclusive=b)),
            start=a, end=b)
        add("phase2b_noop_range", PL(phase2b_noop_range=mcls("Phase2bNoopRange")(
            acceptor_group_index=a, acceptor_index=b, slot_start_inclusive=c, slot_end_exclusive=d, round=e)),
            acceptor_group_index=a, acceptor_index=b, start=c, end=d, round=e)
        add("nack", LI(nack=mcls("Nack")(round=a)), round=a)
    # values: Noop, an empty batch, batches around the 1- / 2-byte length-varint boundaries
    for k, (nc, cl) in enumerate([(-1, 0), (0, 0), (1, 0), (1, 90), (1, 100), (2, 40), (3, 100), (5, 300)]):
        v = payload(g, nc, cl)
        add("chosen", RI(chosen=mcls("Chosen")(slot=EDGE[k % E], command_batch_or_noop=v)), slot=EDGE[k % E],
            value_hex=v.SerializeToString().hex())
    # parser robustness, with what Google's runtime makes of each byte string (it does not enforce `required`)
    ch = RI(chosen=mcls("Chosen")(slot=5, command_batch_or_noop=payload(g, -1, 0))).SerializeToString()
    rg = RI(chosen_noop_range=mcls("ChosenNoopRange")(slot_start_inclusive=7, slot_end_exclusive=700)).SerializeToString()
    odd = {
        "truncated": rg[:-1],
        "truncated value": ch[:-1],
        "overlong varint": bytes([0x12, 15]) + bytes([0x08] + [0x80] * 10 + [0x01]) + bytes.fromhex("1007"),
        "unknown fields": bytes.fromhex("5003") + bytes([0x12, len(rg) - 2 + 12]) + rg[2:]
        + bytes.fromhex("2001" "3a03616263" "4d01020304") + bytes.fromhex("1a00"),
        "oneof set twice: last member wins": ch + rg,
        "oneof set twice, the other order": rg + ch,
        "missing end": bytes.fromhex("1202" "0807"),
        "missing command_batch_or_noop": bytes.fromhex("0a02" "0805"),
        "command_batch_or_noop twice": bytes.fromhex("0a0a" "0805" "12021200" "12021200"),
        "group wire type": bytes([0x12, 5]) + bytes.fromhex("0807" "1009" "0b"),
        "empty message": b"",
        "range end below start": RI(chosen_noop_range=mcls("ChosenNoopRange")(
            slot_start_inclusive=9, slot_end_exclusive=3)).SerializeToString(),
    }
    KIND = {None: 0, "chosen": 1, "chosen_noop_range": 2}
    for name, raw in odd.items():
        m = RI()
        try:
            m.ParseFromString(raw)
            which = m.WhichOneof("request")
            verdict = {"kind": KIND[which], "initialized": m.IsInitialized()}
            if which:
                verdict["fields"] = {f.name: v for f, v in getattr(m, which).ListFields() if f.type != F.TYPE_MESSAGE}
        except Exception as e:          # google.protobuf.message.DecodeError
            verdict = {"error": type(e).__name__}
        cases.append({"type": "robustness", "name": name, "hex": raw.hex(), "verdict": verdict})
    return cases


def main():
    cases = mencius_cases()
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "wire_mencius.json")
    json.dump({"generator": "tests/golden/make_wire_mencius_golden.py (python protobuf runtime "
                            + __import__("google.protobuf").protobuf.__version__ + ")", "cases": cases},
              open(out, "w"), indent=0)
    print(len(cases), "cases ->", out)


if __name__ == "__main__":
    main()
