"""Golden wire vectors for vanilla Mencius: tests/golden/wire_vanilla_mencius.json.

Built the way make_wire_golden.py builds the MultiPaxos and Mencius vectors: the reference serialises with scalapb
over protobuf-java (every *Serializer is ProtoSerializer, shared/src/main/scala/frankenpaxos/ProtoSerializer.scala:
3-11), neither of which runs here, so the bytes come from an INDEPENDENT implementation of the same published
format, Google's Python protobuf runtime, with the message shapes transcribed from
shared/src/main/scala/frankenpaxos/vanillamencius/VanillaMencius.proto.  Its vectors stay in a file of their own.

    python tests/golden/make_wire_vm_golden.py      # rewrites tests/golden/wire_vanilla_mencius.json
"""
import json
import os

import numpy as np
from google.protobuf import descriptor_pb2, descriptor_pool, message_factory

F = descriptor_pb2.FieldDescriptorProto
# int32 values around every varint length boundary, negative ones included (10-byte varints)
EDGE = [0, 1, 127, 128, 255, 300, 16383, 16384, (1 << 21) - 1, 1 << 21, (1 << 28) - 1, 1 << 28, (1 << 31) - 1, -1,
        -(1 << 31)]


VPKG = "frankenpaxos.vanillamencius"


def build_vanilla_pool():
    """S/vanillamencius/VanillaMencius.proto: Noop, CommandId, Command, CommandOrNoop :84-93, ClientRequest :95-100,
    Phase1a, PendingSlotInfo, ChosenSlotInfo, Phase1bSlotInfo, Phase1b, Phase2a :154-162, Skip :164-172, Phase2b
    :174-181, Chosen :183-190, Phase1Nack, Phase2Nack :209-215, ServerInbound :227-241.  A pool of its own: the
    package has its own Noop / Command / CommandId."""
    fdp = descriptor_pb2.FileDescriptorProto()
    fdp.name = "VanillaMencius.proto"; fdp.package = VPKG; fdp.syntax = "proto2"

    def msg(name, fields, oneof=None, oneof_fields=None):
        m = fdp.message_type.add(); m.name = name
        if oneof:
            m.oneof_decl.add().name = oneof
        for (fname, num, ftype, label, tname) in fields:
            f = m.field.add(); f.name = fname; f.number = num; f.type = ftype; f.label = label
            if tname:
                f.type_name = f".{VPKG}.{tname}"
            if oneof and (oneof_fields is None or fname in oneof_fields):
                f.oneof_index = 0

    REQ, OPT, REP = F.LABEL_REQUIRED, F.LABEL_OPTIONAL, F.LABEL_REPEATED
    I32, BYT, MSG, BOOL = F.TYPE_INT32, F.TYPE_BYTES, F.TYPE_MESSAGE, F.TYPE_BOOL
    msg("Noop", [])
    msg("CommandId", [("client_address", 1, BYT, REQ, None), ("client_pseudonym", 2, I32, REQ, None),
                      ("client_id", 3, I32, REQ, None)])
    msg("Command", [("command_id", 1, MSG, REQ, "CommandId"), ("command", 2, BYT, REQ, None)])
    msg("CommandOrNoop", [("command", 1, MSG, OPT, "Command"), ("noop", 2, MSG, OPT, "Noop")], "value")
    msg("ClientRequest", [("command", 1, MSG, REQ, "Command")])
    msg("Phase1a", [("round", 1, I32, REQ, None), ("start_slot_inclusive", 2, I32, REQ, None),
                    ("stop_slot_exclusive", 3, I32, REQ, None)])
    msg("PendingSlotInfo", [("vote_round", 1, I32, REQ, None), ("vote_value", 2, MSG, REQ, "CommandOrNoop")])
    msg("ChosenSlotInfo", [("value", 1, MSG, REQ, "CommandOrNoop"), ("is_revocation", 2, BOOL, REQ, None)])
    msg("Phase1bSlotInfo", [("slot", 1, I32, REQ, None), ("pending_slot_info", 2, MSG, OPT, "PendingSlotInfo"),
                            ("chosen_slot_info", 3, MSG, OPT, "ChosenSlotInfo")], "info",
        ("pending_slot_info", "chosen_slot_info"))
    msg("Phase1b", [("server_index", 1, I32, REQ, None), ("round", 2, I32, REQ, None),
                    ("start_slot_inclusive", 3, I32, REQ, None), ("stop_slot_exclusive", 4, I32, REQ, None),
                    ("info", 5, MSG, REP, "Phase1bSlotInfo")])
    msg("Phase2a", [("sending_server", 1, I32, REQ, None), ("slot", 2, I32, REQ, None), ("round", 3, I32, REQ, None),
                    ("command_or_noop", 4, MSG, REQ, "CommandOrNoop")])
    msg("Skip", [("server_index", 1, I32, REQ, None), ("start_slot_inclusive", 2, I32, REQ, None),
                 ("stop_slot_exclusive", 3, I32, REQ, None)])
    msg("Phase2b", [("server_index", 1, I32, REQ, None), ("slot", 2, I32, REQ, None), ("round", 3, I32, REQ, None)])
    msg("Chosen", [("slot", 1, I32, REQ, None), ("command_or_noop", 2, MSG, REQ, "CommandOrNoop"),
                   ("isRevocation", 3, BOOL, REQ, None)])
    msg("Phase1Nack", [("start_slot_inclusive", 1, I32, REQ, None), ("stop_slot_exclusive", 2, I32, REQ, None),
                       ("round", 3, I32, REQ, None)])
    msg("Phase2Nack", [("slot", 1, I32, REQ, None), ("round", 2, I32, REQ, None)])
    msg("ServerInbound", [("client_request", 1, MSG, OPT, "ClientRequest"), ("phase1a", 2, MSG, OPT, "Phase1a"),
                          ("phase1b", 3, MSG, OPT, "Phase1b"), ("phase2a", 4, MSG, OPT, "Phase2a"),
                          ("phase2b", 5, MSG, OPT, "Phase2b"), ("skip", 6, MSG, OPT, "Skip"),
                          ("chosen", 7, MSG, OPT, "Chosen"), ("phase1_nack", 8, MSG, OPT, "Phase1Nack"),
                          ("phase2_nack", 9, MSG, OPT, "Phase2Nack")], "request")
    pool = descriptor_pool.DescriptorPool()
    pool.Add(fdp)
    return pool


VPOOL = build_vanilla_pool()


def vcls(name):
    return message_factory.GetMessageClass(VPOOL.FindMessageTypeByName(f"{VPKG}.{name}"))


def vcommand(g, cmd_len):
    c = vcls("Command")()
    c.command_id.client_address = bytes(g.integers(0, 256, size=6, dtype=np.uint8))
    c.command_id.client_pseudonym = int(g.integers(0, 1 << 20))
    c.command_id.client_id = int(g.integers(0, 1 << 30))
    c.command = bytes(g.integers(0, 256, size=cmd_len, dtype=np.uint8))
    return c


def vvalue(g, cmd_len):
    """A vanilla CommandOrNoop: cmd_len < 0 -> Noop."""
    v = vcls("CommandOrNoop")()
    if cmd_len < 0:
        v.noop.SetInParent()
    else:
        v.command.CopyFrom(vcommand(g, cmd_len))
    return v


def vanilla_cases():
    g = np.random.Generator(np.random.PCG64(20261017))
    SI = vcls("ServerInbound")
    cases = []

    def add(t, m, **fields):
        cases.append(dict(type=t, hex=m.SerializeToString().hex(), **fields))
    E = len(EDGE)
    for k in range(E):
        a, b, c = EDGE[k], EDGE[(k + 3) % E], EDGE[(k + 6) % E]
        add("phase2b", SI(phase2b=vcls("Phase2b")(server_index=a, slot=b, round=c)), server_index=a, slot=b, round=c)
        add("skip", SI(skip=vcls("Skip")(server_index=b, start_slot_inclusive=c, stop_slot_exclusive=a)),
            server_index=b, start=c, stop=a)
        add("phase2_nack", SI(phase2_nack=vcls("Phase2Nack")(slot=c, round=a)), slot=c, round=a)
    # values: Noop, an empty command, commands around the 1- / 2-byte length-varint boundaries
    shapes = [-1, 0, 1, 90, 100, 101, 102, 200, 300]
    for k, cl in enumerate(shapes):
        v = vvalue(g, cl)
        srv, sl, rd = EDGE[k % E], EDGE[(k + 4) % E], EDGE[(k + 9) % E]
        add("phase2a", SI(phase2a=vcls("Phase2a")(sending_server=srv, slot=sl, round=rd, command_or_noop=v)),
            sending_server=srv, slot=sl, round=rd, value_hex=v.SerializeToString().hex())
        # what a coordinator of 7 servers sends for its own slot: sending_server = slot mod 7
        add("phase2a.coordinator", SI(phase2a=vcls("Phase2a")(sending_server=sl % 7, slot=sl, round=rd, command_or_noop=v)),
            sending_server=sl % 7, slot=sl, round=rd, value_hex=v.SerializeToString().hex())
        for rev in (False, True):
            add("chosen", SI(chosen=vcls("Chosen")(slot=sl, command_or_noop=v, isRevocation=rev)), slot=sl,
                is_revocation=int(rev), value_hex=v.SerializeToString().hex())
        if cl >= 0:
            add("client_request", SI(client_request=vcls("ClientRequest")(command=v.command)),
                value_hex=v.SerializeToString().hex())
    # the messages the host keeps: reported by kind with their body
    p1a = vcls("Phase1a")(round=3, start_slot_inclusive=7, stop_slot_exclusive=700)
    p1b = vcls("Phase1b")(server_index=2, round=3, start_slot_inclusive=7, stop_slot_exclusive=700)
    i = p1b.info.add(); i.slot = 14; i.pending_slot_info.vote_round = 1; i.pending_slot_info.vote_value.noop.SetInParent()
    p1n = vcls("Phase1Nack")(start_slot_inclusive=7, stop_slot_exclusive=700, round=9)
    for t, m in (("phase1a", SI(phase1a=p1a)), ("phase1b", SI(phase1b=p1b)), ("phase1_nack", SI(phase1_nack=p1n))):
        body = getattr(m, t).SerializeToString()
        add(t, m, body_hex=body.hex())
    # parser robustness, with what Google's runtime makes of each byte string (it does not enforce `required`)
    p2b = SI(phase2b=vcls("Phase2b")(server_index=3, slot=300, round=2)).SerializeToString()
    ch = SI(chosen=vcls("Chosen")(slot=5, command_or_noop=vvalue(g, -1), isRevocation=False)).SerializeToString()
    p2a = SI(phase2a=vcls("Phase2a")(sending_server=1, slot=8, round=0, command_or_noop=vvalue(g, 4))).SerializeToString()
    chb = bytes.fromhex("0805" "12021200")                          # Chosen body without isRevocation
    odd = {
        "truncated": p2b[:-1],
        "truncated value": p2a[:-2],
        "overlong varint": bytes([0x2a, 15]) + bytes([0x08] + [0x80] * 10 + [0x01]) + bytes.fromhex("1000" "1800"),
        "unknown fields": bytes.fromhex("5003") + bytes([0x2a, len(p2b) - 2 + 12]) + p2b[2:]
        + bytes.fromhex("2001" "3a03616263" "4d01020304") + bytes.fromhex("6a00"),
        "oneof set twice: last member wins": p2b + ch,
        "oneof set twice, the other order": ch + p2b,
        "missing required bool": bytes([0x3a, len(chb)]) + chb,
        "bool encoded as 2": bytes([0x3a, len(chb) + 2]) + chb + bytes.fromhex("1802"),
        "bool as a ten-byte varint with only bit 63 set": bytes([0x3a, len(chb) + 11]) + chb
        + bytes.fromhex("18" "80808080808080808001"),
        "missing command_or_noop": bytes.fromhex("3a04" "0805" "1800"),
        "Phase2a missing command_or_noop": bytes.fromhex("2206" "0801" "1008" "1800"),
        "command_or_noop twice": bytes([0x3a, len(chb) + 6]) + chb + bytes.fromhex("12021200" "1800"),
        "client_request without command": bytes.fromhex("0a00"),
        "group wire type": bytes([0x2a, 7]) + bytes.fromhex("0803" "1001" "1802" "0b"),
        "empty message": b"",
    }
    KIND = {None: 0, "client_request": 1, "phase1a": 2, "phase1b": 3, "phase2a": 4, "phase2b": 5, "skip": 6,
            "chosen": 7, "phase1_nack": 8, "phase2_nack": 9}
    for name, raw in odd.items():
        m = SI()
        try:
            m.ParseFromString(raw)
            which = m.WhichOneof("request")
            verdict = {"kind": KIND[which], "initialized": m.IsInitialized()}
            if which in ("phase2b", "chosen", "phase2a"):
                verdict["fields"] = {f.name: v for f, v in getattr(m, which).ListFields() if f.type != F.TYPE_MESSAGE}
        except Exception as e:          # google.protobuf.message.DecodeError
            verdict = {"error": type(e).__name__}
        cases.append({"type": "robustness", "name": name, "hex": raw.hex(), "verdict": verdict})
    return cases


def main():
    cases = vanilla_cases()
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "wire_vanilla_mencius.json")
    json.dump({"generator": "tests/golden/make_wire_vm_golden.py (python protobuf runtime "
                            + __import__("google.protobuf").protobuf.__version__ + ")", "cases": cases},
              open(out, "w"), indent=0)
    print(len(cases), "cases ->", out)


if __name__ == "__main__":
    main()
