"""Golden wire vectors of the new leader's Phase 1: LeaderInbound{phase1b} batches and the Phase2a re-proposals.

Produced, like make_wire_golden.py, by Google's Python protobuf runtime (an implementation independent of the
codec) over the shapes of shared/src/main/scala/frankenpaxos/multipaxos/MultiPaxos.proto: Phase1bSlotInfo
:254-261, Phase1b :263-271, Phase2a :273-280, Nack :455-460, LeaderInbound :525-539, ProxyLeaderInbound :541-549.
Each case is one LeaderInbound and what the runtime parses from it (or its error); each Phase2a case the canonical
ProxyLeaderInbound bytes of one record.

    python tests/golden/make_wire_phase1_golden.py      # rewrites tests/golden/wire_phase1.json
"""
import json
import os
import sys

import numpy as np
from google.protobuf import descriptor_pb2

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_wire_golden as base  # noqa: E402

F = descriptor_pb2.FieldDescriptorProto
PKG = base.PKG


def build_pool():
    """make_wire_golden's pool with Phase1b, Phase1bSlotInfo and the LeaderInbound phase1b member."""
    from google.protobuf import descriptor_pool
    fdp = descriptor_pb2.FileDescriptorProto()
    base.POOL.FindFileByName("MultiPaxos.proto").CopyToProto(fdp)
    fdp.name = "MultiPaxosPhase1.proto"
    REQ, REP, OPT = F.LABEL_REQUIRED, F.LABEL_REPEATED, F.LABEL_OPTIONAL
    I32, MSG = F.TYPE_INT32, F.TYPE_MESSAGE

    def add(m, name, num, ftype, label, tname=None, oneof=None):
        f = m.field.add(); f.name = name; f.number = num; f.type = ftype; f.label = label
        if tname:
            f.type_name = f".{PKG}.{tname}"
        if oneof is not None:
            f.oneof_index = oneof

    info = fdp.message_type.add(); info.name = "Phase1bSlotInfo"
    add(info, "slot", 1, I32, REQ); add(info, "vote_round", 2, I32, REQ)
    add(info, "vote_value", 3, MSG, REQ, "CommandBatchOrNoop")
    p1b = fdp.message_type.add(); p1b.name = "Phase1b"
    add(p1b, "group_index", 1, I32, REQ); add(p1b, "acceptor_index", 2, I32, REQ); add(p1b, "round", 3, I32, REQ)
    add(p1b, "info", 4, MSG, REP, "Phase1bSlotInfo")
    li = next(m for m in fdp.message_type if m.name == "LeaderInbound")
    add(li, "phase1b", 1, MSG, OPT, "Phase1b", oneof=0)
    pool = descriptor_pool.DescriptorPool()
    pool.Add(fdp)
    return pool


POOL = build_pool()


def cls(name):
    from google.protobuf import message_factory
    return message_factory.GetMessageClass(POOL.FindMessageTypeByName(f"{PKG}.{name}"))


def payload(g, n_cmds, cmd_len):
    v = cls("CommandBatchOrNoop")()
    v.ParseFromString(base.payload(g, n_cmds, cmd_len).SerializeToString())
    return v


def phase1b(g, group, acceptor, round_, infos):
    m = cls("LeaderInbound")()
    p = m.phase1b
    p.group_index, p.acceptor_index, p.round = group, acceptor, round_
    for slot, vr, shape in infos:
        i = p.info.add()
        i.slot, i.vote_round = slot, vr
        i.vote_value.CopyFrom(payload(g, *shape))
    return m.SerializeToString()


def verdict(raw):
    m = cls("LeaderInbound")()
    try:
        m.ParseFromString(raw)
    except Exception as e:          # google.protobuf.message.DecodeError
        return {"error": type(e).__name__}
    if not m.IsInitialized():       # scalapb's parseFrom: "Message missing required fields"
        return {"error": "missing required fields"}
    which = m.WhichOneof("request")
    out = {"kind": m.DESCRIPTOR.fields_by_name[which].number if which else 0}
    if which == "phase1b":
        p = m.phase1b
        out.update(group_index=p.group_index, acceptor_index=p.acceptor_index, round=p.round,
                   info=[[i.slot, i.vote_round, i.vote_value.SerializeToString().hex()] for i in p.info])
    return out


def main():
    g = np.random.Generator(np.random.PCG64(20261018))
    cases = {}
    cases["zero infos"] = phase1b(g, 0, 1, 5, [])
    cases["one info"] = phase1b(g, 0, 2, 5, [(7, 3, (1, 20))])
    cases["many infos"] = phase1b(g, 1, 0, 9, [(s, int(g.integers(0, 9)), (int(g.integers(-1, 3)), int(g.integers(0, 90))))
                                               for s in range(0, 300, 3)])
    cases["negative rounds and slots (ten-byte varints)"] = phase1b(g, 0, 0, -1, [(-5, -(1 << 31), (1, 4)), (3, -2, (-1, 0))])
    cases["noop values"] = phase1b(g, 0, 1, 4, [(0, 1, (-1, 0)), (1, 1, (-1, 0))])
    good = phase1b(g, 0, 1, 6, [(10, 2, (1, 8)), (11, 3, (-1, 0))])
    info = bytes.fromhex("0805" "1003") + b"\x1a\x02\x12\x00"
    cases["fields out of order"] = b"\x0a" + bytes([len(info) + 2 + 6]) + b"\x22" + bytes([len(info)]) + info + \
        bytes.fromhex("1806" "0801" "1000")
    cases["info fields out of order"] = b"\x0a" + bytes([6 + 2 + len(info)]) + bytes.fromhex("080010001806") + \
        b"\x22" + bytes([len(info)]) + b"\x1a\x02\x12\x00" + bytes.fromhex("1003" "0805")
    cases["repeated member merges"] = good + phase1b(g, 0, 2, 6, [(12, 1, (1, 3))])
    cases["another member replaces"] = good + base.cls("LeaderInbound")(nack=base.cls("Nack")(round=3)).SerializeToString()
    cases["replaced, then phase1b again"] = good + base.cls("LeaderInbound")(nack=base.cls("Nack")(round=3)).SerializeToString() \
        + phase1b(g, 0, 0, 6, [(13, 1, (-1, 0))])
    cases["unknown fields"] = b"\x52\x03abc" + good[:1] + bytes([good[1] + 5]) + good[2:] + b"\x4a\x03xyz" + \
        b"\x5a\x01q"
    cases["unknown field inside an info"] = b"\x0a" + bytes([6 + 2 + len(info) + 3]) + bytes.fromhex("080010001806") + \
        b"\x22" + bytes([len(info) + 3]) + info + b"\x2a\x01z"
    cases["truncated"] = good[:-1]
    cases["truncated info"] = b"\x0a" + bytes([6 + 2 + 5]) + bytes.fromhex("080010001806") + b"\x22\x05" + info[:5]
    cases["info missing vote_value"] = b"\x0a" + bytes([6 + 2 + 4]) + bytes.fromhex("080010001806") + b"\x22\x04" + info[:4]
    cases["phase1b missing round"] = b"\x0a\x04" + bytes.fromhex("08001000")
    cases["a nack"] = base.cls("LeaderInbound")(nack=base.cls("Nack")(round=8)).SerializeToString()
    cases["empty message"] = b""
    decode = [{"name": k, "hex": v.hex(), "verdict": verdict(v)} for k, v in cases.items()]
    # Phase2a: ProxyLeaderInbound{phase2a{slot, round, command_batch_or_noop}}
    enc = []
    for slot, rnd, shape in [(0, 0, (-1, 0)), (5, 2, (1, 10)), (127, 128, (2, 60)), ((1 << 31) - 1, -1, (1, 200)),
                             (300, 16384, (0, 0))]:
        v = base.payload(g, *shape)
        m = base.cls("ProxyLeaderInbound")(phase2a=base.cls("Phase2a")(slot=slot, round=rnd, command_batch_or_noop=v))
        enc.append({"slot": slot, "round": rnd, "noop": shape[0] < 0, "payload_hex": v.SerializeToString().hex(),
                    "hex": m.SerializeToString().hex()})
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "wire_phase1.json")
    json.dump({"generator": "tests/golden/make_wire_phase1_golden.py (python protobuf runtime "
                            + __import__("google.protobuf").protobuf.__version__ + ")", "decode": decode, "phase2a": enc},
              open(out, "w"), indent=0)
    print(len(decode), "+", len(enc), "cases ->", out)


if __name__ == "__main__":
    main()
