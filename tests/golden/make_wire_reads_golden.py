"""Golden wire vectors for the MultiPaxos replica and read path: tests/golden/wire_multipaxos_reads.json.

Built the way make_wire_golden.py builds the MultiPaxos vectors: the reference serialises with scalapb over
protobuf-java (every *Serializer is ProtoSerializer, shared/src/main/scala/frankenpaxos/ProtoSerializer.scala:3-11),
neither of which runs here, so the bytes and what they parse to come from an INDEPENDENT implementation of the same
published format, Google's Python protobuf runtime, with the message shapes transcribed from
shared/src/main/scala/frankenpaxos/multipaxos/MultiPaxos.proto.  The tests import the pool and the message
builders below for their random cases.

    python tests/golden/make_wire_reads_golden.py      # rewrites tests/golden/wire_multipaxos_reads.json
"""
import json
import os

import numpy as np
from google.protobuf import descriptor_pb2, descriptor_pool, message_factory

F = descriptor_pb2.FieldDescriptorProto
PKG = "frankenpaxos.multipaxos"
# int32 values around every varint length boundary, negative ones included (10-byte varints)
EDGE = [0, 1, 127, 128, 255, 300, 16383, 16384, (1 << 21) - 1, 1 << 21, (1 << 28) - 1, 1 << 28, (1 << 31) - 1, -1,
        -(1 << 31)]
REPLICA_MEMBERS = ["chosen", "read_request", "sequential_read_request", "eventual_read_request", "read_request_batch",
                   "sequential_read_request_batch", "eventual_read_request_batch"]
CLIENT_MEMBERS = ["client_reply", "not_leader_client", "leader_info_reply_client", "max_slot_reply", "read_reply"]
BATCHER_MEMBERS = ["read_request", "sequential_read_request", "eventual_read_request", "batch_max_slot_reply"]


def build_pool():
    """MultiPaxos.proto: Noop :183-186, CommandId :188-196, Command :198-204, CommandBatch, CommandBatchOrNoop
    :206-221, Phase1a, Phase2a :273-280, Chosen :292-298, ClientReply :300-307, MaxSlotRequest .. BatchMaxSlotReply
    :316-349, the read requests :351-396, ReadReply :398-405, NotLeaderClient, LeaderInfoReplyClient :419-434,
    ClientInbound :489-500, ReadBatcherInbound :513-523, AcceptorInbound :551-561, ReplicaInbound :563-576."""
    fdp = descriptor_pb2.FileDescriptorProto()
    fdp.name = "MultiPaxosReads.proto"; fdp.package = PKG; fdp.syntax = "proto2"

    def msg(name, fields, oneof=None):
        m = fdp.message_type.add(); m.name = name
        if oneof:
            m.oneof_decl.add().name = oneof
        for (fname, num, ftype, label, tname) in fields:
            f = m.field.add(); f.name = fname; f.number = num; f.type = ftype; f.label = label
            if tname:
                f.type_name = f".{PKG}.{tname}"
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
    msg("Phase1a", [("round", 1, I32, REQ, None), ("chosen_watermark", 2, I32, REQ, None)])
    msg("Phase2a", [("slot", 1, I32, REQ, None), ("round", 2, I32, REQ, None),
                    ("command_batch_or_noop", 3, MSG, REQ, "CommandBatchOrNoop")])
    msg("Chosen", [("slot", 1, I32, REQ, None), ("command_batch_or_noop", 2, MSG, REQ, "CommandBatchOrNoop")])
    msg("ClientReply", [("command_id", 1, MSG, REQ, "CommandId"), ("slot", 2, I32, REQ, None),
                        ("result", 3, BYT, REQ, None)])
    msg("MaxSlotRequest", [("command_id", 1, MSG, REQ, "CommandId")])
    msg("MaxSlotReply", [("command_id", 1, MSG, REQ, "CommandId"), ("group_index", 2, I32, REQ, None),
                         ("acceptor_index", 3, I32, REQ, None), ("slot", 4, I32, REQ, None)])
    msg("BatchMaxSlotRequest", [("read_batcher_index", 1, I32, REQ, None), ("read_batcher_id", 2, I32, REQ, None)])
    msg("BatchMaxSlotReply", [("read_batcher_index", 1, I32, REQ, None), ("read_batcher_id", 2, I32, REQ, None),
                              ("acceptor_index", 3, I32, REQ, None), ("slot", 4, I32, REQ, None)])
    for name in ("ReadRequest", "SequentialReadRequest"):
        msg(name, [("slot", 1, I32, REQ, None), ("command", 2, MSG, REQ, "Command")])
    for name in ("ReadRequestBatch", "SequentialReadRequestBatch"):
        msg(name, [("slot", 1, I32, REQ, None), ("command", 2, MSG, REP, "Command")])
    msg("EventualReadRequest", [("command", 1, MSG, REQ, "Command")])
    msg("EventualReadRequestBatch", [("command", 1, MSG, REP, "Command")])
    msg("ReadReply", [("command_id", 1, MSG, REQ, "CommandId"), ("slot", 2, I32, REQ, None),
                      ("result", 3, BYT, REQ, None)])
    msg("NotLeaderClient", [])
    msg("LeaderInfoReplyClient", [("round", 1, I32, REQ, None)])
    msg("ClientInbound", [("client_reply", 1, MSG, OPT, "ClientReply"), ("not_leader_client", 2, MSG, OPT, "NotLeaderClient"),
                          ("leader_info_reply_client", 3, MSG, OPT, "LeaderInfoReplyClient"),
                          ("max_slot_reply", 4, MSG, OPT, "MaxSlotReply"), ("read_reply", 5, MSG, OPT, "ReadReply")],
        "request")
    msg("ReadBatcherInbound", [("read_request", 1, MSG, OPT, "ReadRequest"),
                               ("sequential_read_request", 2, MSG, OPT, "SequentialReadRequest"),
                               ("eventual_read_request", 3, MSG, OPT, "EventualReadRequest"),
                               ("batch_max_slot_reply", 4, MSG, OPT, "BatchMaxSlotReply")], "request")
    msg("AcceptorInbound", [("phase1a", 1, MSG, OPT, "Phase1a"), ("phase2a", 2, MSG, OPT, "Phase2a"),
                            ("max_slot_request", 3, MSG, OPT, "MaxSlotRequest"),
                            ("batch_max_slot_request", 4, MSG, OPT, "BatchMaxSlotRequest")], "request")
    msg("ReplicaInbound", [("chosen", 1, MSG, OPT, "Chosen"), ("read_request", 2, MSG, OPT, "ReadRequest"),
                           ("sequential_read_request", 3, MSG, OPT, "SequentialReadRequest"),
                           ("eventual_read_request", 4, MSG, OPT, "EventualReadRequest"),
                           ("read_request_batch", 5, MSG, OPT, "ReadRequestBatch"),
                           ("sequential_read_request_batch", 6, MSG, OPT, "SequentialReadRequestBatch"),
                           ("eventual_read_request_batch", 7, MSG, OPT, "EventualReadRequestBatch")], "request")
    # the codec locates a Chosen's value without parsing it (as the Phase2a value of fpx_wire_decode_inbound): the
    # runtime's view of that is the same message with the CommandBatchOrNoop as opaque bytes
    msg("OpaqueChosen", [("slot", 1, I32, REQ, None), ("command_batch_or_noop", 2, BYT, REQ, None)])
    msg("OpaqueReplicaInbound", [("chosen", 1, MSG, OPT, "OpaqueChosen"), ("read_request", 2, MSG, OPT, "ReadRequest"),
                                 ("sequential_read_request", 3, MSG, OPT, "SequentialReadRequest"),
                                 ("eventual_read_request", 4, MSG, OPT, "EventualReadRequest"),
                                 ("read_request_batch", 5, MSG, OPT, "ReadRequestBatch"),
                                 ("sequential_read_request_batch", 6, MSG, OPT, "SequentialReadRequestBatch"),
                                 ("eventual_read_request_batch", 7, MSG, OPT, "EventualReadRequestBatch")], "request")
    pool = descriptor_pool.DescriptorPool()
    pool.Add(fdp)
    return pool


POOL = build_pool()


def cls(name):
    return message_factory.GetMessageClass(POOL.FindMessageTypeByName(f"{PKG}.{name}"))


def command(g, cmd_len=None, pseudo=None, cid=None):
    c = cls("Command")()
    c.command_id.client_address = bytes(g.integers(0, 256, size=int(g.integers(0, 20)), dtype=np.uint8))
    c.command_id.client_pseudonym = int(g.choice(EDGE)) if pseudo is None else pseudo
    c.command_id.client_id = int(g.choice(EDGE)) if cid is None else cid
    n = int(g.integers(0, 40)) if cmd_len is None else cmd_len
    c.command = bytes(g.integers(0, 256, size=n, dtype=np.uint8))
    return c


def value(g):
    v = cls("CommandBatchOrNoop")()
    if g.integers(0, 4) == 0:
        v.noop.SetInParent()
    else:
        v.command_batch.SetInParent()
        for _ in range(int(g.integers(0, 4))):
            v.command_batch.command.add().CopyFrom(command(g))
    return v


def replica_message(g, which, n_cmds=None):
    """A ReplicaInbound with member `which` (1..7); batch members get n_cmds Commands (random if None)."""
    m = cls("ReplicaInbound")()
    name = REPLICA_MEMBERS[which - 1]
    body = getattr(m, name)
    body.SetInParent()
    if which == 1:
        body.slot = int(g.choice(EDGE)); body.command_batch_or_noop.CopyFrom(value(g))
        return m
    if which not in (4, 7):
        body.slot = int(g.choice(EDGE))
    if which in (2, 3, 4):
        body.command.CopyFrom(command(g))
    else:
        for _ in range(int(g.integers(0, 6)) if n_cmds is None else n_cmds):
            body.command.add().CopyFrom(command(g))
    return m


def client_message(g, which):
    m = cls("ClientInbound")()
    if which == 4:
        r = m.max_slot_reply
        r.command_id.CopyFrom(command(g).command_id)
        r.group_index = int(g.choice([0, 1, 2, 0x7fff, 0x8000, -1])); r.acceptor_index = int(g.choice([0, 1, 4, 0x7fff, 0x8000, -1]))
        r.slot = int(g.choice(EDGE))
    elif which == 1:
        m.client_reply.command_id.CopyFrom(command(g).command_id); m.client_reply.slot = 3; m.client_reply.result = b"ok"
    elif which == 2:
        m.not_leader_client.SetInParent()
    elif which == 3:
        m.leader_info_reply_client.round = int(g.choice(EDGE))
    else:
        m.read_reply.command_id.CopyFrom(command(g).command_id); m.read_reply.slot = -1; m.read_reply.result = b""
    return m


def batcher_message(g, which):
    m = cls("ReadBatcherInbound")()
    if which == 4:
        r = m.batch_max_slot_reply
        r.read_batcher_index = int(g.choice(EDGE)); r.read_batcher_id = int(g.choice(EDGE))
        r.acceptor_index = int(g.choice([0, 1, 4, 0x7fff, 0x8000, -1])); r.slot = int(g.choice(EDGE))
    else:
        body = getattr(m, BATCHER_MEMBERS[which - 1])
        if which != 3:
            body.slot = int(g.choice(EDGE))
        body.command.CopyFrom(command(g))
    return m


# ---- what the runtime makes of a message: the codec's expected output ------------------------------------------
def parse(name, raw):
    """The runtime's message, or None where it rejects the bytes or `required` is not met."""
    m = cls(name)()
    try:
        m.ParseFromString(raw)
    except Exception:                                     # google.protobuf.message.DecodeError
        return None
    return m if m.IsInitialized() else None


def expect_replica(raw):
    """{status, kind, slot, value_hex, commands: [canonical Command hex]} of one ReplicaInbound (a Chosen's value
    as opaque bytes)."""
    m = parse("OpaqueReplicaInbound", raw)
    if m is None:
        return {"status": -15}
    w = m.WhichOneof("request")
    if w is None:
        return {"status": 0, "kind": 0}
    k = REPLICA_MEMBERS.index(w) + 1
    body = getattr(m, w)
    if k == 1:
        return {"status": 0, "kind": 1, "slot": body.slot, "value_hex": body.command_batch_or_noop.hex()}
    cmds = [body.command] if k in (2, 3, 4) else list(body.command)
    return {"status": 0, "kind": k, "slot": -1 if k in (4, 7) else body.slot,
            "commands": [c.SerializeToString().hex() for c in cmds]}


def voter(g, a):
    return (g << 16 | a) if 0 <= g < 0x8000 and 0 <= a < 0x8000 else -1


def expect_reads(raw, batcher, key_capacity):
    """{status, kind, key, id, voter, slot} of one ClientInbound / ReadBatcherInbound."""
    m = parse("ReadBatcherInbound" if batcher else "ClientInbound", raw)
    if m is None:
        return {"status": -15}
    w = m.WhichOneof("request")
    if w is None:
        return {"status": 0, "kind": 0, "key": -1, "id": 0, "voter": 0, "slot": 0}
    k = (BATCHER_MEMBERS if batcher else CLIENT_MEMBERS).index(w) + 1
    if k != 4:
        return {"status": 0, "kind": k, "key": -1, "id": 0, "voter": 0, "slot": 0}
    r = getattr(m, w)
    if batcher:
        return {"status": 0, "kind": 4, "key": r.read_batcher_id % key_capacity, "id": r.read_batcher_id,
                "voter": voter(0, r.acceptor_index), "slot": r.slot}
    return {"status": 0, "kind": 4, "key": r.command_id.client_pseudonym, "id": r.command_id.client_id,
            "voter": voter(r.group_index, r.acceptor_index), "slot": r.slot}


def max_slot_reply_bytes(request_raw, group, acceptor, max_voted_slot):
    """What Acceptor.scala:222-254 sends for one AcceptorInbound request (b"" for another member, None if the
    request does not parse)."""
    m = parse("AcceptorInbound", request_raw)
    if m is None:
        return None
    w = m.WhichOneof("request")
    if w == "max_slot_request":
        out = cls("ClientInbound")()
        out.max_slot_reply.command_id.CopyFrom(m.max_slot_request.command_id)
        out.max_slot_reply.group_index = group; out.max_slot_reply.acceptor_index = acceptor
        out.max_slot_reply.slot = max_voted_slot
        return out.SerializeToString()
    if w == "batch_max_slot_request":
        out = cls("ReadBatcherInbound")()
        r = out.batch_max_slot_reply
        r.read_batcher_index = m.batch_max_slot_request.read_batcher_index
        r.read_batcher_id = m.batch_max_slot_request.read_batcher_id
        r.acceptor_index = acceptor; r.slot = max_voted_slot
        return out.SerializeToString()
    return b""


def read_request_bytes(batcher, slot, commands):
    """Client.scala:900-911 (ReadRequest) / ReadBatcher.scala:613-617 (ReadRequestBatch) as ReplicaInbound bytes."""
    m = cls("ReplicaInbound")()
    if batcher:
        m.read_request_batch.slot = slot
        for c in commands:
            m.read_request_batch.command.add().CopyFrom(c)
    else:
        m.read_request.slot = slot; m.read_request.command.CopyFrom(commands[0])
    return m.SerializeToString()


def arena_entry(commands):
    """The `command` field(s) of a read request: 12 len Command, repeated."""
    out = b""
    for c in commands:
        s = c.SerializeToString()
        out += bytes([0x12]) + _varint(len(s)) + s
    return out


def _varint(v):
    out = b""
    while v >= 0x80:
        out += bytes([(v & 0x7f) | 0x80]); v >>= 7
    return out + bytes([v])


def field(num, payload):
    """A length-delimited field, hand-built."""
    return _varint(num << 3 | 2) + _varint(len(payload)) + payload


def cases():
    g = np.random.Generator(np.random.PCG64(20261017))
    out = []

    def add(inbound, name, raw, expect, **extra):
        out.append(dict(inbound=inbound, name=name, hex=raw.hex(), expect=expect, **extra))

    KEY_CAP = 1 << 10
    # every member of the four inbounds, slots over the varint boundaries (negative: 10 bytes, -1 included)
    for which in range(1, 8):
        for k in range(4):
            raw = replica_message(g, which).SerializeToString()
            add("replica", f"member {which}", raw, expect_replica(raw))
    for n_cmds in (0, 1, 64, 130):                                  # empty and large read batches
        for which in (5, 6, 7):
            raw = replica_message(g, which, n_cmds).SerializeToString()
            add("replica", f"batch {which} of {n_cmds}", raw, expect_replica(raw))
    for s in EDGE:
        m = replica_message(g, 2); m.read_request.slot = s
        raw = m.SerializeToString()
        add("replica", f"read_request slot {s}", raw, expect_replica(raw))
    for which in range(1, 6):
        for k in range(3):
            raw = client_message(g, which).SerializeToString()
            add("client", f"member {which}", raw, expect_reads(raw, False, KEY_CAP))
    for which in range(1, 5):
        for k in range(3):
            raw = batcher_message(g, which).SerializeToString()
            add("batcher", f"member {which}", raw, expect_reads(raw, True, KEY_CAP))
    for rid in (-1, 0, KEY_CAP - 1, KEY_CAP, -(1 << 31), (1 << 31) - 1):        # floorMod keys, the primer's -1
        m = batcher_message(g, 4); m.batch_max_slot_reply.read_batcher_id = rid
        raw = m.SerializeToString()
        add("batcher", f"read_batcher_id {rid}", raw, expect_reads(raw, True, KEY_CAP))

    # parser robustness: hand-built bytes, with the runtime's verdict
    cmd = command(g, 3).SerializeToString()
    cid = command(g, 0).command_id.SerializeToString()
    rr = field(2, b"\x08\x05" + field(2, cmd))                           # ReplicaInbound{read_request{5, cmd}}
    odd = {
        "empty message": b"",
        "truncated": rr[:-1],
        "overlong varint": field(2, bytes([0x08] + [0x80] * 10 + [0x01]) + field(2, cmd)),
        "unknown fields everywhere": b"\x50\x03" + field(2, b"\x08\x05\x18\x07" + field(2, cmd + b"\x28\x01")
                                                        + b"\x25\x01\x02\x03\x04") + field(9, b"xyz"),
        "fields out of order": field(2, field(2, cmd) + b"\x08\x05"),
        "slot given twice: the last wins": field(2, b"\x08\x05" + field(2, cmd) + b"\x08\x07"),
        "member given twice: merged": field(5, b"\x08\x05" + field(2, cmd)) + field(5, b"\x08\x06" + field(2, cmd)),
        "member given twice, another between": field(5, field(2, cmd)) + field(1, b"\x08\x01" + field(2, b"\x12\x00"))
        + field(5, b"\x08\x09" + field(2, cmd)),
        "oneof: the last member wins": field(1, b"\x08\x01" + field(2, b"\x12\x00")) + rr,
        "oneof: the last member wins, other order": rr + field(1, b"\x08\x01" + field(2, b"\x12\x00")),
        "command_id given twice: merged": field(2, b"\x08\x05" + field(2, field(1, b"\x0a\x01a\x10\x01") + field(1, b"\x18\x02")
                                                                       + b"\x12\x01z")),
        "command_id given twice: missing a field": field(2, b"\x08\x05" + field(2, field(1, b"\x0a\x01a\x10\x01")
                                                                               + field(1, b"\x10\x02") + b"\x12\x01z")),
        "missing slot": field(2, field(2, cmd)),
        "missing command": field(2, b"\x08\x05"),
        "Command missing command": field(4, field(1, field(1, cid))),
        "Command missing command_id": field(4, field(1, b"\x12\x01z")),
        "CommandId missing client_address": field(7, field(1, field(1, b"\x10\x01\x18\x02") + b"\x12\x00")),
        "batch missing slot": field(5, field(2, cmd)),
        "eventual batch, empty": field(7, b""),
        "Chosen missing value": field(1, b"\x08\x01"),
        "Chosen missing slot": field(1, field(2, b"\x12\x00")),
        "wrong wire type for a member": b"\x10\x05" + rr,
        "length past the end": b"\x12\x7f\x08\x05",
    }
    for name, raw in odd.items():
        add("replica", name, raw, expect_replica(raw))
    # the codec's documented deviations: scalapb would merge, the codec refuses (FPX_ERR_WIRE)
    dev = {
        "second command in read_request": field(2, b"\x08\x05" + field(2, cmd) + field(2, cmd)),
        "second command across merged eventual_read_request": field(4, field(1, cmd)) + field(4, field(1, cmd)),
        "group wire type": field(2, b"\x08\x05\x0b\x0c" + field(2, cmd)),
        "second command_batch_or_noop": field(1, b"\x08\x01" + field(2, b"\x12\x00") + field(2, b"\x12\x00")),
    }
    for name, raw in dev.items():
        add("replica", name, raw, {"status": -15}, runtime=expect_replica(raw), deviation=True)
    msr = field(4, field(1, cid) + b"\x10\x02\x18\x01\x20\x07")          # ClientInbound{max_slot_reply}
    codd = {
        "max_slot_reply merged": field(4, field(1, cid) + b"\x10\x02") + field(4, b"\x18\x01\x20\x07"),
        "max_slot_reply missing slot": field(4, field(1, cid) + b"\x10\x02\x18\x01"),
        "max_slot_reply missing command_id": field(4, b"\x10\x02\x18\x01\x20\x07"),
        "max_slot_reply CommandId missing client_id": field(4, field(1, b"\x0a\x00\x10\x01") + b"\x10\x02\x18\x01\x20\x07"),
        "max_slot_reply truncated": msr[:-1],
        "max_slot_reply unknown fields": b"\x38\x01" + field(4, field(1, cid) + b"\x10\x02\x18\x01\x20\x07\x2a\x00"),
    }
    for name, raw in codd.items():
        add("client", name, raw, expect_reads(raw, False, KEY_CAP))
    bodd = {
        "batch_max_slot_reply missing acceptor_index": field(4, b"\x08\x01\x10\x02\x20\x07"),
        "batch_max_slot_reply merged": field(4, b"\x08\x01\x10\x02") + field(4, b"\x18\x01\x20\x07"),
        "batch_max_slot_reply negative slot": field(4, b"\x08\x01\x10\x02\x18\x01\x20" + bytes([0xff] * 9 + [0x01])),
    }
    for name, raw in bodd.items():
        add("batcher", name, raw, expect_reads(raw, True, KEY_CAP))

    # the acceptor's replies: AcceptorInbound requests -> what Acceptor.scala sends
    A = cls("AcceptorInbound")
    for k in range(12):
        m = A()
        if k % 3 == 0:
            m.batch_max_slot_request.read_batcher_index = int(g.choice(EDGE))
            m.batch_max_slot_request.read_batcher_id = int(g.choice(EDGE))
        elif k % 3 == 1:
            m.max_slot_request.command_id.CopyFrom(command(g).command_id)
        else:
            m.phase1a.round = 1; m.phase1a.chosen_watermark = 0
        raw = m.SerializeToString()
        gi, ai, slot = k % 2, k % 3, int(EDGE[k])
        add("acceptor", f"request {k}", raw, {"status": 0, "reply_hex": max_slot_reply_bytes(raw, gi, ai, slot).hex()},
            group=gi, acceptor=ai, max_voted_slot=slot)
    merged = field(3, field(1, b"\x0a\x02ab\x10\x05") + field(1, b"\x18\x09\x0a\x01c"))
    add("acceptor", "max_slot_request CommandId merged", merged,
        {"status": 0, "reply_hex": max_slot_reply_bytes(merged, 1, 2, 3).hex()}, group=1, acceptor=2, max_voted_slot=3)
    bad = field(3, field(1, b"\x0a\x02ab\x10\x05"))
    add("acceptor", "max_slot_request missing client_id", bad, {"status": -15}, group=0, acceptor=0, max_voted_slot=0)
    # completed reads -> the ReadRequest / ReadRequestBatch a Client / ReadBatcher sends
    for batcher in (False, True):
        for k, s in enumerate(EDGE):
            cmds = [command(g) for _ in range((k % 4) if batcher else 1)]
            add("read_request", f"{'batcher' if batcher else 'client'} slot {s}", read_request_bytes(batcher, s, cmds),
                {"status": 0}, batcher=int(batcher), slot=s, arena_hex=arena_entry(cmds).hex())
    return out


def main():
    cs = cases()
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "wire_multipaxos_reads.json")
    json.dump({"generator": "tests/golden/make_wire_reads_golden.py (python protobuf runtime "
                            + __import__("google.protobuf").protobuf.__version__ + ")", "key_capacity": 1 << 10,
               "cases": cs}, open(path, "w"), indent=0)
    print(len(cs), "cases ->", path)


if __name__ == "__main__":
    main()
