"""Golden wire vectors for EPaxos: tests/golden/wire_epaxos.json.

Built the way make_wire_vm_golden.py builds the vanilla Mencius vectors: the reference serialises with scalapb over
protobuf-java (every *Serializer is ProtoSerializer, shared/src/main/scala/frankenpaxos/ProtoSerializer.scala:3-11),
neither of which runs here, so the bytes come from an INDEPENDENT implementation of the same published format,
Google's Python protobuf runtime, with the message shapes transcribed from
shared/src/main/scala/frankenpaxos/epaxos/EPaxos.proto and shared/src/main/scala/frankenpaxos/compact/IntPrefixSet.proto.
Each case holds the bytes, what the runtime makes of them (its verdict), and the decoded row the codec must give
(include/fpx.h, fpx_epaxos_wire_decode), computed here from the runtime's message.

    python tests/golden/make_wire_ep_golden.py      # rewrites tests/golden/wire_epaxos.json
"""
import json
import os

import numpy as np
from google.protobuf import descriptor_pb2, descriptor_pool, message_factory

F = descriptor_pb2.FieldDescriptorProto
# int32 values around every varint length boundary, negative ones included (10-byte varints)
EDGE = [0, 1, 127, 128, 255, 300, 16383, 16384, (1 << 21) - 1, 1 << 21, (1 << 28) - 1, 1 << 28, (1 << 31) - 1, -1,
        -(1 << 31)]
EPKG, CPKG = "frankenpaxos.epaxos", "frankenpaxos.compact"
VALUE_NOOP = -(1 << 31)
MEMBERS = {None: 0, "client_request": 1, "pre_accept": 2, "pre_accept_ok": 3, "accept": 4, "accept_ok": 5,
           "commit": 6, "prepare": 7, "prepare_ok": 8, "nack": 9}
OK, UNSUPPORTED, WIRE = 0, -11, -15


def build_pool():
    """IntPrefixSet.proto {IntPrefixSetProto} and EPaxos.proto: Instance :35-41, Ballot :46-52, Noop :55-58, Command
    :61-78, CommandOrNoop :80-88, CommandStatus :91-95, InstancePrefixSetProto :97-103, ClientRequest :106-111,
    PreAccept :113-123, PreAcceptOk :125-135, Accept :137-147, AcceptOk :149-156, Commit :158-166, Prepare
    :178-184, PrepareOk :186-209, Nack :211-217, ReplicaInbound :220-235."""
    REQ, OPT, REP = F.LABEL_REQUIRED, F.LABEL_OPTIONAL, F.LABEL_REPEATED
    I32, BYT, MSG, ENUM = F.TYPE_INT32, F.TYPE_BYTES, F.TYPE_MESSAGE, F.TYPE_ENUM
    pool = descriptor_pool.DescriptorPool()

    cfd = descriptor_pb2.FileDescriptorProto()
    cfd.name = "frankenpaxos/compact/IntPrefixSet.proto"; cfd.package = CPKG; cfd.syntax = "proto2"
    m = cfd.message_type.add(); m.name = "IntPrefixSetProto"
    for (fname, num, label) in (("watermark", 1, REQ), ("value", 2, REP)):
        f = m.field.add(); f.name = fname; f.number = num; f.type = I32; f.label = label
    pool.Add(cfd)

    fdp = descriptor_pb2.FileDescriptorProto()
    fdp.name = "EPaxos.proto"; fdp.package = EPKG; fdp.syntax = "proto2"
    fdp.dependency.append(cfd.name)
    e = fdp.enum_type.add(); e.name = "CommandStatus"
    for name, num in (("NotSeen", 0), ("PreAccepted", 1), ("Accepted", 2)):
        v = e.value.add(); v.name = name; v.number = num

    def msg(name, fields, oneof=None):
        m = fdp.message_type.add(); m.name = name
        if oneof:
            m.oneof_decl.add().name = oneof
        for (fname, num, ftype, label, tname) in fields:
            f = m.field.add(); f.name = fname; f.number = num; f.type = ftype; f.label = label
            if tname:
                f.type_name = tname if tname.startswith(".") else f".{EPKG}.{tname}"
            if oneof:
                f.oneof_index = 0

    inst = ("instance", 1, MSG, REQ, "Instance")
    deps = lambda num, label=REQ: ("dependencies", num, MSG, label, "InstancePrefixSetProto")   # noqa: E731
    msg("Instance", [("replica_index", 1, I32, REQ, None), ("instance_number", 2, I32, REQ, None)])
    msg("Ballot", [("ordering", 1, I32, REQ, None), ("replica_index", 2, I32, REQ, None)])
    msg("Noop", [])
    msg("Command", [("client_address", 1, BYT, REQ, None), ("client_pseudonym", 2, I32, REQ, None),
                    ("client_id", 3, I32, REQ, None), ("command", 4, BYT, REQ, None)])
    msg("CommandOrNoop", [("command", 1, MSG, OPT, "Command"), ("noop", 2, MSG, OPT, "Noop")], "value")
    msg("InstancePrefixSetProto", [("numReplicas", 1, I32, REQ, None),
                                   ("int_prefix_set", 2, MSG, REP, f".{CPKG}.IntPrefixSetProto")])
    msg("ClientRequest", [("command", 1, MSG, REQ, "Command")])
    msg("PreAccept", [inst, ("ballot", 2, MSG, REQ, "Ballot"), ("command_or_noop", 3, MSG, REQ, "CommandOrNoop"),
                      ("sequence_number", 4, I32, REQ, None), deps(5)])
    msg("PreAcceptOk", [inst, ("ballot", 2, MSG, REQ, "Ballot"), ("replica_index", 3, I32, REQ, None),
                        ("sequence_number", 4, I32, REQ, None), deps(5)])
    msg("Accept", [inst, ("ballot", 2, MSG, REQ, "Ballot"), ("command_or_noop", 3, MSG, REQ, "CommandOrNoop"),
                   ("sequence_number", 4, I32, REQ, None), deps(5)])
    msg("AcceptOk", [("instance", 2, MSG, REQ, "Instance"), ("ballot", 3, MSG, REQ, "Ballot"),
                     ("replica_index", 7, I32, REQ, None)])
    msg("Commit", [inst, ("command_or_noop", 2, MSG, REQ, "CommandOrNoop"), ("sequence_number", 3, I32, REQ, None),
                   deps(4)])
    msg("Prepare", [inst, ("ballot", 2, MSG, REQ, "Ballot")])
    msg("PrepareOk", [("ballot", 1, MSG, REQ, "Ballot"), ("instance", 2, MSG, REQ, "Instance"),
                      ("replica_index", 3, I32, REQ, None), ("vote_ballot", 4, MSG, REQ, "Ballot"),
                      ("status", 5, ENUM, REQ, "CommandStatus"), ("command_or_noop", 6, MSG, OPT, "CommandOrNoop"),
                      ("sequence_number", 7, I32, OPT, None), deps(8, OPT)])
    msg("Nack", [inst, ("largest_ballot", 2, MSG, REQ, "Ballot")])
    msg("ReplicaInbound", [(name, num, MSG, OPT, "".join(p.capitalize() for p in name.split("_")))
                           for name, num in MEMBERS.items() if name], "request")
    pool.Add(fdp)
    return pool


POOL = build_pool()


def cls(name, pkg=EPKG):
    return message_factory.GetMessageClass(POOL.FindMessageTypeByName(f"{pkg}.{name}"))


RI = cls("ReplicaInbound")


def command(g, cmd_len):
    c = cls("Command")()
    c.client_address = bytes(g.integers(0, 256, size=6, dtype=np.uint8))
    c.client_pseudonym = int(g.integers(0, 1 << 20))
    c.client_id = int(g.integers(0, 1 << 30))
    c.command = bytes(g.integers(0, 256, size=cmd_len, dtype=np.uint8))
    return c


def value(g, cmd_len):
    """A CommandOrNoop: cmd_len < 0 -> Noop."""
    v = cls("CommandOrNoop")()
    if cmd_len < 0:
        v.noop.SetInParent()
    else:
        v.command.CopyFrom(command(g, cmd_len))
    return v


def depset(watermarks, values=()):
    """InstancePrefixSet.toProto: numReplicas and one IntPrefixSetProto per replica"""
    d = cls("InstancePrefixSetProto")(numReplicas=len(watermarks))
    for k, w in enumerate(watermarks):
        e = d.int_prefix_set.add(); e.watermark = w
        e.value.extend(values[k] if k < len(values) else [])
    return d


def expected_row(m, n, value_id):
    """The decoded row (include/fpx.h) of a parsed, initialized ReplicaInbound m."""
    which = m.WhichOneof("request")
    b = getattr(m, which)
    row = [-1, -1, -1, -1, 0, -1, -1, 0, -1, 0, 0, 0] + [0] * n
    has = lambda f: b.DESCRIPTOR.fields_by_name.get(f) is not None and b.HasField(f)   # noqa: E731
    if has("instance"):
        row[0], row[1] = b.instance.replica_index, b.instance.instance_number
    for f in ("ballot", "largest_ballot"):
        if has(f):
            row[2], row[3] = getattr(b, f).ordering, getattr(b, f).replica_index
    if has("replica_index"):
        row[4] = b.replica_index
    if has("vote_ballot"):
        row[5], row[6] = b.vote_ballot.ordering, b.vote_ballot.replica_index
    if has("status"):
        row[7] = b.status
    if which == "client_request" or has("command_or_noop"):
        noop = which != "client_request" and b.command_or_noop.WhichOneof("value") == "noop"
        row[8] = VALUE_NOOP if noop else value_id
    if has("sequence_number"):
        row[9] = b.sequence_number
    if which == "prepare_ok":
        row[10] = int(has("command_or_noop") and has("sequence_number") and has("dependencies"))
    if has("dependencies"):
        row[11] = sum(len(e.value) for e in b.dependencies.int_prefix_set)
        row[12:] = [e.watermark for e in b.dependencies.int_prefix_set]
    return row


def expected_value(m):
    which = m.WhichOneof("request")
    if which == "client_request":
        return cls("CommandOrNoop")(command=m.client_request.command).SerializeToString().hex()
    b = getattr(m, which)
    if "command_or_noop" in b.DESCRIPTOR.fields_by_name and b.HasField("command_or_noop"):
        return b.command_or_noop.SerializeToString().hex()
    return ""


def cases():
    g = np.random.Generator(np.random.PCG64(20261017))
    out = []
    n = 3
    E = len(EDGE)
    I, B = cls("Instance"), cls("Ballot")

    def add(typ, m, **extra):
        out.append(dict(type=typ, n=n, hex=m.SerializeToString().hex(), kind=MEMBERS[m.WhichOneof("request")],
                        status=OK, row=expected_row(m, n, 1000 + len(out)), value_hex=expected_value(m),
                        value_id_base=1000 + len(out), **extra))

    shapes = [-1, 0, 1, 90, 100, 101, 102, 200, 300]
    for k in range(E):
        a, b, c, d = EDGE[k], EDGE[(k + 3) % E], EDGE[(k + 6) % E], EDGE[(k + 9) % E]
        v = value(g, shapes[k % len(shapes)])
        dep = depset([EDGE[(k + j) % E] for j in range(n)])
        add("pre_accept", RI(pre_accept=cls("PreAccept")(instance=I(replica_index=a, instance_number=b),
                                                          ballot=B(ordering=c, replica_index=d), command_or_noop=v,
                                                          sequence_number=b, dependencies=dep)))
        add("pre_accept_ok", RI(pre_accept_ok=cls("PreAcceptOk")(instance=I(replica_index=b, instance_number=c),
                                                                 ballot=B(ordering=d, replica_index=a), replica_index=c,
                                                                 sequence_number=d, dependencies=dep)))
        add("accept", RI(accept=cls("Accept")(instance=I(replica_index=c, instance_number=d),
                                              ballot=B(ordering=a, replica_index=b), command_or_noop=v,
                                              sequence_number=a, dependencies=dep)))
        add("accept_ok", RI(accept_ok=cls("AcceptOk")(instance=I(replica_index=d, instance_number=a),
                                                      ballot=B(ordering=b, replica_index=c), replica_index=a)))
        add("commit", RI(commit=cls("Commit")(instance=I(replica_index=a, instance_number=c), command_or_noop=v,
                                              sequence_number=c, dependencies=dep)))
        add("prepare", RI(prepare=cls("Prepare")(instance=I(replica_index=b, instance_number=d),
                                                 ballot=B(ordering=a, replica_index=c))))
        add("nack", RI(nack=cls("Nack")(instance=I(replica_index=c, instance_number=a),
                                        largest_ballot=B(ordering=d, replica_index=b))))
        st = k % 3
        po = cls("PrepareOk")(ballot=B(ordering=a, replica_index=b), instance=I(replica_index=c, instance_number=d),
                              replica_index=b, vote_ballot=B(ordering=c, replica_index=a), status=st)
        if st:
            po.command_or_noop.CopyFrom(v); po.sequence_number = a; po.dependencies.CopyFrom(dep)
        add("prepare_ok", RI(prepare_ok=po))
    for cl in shapes[1:]:
        add("client_request", RI(client_request=cls("ClientRequest")(command=command(g, cl))))
    # the null ballot of a NotSeen PrepareOk: 10-byte varints, no triple
    add("prepare_ok.not_seen", RI(prepare_ok=cls("PrepareOk")(
        ballot=B(ordering=4, replica_index=1), instance=I(replica_index=2, instance_number=9), replica_index=0,
        vote_ballot=B(ordering=-1, replica_index=-1), status=0)))
    # a set with overflow values, packed (the runtime's default for none of these: written unpacked)
    pa = RI(pre_accept=cls("PreAccept")(instance=I(replica_index=0, instance_number=5), ballot=B(ordering=0, replica_index=0),
                                        command_or_noop=value(g, 4), sequence_number=3,
                                        dependencies=depset([4, 0, 7], [[6, 9], [], [300]])))
    add("pre_accept.overflow_unpacked", pa)
    body = pa.pre_accept
    packed = bytes.fromhex("0803") + bytes.fromhex("1206" "0804" "12020609") + bytes.fromhex("1202" "0800") \
        + bytes.fromhex("1206" "0807" "1202ac02")
    head = cls("PreAccept")(instance=body.instance, ballot=body.ballot, command_or_noop=body.command_or_noop,
                            sequence_number=3).SerializePartialToString(deterministic=True)
    pre = lambda b: bytes([0x12]) + _varint(len(b)) + b   # noqa: E731
    packed_msg = pre(head + bytes([0x2a]) + _varint(len(packed)) + packed)
    m = RI(); m.ParseFromString(packed_msg)
    out.append(dict(type="pre_accept.overflow_packed", n=n, hex=packed_msg.hex(), kind=2, status=OK,
                    row=expected_row(m, n, 7), value_hex=expected_value(m), value_id_base=7))

    # parser robustness: what the runtime makes of each byte string, and the codec's status
    inst = I(replica_index=1, instance_number=2).SerializeToString()
    bal = B(ordering=3, replica_index=1).SerializeToString()
    nack = RI(nack=cls("Nack")(instance=I(replica_index=1, instance_number=2),
                               largest_ballot=B(ordering=3, replica_index=1))).SerializeToString()
    po_ns = RI(prepare_ok=cls("PrepareOk")(ballot=B(ordering=3, replica_index=1), instance=I(replica_index=1, instance_number=2),
                                           replica_index=0, vote_ballot=B(ordering=-1, replica_index=-1),
                                           status=0)).SerializeToString()
    cm = RI(commit=cls("Commit")(instance=I(replica_index=1, instance_number=2), command_or_noop=value(g, -1),
                                 sequence_number=1, dependencies=depset([1, 2, 3]))).SerializeToString()
    ld = lambda f, b: bytes([f << 3 | 2]) + _varint(len(b)) + b   # noqa: E731
    noop = bytes.fromhex("1200")
    dep3 = depset([1, 2, 3]).SerializeToString()
    odd = {
        # Instance given twice: merged (the second copy's instance_number wins, its replica_index is absent)
        "instance twice (merge)": ld(9, ld(1, inst) + ld(2, bal) + ld(1, bytes.fromhex("1007"))),
        "ballot split over two copies (merge)": ld(9, ld(1, inst) + ld(2, bytes.fromhex("0803")) + ld(2, bytes.fromhex("1001"))),
        "member twice (merge)": ld(9, ld(1, inst)) + ld(9, ld(2, bal)),
        "unknown fields at every level": ld(6, ld(1, inst + bytes.fromhex("1801")) + ld(2, noop + bytes.fromhex("2005"))
                                                + bytes.fromhex("1801") + ld(4, bytes.fromhex("0803") + ld(2, bytes.fromhex("0801" "1d01020304"))
                                                                             + ld(2, bytes.fromhex("0802")) + ld(2, bytes.fromhex("0803") + bytes.fromhex("3000")))
                                                + bytes.fromhex("4d01020304")) + bytes.fromhex("5803" "6a00"),
        "oneof set twice: last member wins": cm + nack,
        "oneof set twice, the other order": nack + cm,
        "missing instance_number": ld(9, ld(1, bytes.fromhex("0801")) + ld(2, bal)),
        "missing ballot field": ld(7, ld(1, inst) + ld(2, bytes.fromhex("0803"))),
        "missing largest_ballot": ld(9, ld(1, inst)),
        "missing watermark": ld(6, ld(1, inst) + ld(2, noop) + bytes.fromhex("1801") + ld(4, bytes.fromhex("0803") + ld(2, b"") + ld(2, bytes.fromhex("0802")) + ld(2, bytes.fromhex("0803")))),
        "missing numReplicas": ld(6, ld(1, inst) + ld(2, noop) + bytes.fromhex("1801") + ld(4, ld(2, bytes.fromhex("0801")) + ld(2, bytes.fromhex("0802")) + ld(2, bytes.fromhex("0803")))),
        "command missing client_id": ld(6, ld(1, inst) + ld(2, ld(1, bytes.fromhex("0a00" "1001" "2200"))) + bytes.fromhex("1801") + ld(4, dep3)),
        "client_request without command": bytes.fromhex("0a00"),
        "truncated": cm[:-1],
        "truncated nested length": ld(9, ld(1, inst) + bytes.fromhex("1205" "0803")),
        "nested length past its parent": ld(9, ld(1, bytes.fromhex("0801" "1002")) + bytes.fromhex("12") + bytes([len(bal) + 3]) + bal),
        "overlong varint": ld(7, ld(1, bytes.fromhex("08" "80808080808080808080" "01" "1002")) + ld(2, bal)),
        "packed value truncated": ld(6, ld(1, inst) + ld(2, noop) + bytes.fromhex("1801")
                                         + ld(4, bytes.fromhex("0803") + ld(2, bytes.fromhex("0801" "120280")) + ld(2, bytes.fromhex("0802")) + ld(2, bytes.fromhex("0803")))),
        "group wire type": ld(7, ld(1, inst) + ld(2, bal) + bytes.fromhex("0b")),
        "numReplicas != n": ld(6, ld(1, inst) + ld(2, noop) + bytes.fromhex("1801") + ld(4, bytes.fromhex("0804") + dep3[2:])),
        "set count != n": ld(6, ld(1, inst) + ld(2, noop) + bytes.fromhex("1801") + ld(4, bytes.fromhex("0803") + depset([1, 2]).SerializeToString()[2:])),
        "dependencies twice": ld(6, ld(1, inst) + ld(2, noop) + bytes.fromhex("1801") + ld(4, dep3) + ld(4, dep3)),
        "command_or_noop twice": ld(6, ld(1, inst) + ld(2, noop) + ld(2, noop) + bytes.fromhex("1801") + ld(4, dep3)),
        "unknown status": ld(8, po_ns[2:].replace(bytes.fromhex("2800"), bytes.fromhex("2805"))),
        "empty message": b"",
    }
    expected = {"numReplicas != n": UNSUPPORTED, "set count != n": UNSUPPORTED, "dependencies twice": UNSUPPORTED,
                "unknown status": UNSUPPORTED, "command_or_noop twice": WIRE}
    for name, raw in odd.items():
        m = RI()
        try:
            m.ParseFromString(raw)
            which = m.WhichOneof("request")
            verdict = {"kind": MEMBERS[which], "initialized": m.IsInitialized()}
        except Exception as e:          # google.protobuf.message.DecodeError
            verdict = {"error": type(e).__name__}
        status = expected.get(name, OK if verdict.get("initialized") else WIRE)
        case = {"type": "robustness", "name": name, "n": n, "hex": raw.hex(), "verdict": verdict, "status": status,
                "value_id_base": 0}
        if status == OK:
            case.update(kind=verdict["kind"], row=expected_row(m, n, 0) if verdict["kind"] else None,
                        value_hex=expected_value(m) if verdict["kind"] else "")
        out.append(case)
    return out


def _varint(v):
    b = bytearray()
    while v >= 0x80:
        b.append((v & 0x7f) | 0x80); v >>= 7
    b.append(v)
    return bytes(b)


def main():
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "wire_epaxos.json")
    cs = cases()
    json.dump({"generator": "tests/golden/make_wire_ep_golden.py (python protobuf runtime "
                            + __import__("google.protobuf").protobuf.__version__ + ")", "cases": cs},
              open(out, "w"), indent=0)
    print(len(cs), "cases ->", out)


if __name__ == "__main__":
    main()
