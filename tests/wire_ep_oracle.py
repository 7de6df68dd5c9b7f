"""ctypes binding of the EPaxos wire codec's CPU oracle (tests/wire_ep_oracle.cc).  TEST INFRASTRUCTURE.

The library is compiled with g++ into a temporary directory named after the source's hash, so the tests also
run from a read-only tree."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "wire_ep_oracle.cc")

VALUE_NOOP = -(1 << 31)
OK, INVALID_ARG, UNSUPPORTED, WIRE = 0, -1, -11, -15
# ReplicaInbound members (EPaxos.proto:220-235)
CLIENT_REQUEST, PRE_ACCEPT, PRE_ACCEPT_OK, ACCEPT, ACCEPT_OK, COMMIT, PREPARE, PREPARE_OK, NACK = range(1, 10)
# handler calls (include/fpx.h FPX_EP_CALL_*)
CALL_LEAD, CALL_PREACCEPT, CALL_ACCEPT, CALL_PREACCEPTOK, CALL_ACCEPTOK, CALL_COMMIT, CALL_NACK, CALL_PREPARE_PHASE, \
    CALL_PREPARE, CALL_PREPAREOK, CALL_SLOW_PATH_TIMER = range(11)
# decoded row columns
IREP, INUM, BORD, BREP, REPLICA, VBORD, VBREP, STATUS, VALUE, SEQ, FLAGS, OVERFLOW, DEPS = range(13)


def pack_width(call, n):
    return {CALL_PREACCEPT: 6 + 2 * n, CALL_ACCEPT: 6 + n, CALL_PREACCEPTOK: 6 + n, CALL_ACCEPTOK: 6,
            CALL_COMMIT: 4 + n, CALL_NACK: 4, CALL_PREPARE: 4, CALL_PREPAREOK: 9}[call]


_lib = None


def build():
    src = open(_SRC, "rb").read()
    d = os.path.join(tempfile.gettempdir(), f"fpx_wire_ep_oracle_{os.getuid()}_{hashlib.sha1(src).hexdigest()[:16]}")
    so = os.path.join(d, "libwire_ep_oracle.so")
    if not os.path.exists(so):
        os.makedirs(d, exist_ok=True)
        tmp = f"{so}.{os.getpid()}"
        subprocess.check_call([os.environ.get("CXX", "g++"), "-O2", "-std=c++17", "-fPIC", "-Wall", "-Wextra", "-shared",
                               "-o", tmp, _SRC])
        os.replace(tmp, so)   # atomic: concurrent test processes never load a half-written library
    return so


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(build())
        vp, i32, i64p = C.c_void_p, C.c_int, C.POINTER(C.c_int64)
        L.fpo_wire_decode_ep.argtypes = [vp, vp, i32, i32, C.c_int32, vp, vp, vp, i64p]
        L.fpo_wire_decode_ep.restype = i32
        L.fpo_wire_pack_ep.argtypes = [i32, vp, vp, i32, i32, i32, vp, vp, i64p]
        L.fpo_wire_pack_ep.restype = i32
        _lib = L
    return _lib


def pack(msgs):
    """Messages back to back + offsets[n+1] (the codec's batch layout)."""
    offs = np.zeros(len(msgs) + 1, dtype=np.int32)
    offs[1:] = np.cumsum([len(m) for m in msgs])
    return np.frombuffer(b"".join(msgs) + b"\0" * 16, dtype=np.uint8).copy(), offs


def decode(buf, offs, n, value_id_base=0):
    """-> (status, err_index, kind[m], rows[m, 12 + n], values[m, 2]) for m messages of an n-replica system"""
    buf = np.ascontiguousarray(buf, dtype=np.uint8)
    offs = np.ascontiguousarray(offs, dtype=np.int32)
    m = len(offs) - 1
    pad = np.zeros(max(len(buf), 1), dtype=np.uint8); pad[:len(buf)] = buf
    kind = np.zeros(max(m, 1), dtype=np.int32)
    rows = np.zeros((max(m, 1), 12 + n), dtype=np.int32)
    values = np.zeros((max(m, 1), 2), dtype=np.int32)
    err = C.c_int64(-1)
    st = lib().fpo_wire_decode_ep(pad.ctypes.data, offs.ctypes.data, m, n, value_id_base, kind.ctypes.data,
                                  rows.ctypes.data, values.ctypes.data, C.byref(err))
    return st, err.value, kind[:m], rows[:m], values[:m]


def pack_rows(call, kind, rows, first, count, n, local_deps=None):
    """-> (status, err_index, out[count, pack_width(call, n)])"""
    kind = np.ascontiguousarray(kind, dtype=np.int32)
    rows = np.ascontiguousarray(rows, dtype=np.int32).reshape(-1, 12 + n)
    w = pack_width(call, n) if call in (1, 2, 3, 4, 5, 6, 8, 9) else 1
    out = np.zeros((max(count, 1), w), dtype=np.int32)
    ld = None if local_deps is None else np.ascontiguousarray(local_deps, dtype=np.int32)
    err = C.c_int64(-1)
    st = lib().fpo_wire_pack_ep(call, kind.ctypes.data, rows.ctypes.data, first, count, n,
                                None if ld is None else ld.ctypes.data, out.ctypes.data, C.byref(err))
    return st, err.value, out[:count]


# -- random messages and what Google's runtime makes of bytes (tests of the oracle and of the GPU codec)
def golden_module():
    """tests/golden/make_wire_ep_golden.py: the descriptor pool and the expected rows"""
    import importlib.util
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "make_wire_ep_golden.py")
    spec = importlib.util.spec_from_file_location("make_wire_ep_golden", path)
    G = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(G)
    return G


def random_message(G, g, n):
    """a seeded random, initialized ReplicaInbound of any member over n replicas"""
    I, B = G.cls("Instance"), G.cls("Ballot")

    def i32():
        return int(g.choice(G.EDGE)) if g.random() < 0.3 else int(g.integers(-2, 1 << 20))

    inst = lambda: I(replica_index=i32(), instance_number=i32())       # noqa: E731
    bal = lambda: B(ordering=i32(), replica_index=i32())               # noqa: E731
    dep = lambda: G.depset([i32() for _ in range(n)])                  # noqa: E731
    val = lambda: G.value(g, int(g.integers(-1, 40)))                   # noqa: E731
    which = int(g.integers(1, 10))
    RI = G.RI
    if which == 1:
        return RI(client_request=G.cls("ClientRequest")(command=G.command(g, int(g.integers(0, 40)))))
    if which in (2, 4):
        m = G.cls("PreAccept" if which == 2 else "Accept")(instance=inst(), ballot=bal(), command_or_noop=val(),
                                                          sequence_number=i32(), dependencies=dep())
        return RI(pre_accept=m) if which == 2 else RI(accept=m)
    if which == 3:
        return RI(pre_accept_ok=G.cls("PreAcceptOk")(instance=inst(), ballot=bal(), replica_index=i32(),
                                                     sequence_number=i32(), dependencies=dep()))
    if which == 5:
        return RI(accept_ok=G.cls("AcceptOk")(instance=inst(), ballot=bal(), replica_index=i32()))
    if which == 6:
        return RI(commit=G.cls("Commit")(instance=inst(), command_or_noop=val(), sequence_number=i32(),
                                         dependencies=dep()))
    if which == 7:
        return RI(prepare=G.cls("Prepare")(instance=inst(), ballot=bal()))
    if which == 9:
        return RI(nack=G.cls("Nack")(instance=inst(), largest_ballot=bal()))
    st = int(g.integers(0, 3))
    po = G.cls("PrepareOk")(ballot=bal(), instance=inst(), replica_index=i32(), vote_ballot=bal(), status=st)
    if st:
        po.command_or_noop.CopyFrom(val()); po.sequence_number = i32(); po.dependencies.CopyFrom(dep())
    return RI(prepare_ok=po)


def mutate(raw, g):
    """one random byte-level change: flip, delete, insert or truncate"""
    b = bytearray(raw)
    op = int(g.integers(0, 4))
    if not b or op == 2:
        b.insert(int(g.integers(0, len(b) + 1)), int(g.integers(0, 256)))
    elif op == 0:
        b[int(g.integers(0, len(b)))] ^= 1 << int(g.integers(0, 8))
    elif op == 1:
        del b[int(g.integers(0, len(b)))]
    else:
        b = b[:int(g.integers(0, len(b)))]
    return bytes(b)


def _fields(raw):
    """top-level (field, wire type, body) of well-formed bytes"""
    out, p = [], 0
    while p < len(raw):
        t, p = _varint(raw, p)
        f, wt = t >> 3, t & 7
        if wt == 0:
            _, p = _varint(raw, p); out.append((f, wt, b""))
        elif wt == 2:
            ln, p = _varint(raw, p); out.append((f, wt, raw[p:p + ln])); p += ln
        else:
            p += 8 if wt == 1 else 4; out.append((f, wt, b""))
    return out


def _varint(raw, p):
    v, s = 0, 0
    while True:
        c = raw[p]; p += 1
        v |= (c & 0x7f) << s; s += 7
        if not c & 0x80:
            return v, p


VALUE_FIELD = {1: 1, 2: 3, 4: 3, 6: 2, 8: 6}    # the member's CommandOrNoop (ClientRequest: its Command)


def runtime_status(G, raw, n):
    """The codec's status for bytes the runtime parses (include/fpx.h), from the runtime's message:
    (status, message or None)."""
    m = G.RI()
    try:
        m.ParseFromString(raw)
    except Exception:                     # google.protobuf.message.DecodeError
        return WIRE, None
    which = m.WhichOneof("request")
    if which is None:
        return OK, m
    k = G.MEMBERS[which]
    body = getattr(m, which)
    if not m.IsInitialized():
        # a CommandStatus the runtime does not know is kept as an unknown field (proto2 closed enum): scalapb keeps it
        if which == "prepare_ok" and not body.HasField("status"):
            from google.protobuf import unknown_fields
            if any(u.field_number == 5 and u.wire_type == 0 for u in unknown_fields.UnknownFieldSet(body)):
                probe = G.RI(); probe.CopyFrom(m); getattr(probe, which).status = 0
                if probe.IsInitialized():
                    return UNSUPPORTED, m
        return WIRE, m
    # a second command_or_noop in the last run of the member
    run = []
    for f, wt, b in _fields(raw):
        if wt == 2 and 1 <= f <= 9:
            run = run + [b] if f == k else []
    if k in VALUE_FIELD and sum(1 for b in run for f, wt, _ in _fields(b) if f == VALUE_FIELD[k] and wt == 2) > 1:
        return WIRE, m
    if "dependencies" in body.DESCRIPTOR.fields_by_name and body.HasField("dependencies"):
        d = body.dependencies
        if d.numReplicas != n or len(d.int_prefix_set) != n:
            return UNSUPPORTED, m
    return OK, m


def preaccept_messages(G, rows, n):
    """ReplicaInbound{pre_accept} bytes of fpx_epaxos_preaccept rows {rep, num, b_ord, b_rep, value_id, seq,
    local_deps[n], msg_deps[n]}: the message's dependencies are msg_deps, its value a Command whose client_id is
    value_id"""
    m = G.RI()
    b = m.pre_accept
    b.command_or_noop.command.client_address = b"c"; b.command_or_noop.command.client_pseudonym = 0
    b.command_or_noop.command.command = b"x"
    b.dependencies.numReplicas = n
    for _ in range(n):
        b.dependencies.int_prefix_set.add().watermark = 0
    out = []
    for r in rows.tolist():
        b.instance.replica_index, b.instance.instance_number, b.ballot.ordering, b.ballot.replica_index = r[:4]
        b.command_or_noop.command.client_id = r[4]
        b.sequence_number = r[5]
        for k in range(n):
            b.dependencies.int_prefix_set[k].watermark = r[6 + n + k]
        out.append(m.SerializeToString())
    return out


def preacceptok_messages(G, rows, n):
    """ReplicaInbound{pre_accept_ok} bytes of fpx_epaxos_preacceptok rows {rep, num, b_ord, b_rep, from, seq, deps[n]}"""
    m = G.RI()
    b = m.pre_accept_ok
    b.dependencies.numReplicas = n
    for _ in range(n):
        b.dependencies.int_prefix_set.add().watermark = 0
    out = []
    for r in rows.tolist():
        b.instance.replica_index, b.instance.instance_number, b.ballot.ordering, b.ballot.replica_index = r[:4]
        b.replica_index, b.sequence_number = r[4], r[5]
        for k in range(n):
            b.dependencies.int_prefix_set[k].watermark = r[6 + k]
        out.append(m.SerializeToString())
    return out


# -- handler rows <-> the messages the reference sends (Replica.scala), built with Google's runtime
def value_arena(count):
    """value_id v -> a CommandOrNoop{command{client_address = v (4 bytes LE), 0, 0, ""}} of 14 bytes, v < count"""
    v = np.arange(count, dtype=np.uint32)
    a = np.zeros((count, 14), dtype=np.uint8)
    a[:, :4] = [0x0a, 0x0c, 0x0a, 0x04]
    a[:, 4:8] = v.view(np.uint8).reshape(count, 4)
    a[:, 8:] = [0x10, 0x00, 0x18, 0x00, 0x22, 0x00]
    return a.reshape(-1), (np.arange(count + 1) * 14).astype(np.int32)


def _set_value(G, field, v):
    if v == VALUE_NOOP:
        field.noop.SetInParent()
    else:
        field.command.client_address = int(v).to_bytes(4, "little", signed=False)
        field.command.client_pseudonym = 0; field.command.client_id = 0; field.command.command = b""


def _set_deps(G, d, ws):
    d.numReplicas = len(ws)
    for w in ws:
        d.int_prefix_set.add().watermark = int(w)


def inbound_message(G, call, r, n):
    """the ReplicaInbound whose decode + pack gives the input row r of handler call `call`"""
    m = G.RI()
    r = [int(x) for x in r]
    if call in (CALL_PREACCEPT, CALL_ACCEPT):
        b = m.pre_accept if call == CALL_PREACCEPT else m.accept
        b.ballot.ordering, b.ballot.replica_index = r[2], r[3]
        _set_value(G, b.command_or_noop, r[4]); b.sequence_number = r[5]
        _set_deps(G, b.dependencies, r[6 + n:6 + 2 * n] if call == CALL_PREACCEPT else r[6:6 + n])
    elif call == CALL_PREACCEPTOK:
        b = m.pre_accept_ok
        b.ballot.ordering, b.ballot.replica_index = r[2], r[3]
        b.replica_index, b.sequence_number = r[4], r[5]
        _set_deps(G, b.dependencies, r[6:6 + n])
    elif call == CALL_ACCEPTOK:
        b = m.accept_ok
        b.ballot.ordering, b.ballot.replica_index = r[2], r[3]
        b.replica_index = r[4]
    elif call == CALL_COMMIT:
        b = m.commit
        _set_value(G, b.command_or_noop, r[2]); b.sequence_number = r[3]
        _set_deps(G, b.dependencies, r[4:4 + n])
    elif call in (CALL_NACK, CALL_PREPARE):
        b = m.nack if call == CALL_NACK else m.prepare
        bb = b.largest_ballot if call == CALL_NACK else b.ballot
        bb.ordering, bb.replica_index = r[2], r[3]
    elif call == CALL_PREPAREOK:
        b = m.prepare_ok
        b.ballot.ordering, b.ballot.replica_index = r[2], r[3]
        b.replica_index = r[4]
        b.vote_ballot.ordering, b.vote_ballot.replica_index = r[5], r[6]
        b.status = r[7]
        if r[7]:
            _set_value(G, b.command_or_noop, r[8]); b.sequence_number = 0
            _set_deps(G, b.dependencies, [0] * n)
    else:
        raise ValueError(call)
    b.instance.replica_index, b.instance.instance_number = r[0], r[1]
    return m.SerializeToString()


def expected_encode(G, call, in_rows, out_rows, n, me, cmd_value, entries=None):
    """SerializeToString of what the reference sends for each record (include/fpx.h fpx_epaxos_wire_encode);
    cmd_value(rep, num) = the instance's value_id in the replica's cmdLog.  entries: value_id v is the CommandOrNoop
    whose bytes are entries[v] (None: value_arena's values)"""
    def put(field, v):
        if entries is None or v == VALUE_NOOP:
            _set_value(G, field, v)
        else:
            field.SetInParent()
            field.MergeFromString(entries[v])

    out = []
    for i, r in enumerate(np.asarray(in_rows).tolist()):
        o = [] if out_rows is None else [int(x) for x in out_rows[i]]
        m = G.RI()
        inst = (r[0], r[1])

        def commit(v, seq, deps):
            b = m.commit
            put(b.command_or_noop, v); b.sequence_number = seq; _set_deps(G, b.dependencies, deps)
            return b

        b = None
        if call == CALL_LEAD:
            b = m.pre_accept
            b.ballot.ordering, b.ballot.replica_index = r[2], r[3]
            put(b.command_or_noop, r[4]); b.sequence_number = r[5]; _set_deps(G, b.dependencies, r[8:8 + n])
        elif call in (CALL_PREACCEPT, CALL_ACCEPT):
            if o[0] == 1 and call == CALL_PREACCEPT:
                b = m.pre_accept_ok
                b.ballot.ordering, b.ballot.replica_index = o[1], o[2]
                b.replica_index, b.sequence_number = me, o[3]; _set_deps(G, b.dependencies, o[4:4 + n])
            elif o[0] == 1:
                b = m.accept_ok
                b.ballot.ordering, b.ballot.replica_index = o[1], o[2]
                b.replica_index = me
            elif o[0] == 2:
                b = m.nack
                b.largest_ballot.ordering, b.largest_ballot.replica_index = o[1], o[2]
            elif o[0] == 3:
                b = commit(cmd_value(*inst), o[3], o[4:4 + n])
        elif call in (CALL_PREACCEPTOK, CALL_ACCEPTOK, CALL_SLOW_PATH_TIMER):
            if o[0] in (1, 4):
                b = commit(cmd_value(*inst), o[1], o[2:2 + n])
            elif o[0] == 2:
                b = m.accept
                b.ballot.ordering, b.ballot.replica_index = r[2], r[3]
                put(b.command_or_noop, cmd_value(*inst)); b.sequence_number = o[1]
                _set_deps(G, b.dependencies, o[2:2 + n])
        elif call == CALL_PREPARE_PHASE:
            b = m.prepare
            b.ballot.ordering, b.ballot.replica_index = o[0], o[1]
        elif call == CALL_PREPARE:
            if o[0] == 1:
                b = m.prepare_ok
                b.ballot.ordering, b.ballot.replica_index = o[2], o[3]
                b.replica_index = me
                b.vote_ballot.ordering, b.vote_ballot.replica_index = o[4], o[5]
                b.status = o[6]
                if o[6]:
                    put(b.command_or_noop, o[7]); b.sequence_number = o[8]
                    _set_deps(G, b.dependencies, o[9:9 + n])
            elif o[0] == 2:
                b = m.nack
                b.largest_ballot.ordering, b.largest_ballot.replica_index = o[2], o[3]
            elif o[0] == 3:
                b = commit(o[7], o[8], o[9:9 + n])
        if b is None:
            out.append(b"")
            continue
        b.instance.replica_index, b.instance.instance_number = inst
        out.append(m.SerializeToString())
    return out


def split(out, offs):
    return [bytes(out[offs[i]: offs[i + 1]]) for i in range(len(offs) - 1)]
