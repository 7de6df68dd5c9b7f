"""ctypes binding of the MultiPaxos replica / read-path wire codec's CPU oracle (tests/wire_reads_oracle.cc).
TEST INFRASTRUCTURE.

The library is compiled with g++ into a temporary directory named after the source's hash, so the tests also
run from a read-only tree."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "wire_reads_oracle.cc")

WIRE_REC = np.dtype([("a", "<i4"), ("b", "<i4"), ("c", "<i4"), ("d", "<i4")])
CHOSEN = np.dtype([("slot", "<i4"), ("value_id", "<i4")])
READ_REQUEST = np.dtype([("slot", "<i4"), ("handle", "<i4")])
MAX_SLOT_REPLY = np.dtype([("key", "<i4"), ("id", "<i4"), ("voter", "<i4"), ("slot", "<i4")])
READ_SLOT = np.dtype([("key", "<i4"), ("id", "<i4"), ("slot", "<i4"), ("reserved", "<i4")])
# ReplicaInbound members (MultiPaxos.proto:563-576)
CHOSEN_KIND, READ_REQUEST_KIND, SEQUENTIAL, EVENTUAL, READ_BATCH, SEQUENTIAL_BATCH, EVENTUAL_BATCH = range(1, 8)

_lib = None


def build():
    src = open(_SRC, "rb").read()
    d = os.path.join(tempfile.gettempdir(), f"fpx_wire_reads_oracle_{os.getuid()}_{hashlib.sha1(src).hexdigest()[:16]}")
    so = os.path.join(d, "libwire_reads_oracle.so")
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
        L.fpo_wire_decode_replica.argtypes = [vp, vp, i32, i32, i32, i32, vp, vp, vp, vp, vp, vp, i64p]
        L.fpo_wire_decode_replica.restype = i32
        L.fpo_reads_wire_decode.argtypes = [vp, vp, i32, i32, i32, vp, vp, vp, i64p]
        L.fpo_reads_wire_decode.restype = i32
        L.fpo_wire_encode_max_slot_replies.argtypes = [vp, i32, vp, vp, i32, i32, i32, vp, vp, i64p]
        L.fpo_wire_encode_max_slot_replies.restype = C.c_int64
        L.fpo_reads_wire_encode_read_requests.argtypes = [vp, i32, i32, vp, vp, i32, vp, vp, i64p]
        L.fpo_reads_wire_encode_read_requests.restype = C.c_int64
        _lib = L
    return _lib


def pack(msgs):
    """Messages back to back + offsets[n+1] (the codec's batch layout)."""
    offs = np.zeros(len(msgs) + 1, dtype=np.int32)
    offs[1:] = np.cumsum([len(m) for m in msgs])
    return np.frombuffer(b"".join(msgs) + b"\0" * 16, dtype=np.uint8).copy(), offs


def _pad(buf):
    buf = np.ascontiguousarray(buf, dtype=np.uint8)
    pad = np.zeros(max(len(buf), 1), dtype=np.uint8)
    pad[:len(buf)] = buf
    return pad


def decode_replica(buf, offs, value_id_base=0, handle_base=0, reads_capacity=None):
    """-> (status, err_index, kind[n], chosen, chosen_values[k, 2], reads, read_commands[k, 2], split)"""
    pad = _pad(buf)
    offs = np.ascontiguousarray(offs, dtype=np.int32)
    n = len(offs) - 1
    cap = int(offs[-1] - offs[0]) // 12 + 1 if reads_capacity is None else reads_capacity   # Engine's default
    kind = np.zeros(max(n, 1), dtype=np.int32)
    chosen = np.zeros(max(n, 1), dtype=CHOSEN)
    cvals = np.zeros((max(n, 1), 2), dtype=np.int32)
    room = max(cap, 1)                  # the oracle writes no record past the capacity, as the codec
    reads = np.zeros(room, dtype=READ_REQUEST)
    rcmds = np.zeros((room, 2), dtype=np.int32)
    counts = np.zeros(3, dtype=np.int32)
    err = C.c_int64(-1)
    st = lib().fpo_wire_decode_replica(pad.ctypes.data, offs.ctypes.data, n, value_id_base, handle_base, cap,
                                       kind.ctypes.data, chosen.ctypes.data, cvals.ctypes.data, reads.ctypes.data,
                                       rcmds.ctypes.data, counts.ctypes.data, C.byref(err))
    nc, nr, split = (int(x) for x in counts)
    return st, err.value, kind[:n], chosen[:nc], cvals[:nc], reads[:nr], rcmds[:nr], split


def decode_reads(buf, offs, batcher, key_capacity):
    """-> (status, err_index, kind[n], MAX_SLOT_REPLY[n], spans[n, 2])"""
    pad = _pad(buf)
    offs = np.ascontiguousarray(offs, dtype=np.int32)
    n = len(offs) - 1
    kind = np.zeros(max(n, 1), dtype=np.int32)
    out = np.zeros(max(n, 1), dtype=MAX_SLOT_REPLY)
    spans = np.zeros((max(n, 1), 2), dtype=np.int32)
    err = C.c_int64(-1)
    st = lib().fpo_reads_wire_decode(pad.ctypes.data, offs.ctypes.data, n, int(batcher), key_capacity, kind.ctypes.data,
                                     out.ctypes.data, spans.ctypes.data, C.byref(err))
    return st, err.value, kind[:n], out[:n], spans[:n]


def _encode(fn, args, n):
    offs = np.zeros(n + 1, dtype=np.int32)
    err = C.c_int64(-1)
    total = fn(*args[0], None, offs.ctypes.data, C.byref(err))
    if total < 0:
        return int(total), err.value, np.zeros(0, dtype=np.uint8), offs
    out = np.zeros(max(total, 1), dtype=np.uint8)
    fn(*args[0], out.ctypes.data, offs.ctypes.data, C.byref(err))
    return 0, -1, out[:total], offs


def encode_max_slot_replies(buf, kind, recs, groups, per_group):
    """-> (status, err_index, bytes, offsets[n+1])"""
    pad = _pad(buf)
    kind = np.ascontiguousarray(kind, dtype=np.int32)
    recs = np.ascontiguousarray(recs, dtype=WIRE_REC)
    return _encode(lib().fpo_wire_encode_max_slot_replies,
                   [(pad.ctypes.data, len(buf), kind.ctypes.data, recs.ctypes.data, len(recs), groups, per_group)],
                   len(recs))


def encode_read_requests(recs, batcher, arena, value_offsets):
    """-> (status, err_index, bytes, offsets[n+1])"""
    recs = np.ascontiguousarray(recs, dtype=READ_SLOT)
    arena = _pad(arena)
    value_offsets = np.ascontiguousarray(value_offsets, dtype=np.int32)
    return _encode(lib().fpo_reads_wire_encode_read_requests,
                   [(recs.ctypes.data, len(recs), int(batcher), arena.ctypes.data, value_offsets.ctypes.data,
                     len(value_offsets) - 1)], len(recs))


def split(out, offs):
    return [bytes(out[offs[i]: offs[i + 1]]) for i in range(len(offs) - 1)]


def _varint(v):
    out = b""
    while v >= 0x80:
        out += bytes([(v & 0x7f) | 0x80]); v >>= 7
    return out + bytes([v])


def padded(msg, size):
    """msg with an unknown top-level bytes field (9) appended so that it is exactly `size` bytes."""
    need = size - len(msg)
    for p in range(need, -1, -1):
        if 1 + len(_varint(p)) + p == need:
            return msg + b"\x4a" + _varint(p) + bytes(p)
    raise ValueError(size)


def overlapping_batch(big):
    """Four ReplicaInbound messages whose offsets are not monotone: [0, R0 C R1), [end of R1, 100) (refused),
    [C), [R1 T).  Message 0 is a valid read that spans messages 2 and 3, message 2 a Chosen and message 3 a read,
    so split falls inside the tile.  big: R1 is 29800 bytes (the tile's span exceeds the shared-memory stage), else
    200."""
    cmd = bytes.fromhex("0a0a0a0461626364100118021203787978")
    read = b"\x12" + _varint(4 + len(cmd)) + b"\x08\x05\x12" + bytes([len(cmd)]) + cmd
    chosen = bytes.fromhex("0a06" "0807" "12021200")
    s0, s1 = (100, 29800) if big else (40, 200)
    r0, c, r1 = padded(read, s0), padded(chosen, s0), padded(read, s1)
    t = padded(b"", 10)
    buf = np.frombuffer(r0 + c + r1 + t + bytes(16), np.uint8).copy()
    e1 = 2 * s0 + s1
    return buf, np.array([0, e1, s0, 2 * s0, e1 + 10], np.int32)
