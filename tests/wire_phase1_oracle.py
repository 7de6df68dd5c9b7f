"""ctypes binding of the leader's Phase-1 wire path CPU oracle (tests/wire_phase1_oracle.cc).  TEST INFRASTRUCTURE.

The library is compiled with g++ into a temporary directory named after the source's hash (the oracle it includes
too), so the tests also run from a read-only tree."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "wire_phase1_oracle.cc")
_DEP = os.path.join(_HERE, "..", "oracle", "fpx_oracle.cc")

P2A = np.dtype([("slot", "<i4"), ("round", "<i4"), ("value_id", "<i4"), ("dst", "<i4")])
VALUE_NOOP = -(1 << 31)
NOOP_BYTES = b"\x12\x00"

_lib = None


def build():
    h = hashlib.sha1(open(_SRC, "rb").read() + open(_DEP, "rb").read()).hexdigest()[:16]
    d = os.path.join(tempfile.gettempdir(), f"fpx_wire_phase1_oracle_{os.getuid()}_{h}")
    so = os.path.join(d, "libwire_phase1_oracle.so")
    if not os.path.exists(so):
        os.makedirs(d, exist_ok=True)
        tmp = f"{so}.{os.getpid()}"
        subprocess.check_call([os.environ.get("CXX", "g++"), "-O2", "-std=c++17", "-fPIC", "-Wall", "-Wextra", "-shared",
                               "-pthread", "-o", tmp, _SRC])
        os.replace(tmp, so)   # atomic: concurrent test processes never load a half-written library
    return so


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(build())
        vp, i32, i64p = C.c_void_p, C.c_int, C.POINTER(C.c_int64)
        L.fpo_leader_phase1b.argtypes = [i32] * 6 + [vp, vp, i32, i32, vp, vp, i32, vp, i64p]
        L.fpo_leader_phase1b.restype = i32
        L.fpo_wire_encode_phase2a.argtypes = [vp, i32, vp, i32, vp, i32, i32, vp, vp, i64p]
        L.fpo_wire_encode_phase2a.restype = C.c_int64
        L.fpo_encode_phase1b.argtypes = [i32, i32, i32, vp, vp, vp, i32, vp, vp, vp]
        L.fpo_encode_phase1b.restype = C.c_int64
        L.fpo_mp_new.argtypes = [i32] * 6
        L.fpo_mp_new.restype = vp
        L.fpo_mp_free.argtypes = [vp]
        L.fpo_mp_acceptor_phase2a.argtypes = [vp, vp, i32, vp, vp, vp, vp, i64p]
        L.fpo_mp_acceptor_phase2a.restype = i32
        L.fpo_acceptor_phase1a_wire.argtypes = [vp, i32, vp, i32, vp, vp, i32, vp, vp, i32, vp, vp, i64p]
        L.fpo_acceptor_phase1a_wire.restype = C.c_int64
        L.fpo_p1_acceptor_round.argtypes = [vp, i32, i32]
        L.fpo_p1_acceptor_round.restype = i32
        _lib = L
    return _lib


def pack(msgs):
    """Messages back to back + offsets[n+1] (the codec's batch layout)."""
    offs = np.zeros(len(msgs) + 1, dtype=np.int32)
    offs[1:] = np.cumsum([len(m) for m in msgs])
    return np.frombuffer(b"".join(msgs) + b"\0" * 16, dtype=np.uint8).copy(), offs


def leader_phase1b(f, groups, per_group, flexible, round_, chosen_watermark, buf, offs, value_id_base=0, cap=None):
    """-> (status, err_index, complete, max_slot, P2A records, spans[k, 2])"""
    buf = np.ascontiguousarray(buf, dtype=np.uint8)
    offs = np.ascontiguousarray(offs, dtype=np.int32)
    n = len(offs) - 1
    cap = (1 << 20) if cap is None else cap
    out = np.zeros(max(cap, 1), dtype=P2A)
    spans = np.zeros((max(cap, 1), 2), dtype=np.int32)
    res = np.zeros(3, dtype=np.int32)
    err = C.c_int64(-1)
    st = lib().fpo_leader_phase1b(f, groups, per_group, int(flexible), round_, chosen_watermark,
                                  buf.ctypes.data if len(buf) else None, offs.ctypes.data, n, value_id_base,
                                  out.ctypes.data, spans.ctypes.data, cap, res.ctypes.data, C.byref(err))
    k = int(res[2]) if st == 0 else 0
    return st, err.value, int(res[0]), int(res[1]), out[:k].copy(), spans[:k].copy()


def encode_phase2a(recs, buf, spans, value_id_base=0):
    """-> (status, err_index, bytes, offsets[n+1])"""
    recs = np.ascontiguousarray(recs, dtype=P2A)
    buf = np.ascontiguousarray(buf, dtype=np.uint8)
    spans = np.ascontiguousarray(spans, dtype=np.int32).reshape(-1, 2)
    n = len(recs)
    offs = np.zeros(n + 1, dtype=np.int32)
    err = C.c_int64(-1)
    args = (recs.ctypes.data, n, buf.ctypes.data if len(buf) else None, len(buf), spans.ctypes.data, len(spans),
            value_id_base)
    total = lib().fpo_wire_encode_phase2a(*args, None, offs.ctypes.data, C.byref(err))
    if total < 0:
        return int(total), err.value, np.zeros(0, dtype=np.uint8), offs
    out = np.zeros(max(total, 1), dtype=np.uint8)
    lib().fpo_wire_encode_phase2a(*args, out.ctypes.data, offs.ctypes.data, C.byref(err))
    return 0, -1, out[:total], offs


def encode_phase1b(group, acceptor, round_, slots, vote_rounds, value_ids, arena, value_offsets):
    """LeaderInbound{phase1b} bytes, canonical: value_ids index (arena, value_offsets), VALUE_NOOP is the Noop."""
    slots, vote_rounds, value_ids = (np.ascontiguousarray(x, dtype=np.int32) for x in (slots, vote_rounds, value_ids))
    arena = np.ascontiguousarray(arena, dtype=np.uint8)
    value_offsets = np.ascontiguousarray(value_offsets, dtype=np.int32)
    args = (group, acceptor, round_, slots.ctypes.data, vote_rounds.ctypes.data, value_ids.ctypes.data, len(slots),
            arena.ctypes.data if len(arena) else None, value_offsets.ctypes.data)
    total = lib().fpo_encode_phase1b(*args, None)
    out = np.zeros(max(total, 1), dtype=np.uint8)
    lib().fpo_encode_phase1b(*args, out.ctypes.data)
    return bytes(out[:total])


def split(out, offs):
    return [bytes(out[offs[i]: offs[i + 1]]) for i in range(len(offs) - 1)]


WIRE_REC = np.dtype([("a", "<i4"), ("b", "<i4"), ("c", "<i4"), ("d", "<i4")])
P2B = np.dtype([("group", "<i4"), ("acceptor", "<i4"), ("slot", "<i4"), ("round", "<i4")])
NACK = np.dtype([("leader", "<i4"), ("round", "<i4")])


class Acceptors:
    """The oracle's MultiPaxos acceptors (oracle/fpx_oracle.cc) for the acceptor side of Phase 1."""

    def __init__(self, f, groups, per_group, flexible=False):
        self.groups, self.per_group = groups, per_group
        self.p = lib().fpo_mp_new(f, groups, per_group, int(flexible), f + 1, f + 1)

    def __del__(self):
        lib().fpo_mp_free(self.p)

    def phase2a(self, p2a):
        p2a = np.ascontiguousarray(p2a, dtype=P2A)
        n = len(p2a)
        a, b = np.zeros(max(n, 1), P2B), np.zeros(max(n, 1), NACK)
        n1, n2, err = C.c_int(0), C.c_int(0), C.c_int64(-1)
        st = lib().fpo_mp_acceptor_phase2a(self.p, p2a.ctypes.data, n, a.ctypes.data, C.byref(n1), b.ctypes.data,
                                           C.byref(n2), C.byref(err))
        assert st == 0

    def phase1a_wire(self, first_held, buf, kind, recs, arena, value_offsets):
        """-> (status, err_index, bytes, offsets[n+1]); applied only when the status is 0"""
        buf = np.ascontiguousarray(buf, dtype=np.uint8)
        kind = np.ascontiguousarray(kind, dtype=np.int32)
        recs = np.ascontiguousarray(recs, dtype=WIRE_REC)
        arena = np.ascontiguousarray(arena, dtype=np.uint8)
        value_offsets = np.ascontiguousarray(value_offsets, dtype=np.int32)
        n = len(recs)
        offs = np.zeros(n + 1, dtype=np.int32)
        err = C.c_int64(-1)
        args = (self.p, first_held, buf.ctypes.data if len(buf) else None, len(buf), kind.ctypes.data, recs.ctypes.data,
                n, arena.ctypes.data if len(arena) else None, value_offsets.ctypes.data, len(value_offsets) - 1)
        total = lib().fpo_acceptor_phase1a_wire(*args, None, offs.ctypes.data, C.byref(err))
        if total < 0:
            return int(total), err.value, np.zeros(0, np.uint8), offs
        out = np.zeros(max(total, 1), dtype=np.uint8)
        lib().fpo_acceptor_phase1a_wire(*args, out.ctypes.data, offs.ctypes.data, C.byref(err))
        return 0, -1, out[:total], offs

    def round(self, g, a):
        return lib().fpo_p1_acceptor_round(self.p, g, a)
