"""ctypes binding of compartmentalized Mencius' leader-change wire path CPU oracle (tests/wire_mencius_phase1_oracle.cc).
TEST INFRASTRUCTURE.

The library is compiled with g++ into a temporary directory named after the hash of its sources, so the tests also
run from a read-only tree.  The MultiPaxos helpers (pack, split, encode_phase1b, the record dtypes) come from
tests/wire_phase1_oracle.py."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from wire_phase1_oracle import NACK, NOOP_BYTES, P2A, P2B, VALUE_NOOP, WIRE_REC, encode_phase1b, pack, split  # noqa: F401

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "wire_mencius_phase1_oracle.cc")
_DEPS = [os.path.join(_HERE, "wire_phase1_oracle.cc"), os.path.join(_HERE, "..", "oracle", "fpx_oracle.cc")]

P2A_RANGE = np.dtype([("slot_start", "<i4"), ("slot_end", "<i4"), ("round", "<i4"), ("dst", "<i4")])
P2B_RANGE = P2A_RANGE

_lib = None


def build():
    h = hashlib.sha1(b"".join(open(p, "rb").read() for p in [_SRC] + _DEPS)).hexdigest()[:16]
    d = os.path.join(tempfile.gettempdir(), f"fpx_wire_mencius_phase1_oracle_{os.getuid()}_{h}")
    so = os.path.join(d, "libwire_mencius_phase1_oracle.so")
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
        L.fpo_mencius_leader_phase1b.argtypes = [i32] * 8 + [vp, vp, i32, i32, vp, vp, i32, vp, i64p]
        L.fpo_mencius_leader_phase1b.restype = i32
        L.fpo_wire_encode_mencius_phase2a.argtypes = [vp, i32, vp, i32, vp, i32, i32, vp, vp, i64p]
        L.fpo_wire_encode_mencius_phase2a.restype = C.c_int64
        L.fpo_mencius_new.argtypes = [i32] * 6
        L.fpo_mencius_new.restype = vp
        L.fpo_mp_free.argtypes = [vp]
        L.fpo_mp_acceptor_phase2a.argtypes = [vp, vp, i32, vp, vp, vp, vp, i64p]
        L.fpo_mp_acceptor_phase2a.restype = i32
        L.fpo_mp_acceptor_noop_range.argtypes = [vp, vp, i32, i32, vp, vp, vp, vp, i64p]
        L.fpo_mp_acceptor_noop_range.restype = i32
        L.fpo_mencius_acceptor_phase1a_wire.argtypes = [vp, i32, vp, i32, vp, vp, i32, vp, vp, i32, vp, vp, i64p]
        L.fpo_mencius_acceptor_phase1a_wire.restype = C.c_int64
        L.fpo_p1_acceptor_round.argtypes = [vp, i32, i32]
        L.fpo_p1_acceptor_round.restype = i32
        _lib = L
    return _lib


def leader_phase1b(f, lgroups, agroups, per_group, leader_group, round_, chosen_watermark, buf, offs, recover_slot=-1,
                   value_id_base=0, cap=None):
    """-> (status, err_index, complete, max_slot, next_slot, P2A records, spans[k, 2])"""
    buf = np.ascontiguousarray(buf, dtype=np.uint8)
    offs = np.ascontiguousarray(offs, dtype=np.int32)
    n = len(offs) - 1
    cap = (1 << 20) if cap is None else cap
    out = np.zeros(max(cap, 1), dtype=P2A)
    spans = np.zeros((max(cap, 1), 2), dtype=np.int32)
    res = np.zeros(4, dtype=np.int32)
    err = C.c_int64(-1)
    st = lib().fpo_mencius_leader_phase1b(f, lgroups, agroups, per_group, leader_group, round_, chosen_watermark,
                                          recover_slot, buf.ctypes.data if len(buf) else None, offs.ctypes.data, n,
                                          value_id_base, out.ctypes.data, spans.ctypes.data, cap, res.ctypes.data,
                                          C.byref(err))
    k = int(res[2]) if st == 0 else 0
    return st, err.value, int(res[0]), int(res[1]), int(res[3]), out[:k].copy(), spans[:k].copy()


def encode_phase2a(recs, buf, spans, value_id_base=0):
    """-> (status, err_index, bytes, offsets[n+1]) of ProxyLeaderInbound{phase2a = 2}"""
    recs = np.ascontiguousarray(recs, dtype=P2A)
    buf = np.ascontiguousarray(buf, dtype=np.uint8)
    spans = np.ascontiguousarray(spans, dtype=np.int32).reshape(-1, 2)
    n = len(recs)
    offs = np.zeros(n + 1, dtype=np.int32)
    err = C.c_int64(-1)
    args = (recs.ctypes.data, n, buf.ctypes.data if len(buf) else None, len(buf), spans.ctypes.data, len(spans),
            value_id_base)
    total = lib().fpo_wire_encode_mencius_phase2a(*args, None, offs.ctypes.data, C.byref(err))
    if total < 0:
        return int(total), err.value, np.zeros(0, dtype=np.uint8), offs
    out = np.zeros(max(total, 1), dtype=np.uint8)
    lib().fpo_wire_encode_mencius_phase2a(*args, out.ctypes.data, offs.ctypes.data, C.byref(err))
    return 0, -1, out[:total], offs


class Acceptors:
    """The oracle's compartmentalized Mencius acceptors (oracle/fpx_oracle.cc), engine group lg * AG + ag."""

    def __init__(self, f, lgroups, agroups):
        self.lgroups, self.agroups, self.per_group = lgroups, agroups, 2 * f + 1
        self.p = lib().fpo_mencius_new(f, lgroups, agroups, 2 * f + 1, f + 1, f + 1)
        assert self.p

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

    def noop_range(self, recs, capacity):
        recs = np.ascontiguousarray(recs, dtype=P2A_RANGE)
        n = len(recs)
        a, b = np.zeros(max(n, 1), P2B_RANGE), np.zeros(max(n, 1), NACK)
        n1, n2, err = C.c_int(0), C.c_int(0), C.c_int64(-1)
        st = lib().fpo_mp_acceptor_noop_range(self.p, recs.ctypes.data, n, capacity, a.ctypes.data, C.byref(n1),
                                              b.ctypes.data, C.byref(n2), C.byref(err))
        assert st == 0, (st, err.value)

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
        total = lib().fpo_mencius_acceptor_phase1a_wire(*args, None, offs.ctypes.data, C.byref(err))
        if total < 0:
            return int(total), err.value, np.zeros(0, np.uint8), offs
        out = np.zeros(max(total, 1), dtype=np.uint8)
        lib().fpo_mencius_acceptor_phase1a_wire(*args, out.ctypes.data, offs.ctypes.data, C.byref(err))
        return 0, -1, out[:total], offs

    def round(self, g, a):
        return lib().fpo_p1_acceptor_round(self.p, g, a)
