"""ctypes binding of the Compartmentalized Mencius wire codec's CPU oracle and of its per-message replica
(tests/wire_mencius_oracle.cc).  TEST INFRASTRUCTURE.

The library is compiled with g++ into a temporary directory named after the source's hash, so the tests also
run from a read-only tree."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "wire_mencius_oracle.cc")

MENCIUS_CHOSEN = np.dtype([("slot_start", "<i4"), ("slot_end", "<i4"), ("value_id", "<i4"), ("reserved", "<i4")])
P2B_RANGE = np.dtype([("dst", "<i4"), ("slot_start", "<i4"), ("slot_end", "<i4"), ("round", "<i4")])
CHOSEN_RANGE = np.dtype([("slot_start", "<i4"), ("slot_end", "<i4")])
NACK = np.dtype([("leader", "<i4"), ("round", "<i4")])
VALUE_NOOP = -(1 << 31)
MAX_RANGE_BATCH = 65535
CHOSEN_KIND, CHOSEN_NOOP_RANGE_KIND = 1, 2      # ReplicaInbound members (Mencius.proto:363-371)

_lib = None


def build():
    src = open(_SRC, "rb").read()
    d = os.path.join(tempfile.gettempdir(), f"fpx_wire_mencius_oracle_{os.getuid()}_{hashlib.sha1(src).hexdigest()[:16]}")
    so = os.path.join(d, "libwire_mencius_oracle.so")
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
        vp, i32, i64, i64p = C.c_void_p, C.c_int, C.c_int64, C.POINTER(C.c_int64)
        L.fpo_wire_decode_mencius_replica.argtypes = [vp, vp, i32, i32, vp, vp, vp, i64p]
        L.fpo_wire_decode_mencius_replica.restype = i32
        L.fpo_wire_encode_mencius.argtypes = [i32, vp, i32, i32, vp, vp]
        L.fpo_wire_encode_mencius.restype = i64
        L.fpo_mencius_split.argtypes = [vp, i32, i32, i64]
        L.fpo_mencius_split.restype = i32
        L.fpo_mencius_apply.argtypes = [vp, i32, i32, i64, i64, vp, i64p]
        L.fpo_mencius_apply.restype = i32
        _lib = L
    return _lib


def pack(msgs):
    """Messages back to back + offsets[n+1] (the codec's batch layout)."""
    offs = np.zeros(len(msgs) + 1, dtype=np.int32)
    offs[1:] = np.cumsum([len(m) for m in msgs])
    return np.frombuffer(b"".join(msgs) + b"\0" * 16, dtype=np.uint8).copy(), offs


def decode(buf, offs, value_id_base=0):
    """ReplicaInbound batch -> (status, err_index, kind[n], recs[n], values[n, 2])"""
    buf = np.ascontiguousarray(buf, dtype=np.uint8)
    offs = np.ascontiguousarray(offs, dtype=np.int32)
    n = len(offs) - 1
    pad = np.zeros(max(len(buf), 1), dtype=np.uint8); pad[:len(buf)] = buf
    kind = np.zeros(max(n, 1), dtype=np.int32)
    recs = np.zeros(max(n, 1), dtype=MENCIUS_CHOSEN)
    values = np.zeros((max(n, 1), 2), dtype=np.int32)
    err = C.c_int64(-1)
    st = lib().fpo_wire_decode_mencius_replica(pad.ctypes.data, offs.ctypes.data, n, value_id_base, kind.ctypes.data,
                                               recs.ctypes.data, values.ctypes.data, C.byref(err))
    return st, err.value, kind[:n], recs[:n], values[:n]


_KINDS = {"phase2b_range": (0, P2B_RANGE), "chosen_range": (1, CHOSEN_RANGE), "nack": (2, NACK)}


def encode(what, recs, agroups=1):
    """what: phase2b_range / chosen_range / nack -> (bytes, offsets[n+1])"""
    k, dt = _KINDS[what]
    recs = np.ascontiguousarray(recs, dtype=dt)
    n = len(recs)
    offs = np.zeros(n + 1, dtype=np.int32)
    total = lib().fpo_wire_encode_mencius(k, recs.ctypes.data, n, agroups, None, offs.ctypes.data)
    out = np.zeros(max(total, 1), dtype=np.uint8)
    lib().fpo_wire_encode_mencius(k, recs.ctypes.data, n, agroups, out.ctypes.data, offs.ctypes.data)
    return out[:total], offs


def split_messages(out, offs):
    return [bytes(out[offs[i]: offs[i + 1]]) for i in range(len(offs) - 1)]


class Replica:
    """The Mencius replica's log, one message at a time (Replica.handleChosen / handleChosenNoopRange)."""

    def __init__(self, lg, capacity):
        self.lg, self.cap, self.retired = lg, capacity, 0
        self.log = np.full(capacity, -1, dtype=np.int32)

    def _bound(self, limit):
        """The slot bound of a call: the engine's live bound (base + slot_capacity) of a log that slides, so that
        one oracle log can cover a log many times the engine's capacity; the whole log by default."""
        if limit is None:
            return self.cap
        assert 0 <= limit <= self.cap, (limit, self.cap)
        return limit

    def split(self, recs, limit=None):
        recs = np.ascontiguousarray(recs, dtype=MENCIUS_CHOSEN)
        return lib().fpo_mencius_split(recs.ctypes.data, len(recs), self.lg, self._bound(limit))

    def apply(self, recs, limit=None):
        """-> (status, err_index).  A record past `limit` is FPX_ERR_SLOT_RANGE, as past the engine's live bound."""
        recs = np.ascontiguousarray(recs, dtype=MENCIUS_CHOSEN)
        err = C.c_int64(-1)
        st = lib().fpo_mencius_apply(recs.ctypes.data, len(recs), self.lg, self._bound(limit), self.retired,
                                     self.log.ctypes.data, C.byref(err))
        return st, err.value

    def retire_below(self, slot):
        self.retired = max(self.retired, slot)

    def watermark(self):
        holes = np.nonzero(self.log[self.retired:] == -1)[0]
        return int(self.retired + holes[0]) if len(holes) else self.cap
