"""ctypes binding of the read path's CPU oracle (tests/reads_oracle.cc).  TEST INFRASTRUCTURE.

The library is compiled with g++ into a temporary directory named after the source's hash, so the tests also
run from a read-only tree."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reads_oracle.cc")

READ_OPEN = np.dtype([("key", "<i4"), ("id", "<i4")])
MAX_SLOT_REPLY = np.dtype([("key", "<i4"), ("id", "<i4"), ("voter", "<i4"), ("slot", "<i4")])
READ_SLOT = np.dtype([("key", "<i4"), ("id", "<i4"), ("slot", "<i4"), ("reserved", "<i4")])
READ_REQUEST = np.dtype([("slot", "<i4"), ("handle", "<i4")])
READ_REPLY = np.dtype([("handle", "<i4"), ("reply_slot", "<i4"), ("after_slot", "<i4"), ("reserved", "<i4")])

_lib = None


def build():
    src = open(_SRC, "rb").read()
    d = os.path.join(tempfile.gettempdir(), f"fpx_reads_oracle_{os.getuid()}_{hashlib.sha1(src).hexdigest()[:16]}")
    so = os.path.join(d, "libreads_oracle.so")
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
        vp, i32, ip, i64p = C.c_void_p, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int64)
        L.fpo_rt_new.argtypes = [i32, i32, i32, i32, i32]; L.fpo_rt_new.restype = vp
        L.fpo_rt_free.argtypes = [vp]
        L.fpo_rt_open.argtypes = [vp, vp, i32]
        L.fpo_rt_replies.argtypes = [vp, vp, i32, vp, ip, i64p]; L.fpo_rt_replies.restype = i32
        L.fpo_dr_new.argtypes = [i32]; L.fpo_dr_new.restype = vp
        L.fpo_dr_free.argtypes = [vp]
        L.fpo_dr_request.argtypes = [vp, vp, i32, vp, ip, i64p]; L.fpo_dr_request.restype = i32
        L.fpo_dr_advance.argtypes = [vp, i32, vp, ip]; L.fpo_dr_advance.restype = i32
        L.fpo_dr_pending.argtypes = [vp]; L.fpo_dr_pending.restype = i32
        _lib = L
    return _lib


class ReadTally:
    """Client (kind 0) / ReadBatcher (kind 1) MaxSlotReply tally; same call shapes as frankenpaxos_b200.Reads."""

    def __init__(self, kind, f, groups, per_group, flexible=False):
        self.h = lib().fpo_rt_new(kind, f, groups, per_group, int(bool(flexible)))

    def __del__(self):
        try:
            lib().fpo_rt_free(self.h)
        except Exception:
            pass

    def open(self, keys, ids):
        recs = np.zeros(len(keys), READ_OPEN)
        recs["key"], recs["id"] = keys, ids
        lib().fpo_rt_open(self.h, recs.ctypes.data, len(recs))

    def max_slot_replies(self, recs):
        """-> (status, err_index, READ_SLOT records)"""
        recs = np.ascontiguousarray(recs, dtype=MAX_SLOT_REPLY)
        out = np.zeros(max(len(recs), 1), READ_SLOT)
        n, err = C.c_int(0), C.c_int64(-1)
        st = lib().fpo_rt_replies(self.h, recs.ctypes.data, len(recs), out.ctypes.data, C.byref(n), C.byref(err))
        return st, err.value, out[:n.value].copy()


class DeferredReads:
    """Replica's deferred reads with a pending capacity; same call shapes as frankenpaxos_b200.Reads."""

    def __init__(self, capacity):
        self.h = lib().fpo_dr_new(capacity)

    def __del__(self):
        try:
            lib().fpo_dr_free(self.h)
        except Exception:
            pass

    def replica(self, recs):
        """-> (status, err_index, READ_REPLY records answered now)"""
        recs = np.ascontiguousarray(recs, dtype=READ_REQUEST)
        out = np.zeros(max(len(recs), 1), READ_REPLY)
        n, err = C.c_int(0), C.c_int64(-1)
        st = lib().fpo_dr_request(self.h, recs.ctypes.data, len(recs), out.ctypes.data, C.byref(n), C.byref(err))
        return st, err.value, out[:n.value].copy()

    def advance(self, w):
        """-> (status, READ_REPLY records released)"""
        out = np.zeros(max(lib().fpo_dr_pending(self.h), 1), READ_REPLY)
        n = C.c_int(0)
        st = lib().fpo_dr_advance(self.h, w, out.ctypes.data, C.byref(n))
        return st, out[:n.value].copy()

    @property
    def pending(self):
        return lib().fpo_dr_pending(self.h)
