"""ctypes binding of the vanilla Mencius wire codec's CPU oracle (tests/wire_vm_oracle.cc).  TEST INFRASTRUCTURE.

The library is compiled with g++ into a temporary directory named after the source's hash, so the tests also
run from a read-only tree."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "wire_vm_oracle.cc")

WIRE_REC = np.dtype([("a", "<i4"), ("b", "<i4"), ("c", "<i4"), ("d", "<i4")])
P2A = np.dtype([("slot", "<i4"), ("round", "<i4"), ("value_id", "<i4"), ("dst", "<i4")])
P2B = np.dtype([("group", "<i4"), ("acceptor", "<i4"), ("slot", "<i4"), ("round", "<i4")])
CHOSEN = np.dtype([("slot", "<i4"), ("value_id", "<i4")])
VM_SKIP = np.dtype([("server", "<i4"), ("slot_start", "<i4"), ("slot_stop", "<i4"), ("own", "<i4")])
VALUE_NOOP = -(1 << 31)
# ServerInbound members (VanillaMencius.proto:227-241)
CLIENT_REQUEST, PHASE1A, PHASE1B, PHASE2A, PHASE2B, SKIP, CHOSEN_KIND, PHASE1_NACK, PHASE2_NACK = range(1, 10)

_lib = None


def build():
    src = open(_SRC, "rb").read()
    d = os.path.join(tempfile.gettempdir(), f"fpx_wire_vm_oracle_{os.getuid()}_{hashlib.sha1(src).hexdigest()[:16]}")
    so = os.path.join(d, "libwire_vm_oracle.so")
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
        L.fpo_wire_decode_vm.argtypes = [vp, vp, i32, vp, vp, vp, i64p]; L.fpo_wire_decode_vm.restype = i32
        L.fpo_wire_encode_vm.argtypes = [i32, vp, i32, i32, vp, vp, i32, vp, vp, i64p]
        L.fpo_wire_encode_vm.restype = C.c_int64
        _lib = L
    return _lib


def pack(msgs):
    """Messages back to back + offsets[n+1] (the codec's batch layout)."""
    offs = np.zeros(len(msgs) + 1, dtype=np.int32)
    offs[1:] = np.cumsum([len(m) for m in msgs])
    return np.frombuffer(b"".join(msgs) + b"\0" * 16, dtype=np.uint8).copy(), offs


def decode(buf, offs):
    """-> (status, err_index, kind[n], rec[n], sender[n])"""
    buf = np.ascontiguousarray(buf, dtype=np.uint8)
    offs = np.ascontiguousarray(offs, dtype=np.int32)
    n = len(offs) - 1
    pad = np.zeros(max(len(buf), 1), dtype=np.uint8); pad[:len(buf)] = buf
    kind = np.zeros(max(n, 1), dtype=np.int32)
    rec = np.zeros(max(n, 1), dtype=WIRE_REC)
    sender = np.zeros(max(n, 1), dtype=np.int32)
    err = C.c_int64(-1)
    st = lib().fpo_wire_decode_vm(pad.ctypes.data, offs.ctypes.data, n, kind.ctypes.data, rec.ctypes.data,
                                  sender.ctypes.data, C.byref(err))
    return st, err.value, kind[:n], rec[:n], sender[:n]


_KINDS = {"replies": (0, P2B), "chosen": (1, CHOSEN), "phase2a": (2, P2A), "skip": (3, VM_SKIP)}


def encode(what, recs, arena=None, value_offsets=None, servers=7):
    """what: replies / chosen / phase2a / skip -> (status, err_index, bytes, offsets[n+1])"""
    k, dt = _KINDS[what]
    recs = np.ascontiguousarray(recs, dtype=dt)
    arena = np.zeros(1, dtype=np.uint8) if arena is None or len(arena) == 0 else np.ascontiguousarray(arena, dtype=np.uint8)
    value_offsets = np.zeros(1, dtype=np.int32) if value_offsets is None else np.ascontiguousarray(value_offsets, dtype=np.int32)
    n = len(recs)
    offs = np.zeros(n + 1, dtype=np.int32)
    err = C.c_int64(-1)
    args = (k, recs.ctypes.data, n, servers, arena.ctypes.data, value_offsets.ctypes.data, len(value_offsets) - 1)
    total = lib().fpo_wire_encode_vm(*args, None, offs.ctypes.data, C.byref(err))
    if total < 0:
        return int(total), err.value, np.zeros(0, dtype=np.uint8), offs
    out = np.zeros(max(total, 1), dtype=np.uint8)
    lib().fpo_wire_encode_vm(*args, out.ctypes.data, offs.ctypes.data, C.byref(err))
    return 0, -1, out[:total], offs


def split(out, offs):
    return [bytes(out[offs[i]: offs[i + 1]]) for i in range(len(offs) - 1)]
