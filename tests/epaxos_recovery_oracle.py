"""ctypes binding of the EPaxos recovery oracle (tests/epaxos_recovery_oracle.cc).  TEST INFRASTRUCTURE.

One replica with all eleven fpx_epaxos_* calls: the handlers on the path come from oracle/fpx_oracle.cc (compiled
into the same library), the recovery handlers and timer-driven transitions from the derived struct.  Same row
formats as frankenpaxos_b200.epaxos.EpaxosReplica, one message at a time.  The library is compiled with g++ into a
temporary directory named after the sources' hash, so the tests also run from a read-only tree."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "epaxos_recovery_oracle.cc")
_BASE = os.path.join(os.path.dirname(_HERE), "oracle", "fpx_oracle.cc")

_lib = None


def build():
    h = hashlib.sha1(open(_SRC, "rb").read() + open(_BASE, "rb").read()).hexdigest()[:16]
    d = os.path.join(tempfile.gettempdir(), f"fpx_epaxos_recovery_oracle_{os.getuid()}_{h}")
    so = os.path.join(d, "libepaxos_recovery_oracle.so")
    if not os.path.exists(so):
        os.makedirs(d, exist_ok=True)
        tmp = f"{so}.{os.getpid()}"
        subprocess.check_call([os.environ.get("CXX", "g++"), "-O2", "-std=c++17", "-fPIC", "-Wall", "-Wextra",
                               "-fno-strict-aliasing", "-shared", "-pthread", "-o", tmp, _SRC])
        os.replace(tmp, so)   # atomic: concurrent test processes never load a half-written library
    return so


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(build())
        vp, i32, ip = C.c_void_p, C.c_int, C.POINTER(C.c_int)
        L.fpo_epr_new.argtypes = [i32, i32]; L.fpo_epr_new.restype = vp
        L.fpo_epr_free.argtypes = [vp]
        L.fpo_epr_base.argtypes = [vp]; L.fpo_epr_base.restype = vp
        L.fpo_ep_lead.argtypes = [vp, i32, i32, i32, i32, i32, i32, vp, i32]; L.fpo_ep_lead.restype = i32
        L.fpo_ep_pre_accept.argtypes = [vp, i32, i32, i32, i32, i32, i32, vp, vp, vp, ip]
        L.fpo_ep_accept.argtypes = [vp, i32, i32, i32, i32, i32, i32, vp, vp, ip]
        L.fpo_ep_pre_accept_ok.argtypes = [vp, i32, i32, i32, i32, i32, i32, vp, vp, ip]
        L.fpo_ep_accept_ok.argtypes = [vp, i32, i32, i32, i32, i32, vp, ip]
        L.fpo_ep_entry.argtypes = [vp, i32, i32, vp]; L.fpo_ep_entry.restype = i32
        L.fpo_ep_leader_kind.argtypes = [vp, i32, i32]; L.fpo_ep_leader_kind.restype = i32
        L.fpo_ep_largest_ballot.argtypes = [vp, vp]
        L.fpo_epr_commit.argtypes = [vp, i32, i32, i32, i32, vp]
        L.fpo_epr_nack.argtypes = [vp, i32, i32, i32, i32]; L.fpo_epr_nack.restype = i32
        L.fpo_epr_prepare_phase.argtypes = [vp, i32, i32, vp]; L.fpo_epr_prepare_phase.restype = i32
        L.fpo_epr_prepare.argtypes = [vp, i32, i32, i32, i32, vp, ip]
        L.fpo_epr_prepare_ok.argtypes = [vp] + [i32] * 9 + [vp]; L.fpo_epr_prepare_ok.restype = i32
        L.fpo_epr_slow_path_timer.argtypes = [vp, i32, i32, i32, i32, vp, ip]
        _lib = L
    return _lib


def _i(xs):
    return [int(x) for x in xs]


class EPaxos:
    """One epaxos.Replica; calls that can fail return (status, err_index[, out])."""

    def __init__(self, f, index):
        self.f, self.n, self.index = f, 2 * f + 1, index
        self.h = lib().fpo_epr_new(f, index)
        self.hb = lib().fpo_epr_base(self.h)     # the handlers on the path take the base object
        self.saw_sparse = False

    def __del__(self):
        try:
            lib().fpo_epr_free(self.h)
        except Exception:
            pass

    def _rows(self, rows, w):
        return np.ascontiguousarray(rows, dtype=np.int32).reshape(-1, w)

    def _deps(self, r):
        return np.ascontiguousarray(r, dtype=np.int32)

    # ---- the handlers on the path (oracle/fpx_oracle.cc)
    def lead(self, rows):
        n = self.n
        for i, r in enumerate(self._rows(rows, 8 + n)):
            if lib().fpo_ep_lead(self.hb, *_i(r[:6]), self._deps(r[8:8 + n]).ctypes.data, int(r[6])) != 0:
                return -13, i
        return 0, -1

    def _each(self, rows, w, w_out, call):
        out = np.zeros((len(rows), w_out), dtype=np.int32)
        sp = C.c_int(0)
        for i, r in enumerate(rows):
            call(r, out[i].ctypes.data, C.byref(sp))
            self.saw_sparse |= bool(sp.value)
        return out

    def preaccept(self, rows):
        n = self.n
        rows = self._rows(rows, 6 + 2 * n)
        return self._each(rows, 6 + 2 * n, 4 + n, lambda r, o, sp: lib().fpo_ep_pre_accept(
            self.hb, *_i(r[:6]), self._deps(r[6:6 + n]).ctypes.data, self._deps(r[6 + n:]).ctypes.data, o, sp))

    def accept(self, rows):
        n = self.n
        rows = self._rows(rows, 6 + n)
        return self._each(rows, 6 + n, 4 + n, lambda r, o, sp: lib().fpo_ep_accept(
            self.hb, *_i(r[:6]), self._deps(r[6:]).ctypes.data, o, sp))

    def preacceptok(self, rows):
        n = self.n
        rows = self._rows(rows, 6 + n)
        return self._each(rows, 6 + n, 2 + n, lambda r, o, sp: lib().fpo_ep_pre_accept_ok(
            self.hb, *_i(r[:6]), self._deps(r[6:]).ctypes.data, o, sp))

    def acceptok(self, rows):
        rows = self._rows(rows, 6)
        return self._each(rows, 6, 2 + self.n, lambda r, o, sp: lib().fpo_ep_accept_ok(self.hb, *_i(r[:5]), o, sp))

    def entry(self, rep, num):
        out = np.zeros(7 + self.n, dtype=np.int32)
        if not lib().fpo_ep_entry(self.hb, rep, num, out.ctypes.data):
            out[:] = 0
            out[1:5] = -1
        elif out[0] == 4:
            out[1:5] = -1
        lb = np.zeros(2, dtype=np.int32)
        lib().fpo_ep_largest_ballot(self.hb, lb.ctypes.data)
        return out, lib().fpo_ep_leader_kind(self.hb, rep, num), lb

    # ---- recovery and the timer-driven transitions (tests/epaxos_recovery_oracle.cc)
    def commit(self, rows):
        n = self.n
        for r in self._rows(rows, 4 + n):
            lib().fpo_epr_commit(self.h, *_i(r[:4]), self._deps(r[4:]).ctypes.data)

    def nack(self, rows):
        rows = self._rows(rows, 4)
        return np.array([[lib().fpo_epr_nack(self.h, *_i(r))] for r in rows], dtype=np.int32).reshape(-1, 1)

    def prepare_phase(self, rows):
        rows = self._rows(rows, 2)
        out = np.full((len(rows), 2), -1, dtype=np.int32)
        for i, r in enumerate(rows):
            st = lib().fpo_epr_prepare_phase(self.h, *_i(r), out[i].ctypes.data)
            if st != 0:
                return st, i, out
        return 0, -1, out

    def prepare(self, rows):
        rows = self._rows(rows, 4)
        return self._each(rows, 4, 9 + self.n, lambda r, o, sp: lib().fpo_epr_prepare(self.h, *_i(r), o, sp))

    def prepareok(self, rows):
        rows = self._rows(rows, 9)
        out = np.zeros((len(rows), 4), dtype=np.int32)
        for i, r in enumerate(rows):
            st = lib().fpo_epr_prepare_ok(self.h, *_i(r), out[i].ctypes.data)
            if st != 0:
                return st, i, out
        return 0, -1, out

    def slow_path_timer(self, rows):
        rows = self._rows(rows, 4)
        return self._each(rows, 4, 2 + self.n, lambda r, o, sp: lib().fpo_epr_slow_path_timer(self.h, *_i(r), o, sp))
