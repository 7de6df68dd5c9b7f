"""ctypes loader for libfpx.so (the C ABI of include/fpx.h).

There is no CPU fallback: if the shared library is missing it is built with
nvcc; if that fails, or a symbol declared in include/fpx.h is missing, import
of the product raises.  Every entry point is bound from its prototype in the
header, so no signature is written down twice.
"""
import ctypes as C
import os
import re

from . import build as _build

HEADER = os.path.join(_build.ROOT, "include", "fpx.h")
DEBUG_HEADER = os.path.join(_build.CSRC, "fpx_debug.h")     # test and profiling aids, not part of the ABI

_lib = None


def prototypes(path):
    """[(return type, name, [(parameter type, parameter name)])] of every fpx_* function the C header declares."""
    with open(path) as f:
        src = f.read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    src = re.sub(r"#.*", "", src)
    protos = []
    for m in re.finditer(r"([A-Za-z_][A-Za-z0-9_ \*]*?)\b(fpx_[a-z0-9_]+)\s*\(([^;{}]*?)\)\s*;", src, flags=re.S):
        ret, name, args = m.group(1).strip(), m.group(2), " ".join(m.group(3).split())
        if "typedef" in ret or "struct" in ret.split()[:1]:
            continue
        params = []
        if args and args != "void":
            for a in args.split(","):
                a = a.strip()
                mm = re.match(r"(.*?)([A-Za-z_][A-Za-z0-9_]*)$", a)
                params.append((mm.group(1).strip(), mm.group(2)))
        protos.append((ret, name, params))
    return protos


_SCALARS = {"int": C.c_int32, "int32_t": C.c_int32, "uint32_t": C.c_uint32, "int64_t": C.c_int64, "float": C.c_float}


def ctype(c_type, ret=False):
    """The ctypes type of a parameter or return type of the header.  Every pointer but a returned string is a
    c_void_p: callers pass array addresses, byref(...), None, device addresses and string buffers alike."""
    t = c_type.replace("const", "").replace(" ", "")
    if ret and t == "void":
        return None
    if ret and t == "char*":
        return C.c_char_p
    if "*" in t:
        return C.c_void_p
    return _SCALARS[t]


class Config(C.Structure):
    """struct fpx_config (include/fpx.h)."""
    _fields_ = [(n, C.c_int32) for n in (
        "struct_size", "protocol", "f", "num_acceptor_groups", "acceptors_per_group", "flexible",
        "num_leaders", "num_replicas", "slot_capacity", "overflow_capacity", "max_batch", "device",
        "shard_index", "shard_count", "num_leader_groups")]


class SyncResult(C.Structure):
    """struct fpx_sync_result (include/fpx.h)."""
    _fields_ = [("status", C.c_int32), ("reserved", C.c_int32), ("err_index", C.c_int64),
                ("n_p2b", C.c_int32), ("n_nack", C.c_int32), ("n_chosen", C.c_int32),
                ("watermark", C.c_int32)]


class ReadsSyncResult(C.Structure):
    """struct fpx_reads_sync_result (include/fpx.h)."""
    _fields_ = [("status", C.c_int32), ("watermark", C.c_int32), ("err_index", C.c_int64),
                ("n_slots", C.c_int32), ("n_replies", C.c_int32), ("n_released", C.c_int32), ("n_pending", C.c_int32)]


class EpaxosConfig(C.Structure):
    """struct fpx_epaxos_config (include/fpx.h)."""
    _fields_ = [(n, C.c_int32) for n in ("struct_size", "f", "replica_index", "instances_per_replica",
                                         "max_batch", "device")]


def lib():
    global _lib
    if _lib is not None:
        return _lib
    path = os.environ.get("FPX_LIB_OVERRIDE") or _build.LIB      # override: A/B against another build (profiles/)
    if path == _build.LIB and (not os.path.exists(path) or (_build.stale() and _build.have_nvcc())):
        path = _build.build(force=True)
    L = C.CDLL(path)
    protos = prototypes(HEADER)
    missing = [name for _, name, _ in protos if not hasattr(L, name)]
    if missing:
        raise ImportError(f"libfpx.so lacks symbols declared in include/fpx.h: {missing}")
    # the test aids are not part of the ABI: a build loaded through FPX_LIB_OVERRIDE may predate some of them
    for ret, name, params in protos + [p for p in prototypes(DEBUG_HEADER) if hasattr(L, p[1])]:
        fn = getattr(L, name)
        fn.argtypes = [ctype(t) for t, _ in params]
        fn.restype = ctype(ret, ret=True)
    if L.fpx_abi_version() != 1:
        raise ImportError("libfpx.so ABI version mismatch")
    _lib = L
    return L
