"""The C-ABI library builds, loads and exports every symbol include/fpx.h declares, bound with the ctypes types
of its prototype (no compute calls: this runs without a GPU)."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "fpx.h")
DEBUG_HEADER = os.path.join(ROOT, "frankenpaxos_b200", "csrc", "fpx_debug.h")


def declared_symbols(path=HEADER):
    src = open(path).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(fpx_\w+)\s*\(", src)))


def mapped(c_type, ret=False):
    """The ctypes type a C type of the headers is bound with."""
    if ret and c_type == "const char*":
        return ctypes.c_char_p
    if "*" in c_type:
        return ctypes.c_void_p
    if ret and c_type == "void":
        return None
    return {"int": ctypes.c_int32, "int32_t": ctypes.c_int32, "uint32_t": ctypes.c_uint32,
            "int64_t": ctypes.c_int64, "float": ctypes.c_float}[c_type]


def check_bound(L, path):
    from frankenpaxos_b200 import _lib
    protos = _lib.prototypes(path)
    names = [name for _, name, _ in protos]
    assert sorted(names) == declared_symbols(path), f"prototypes() skips or invents a declaration of {path}"
    missing = [s for s in names if not hasattr(L, s)]
    assert not missing, missing
    for ret, name, params in protos:
        fn = getattr(L, name)
        assert fn.argtypes == [mapped(t) for t, _ in params], (name, fn.argtypes)
        assert fn.restype is mapped(ret, ret=True), (name, fn.restype)
    return names


def test_header_prototypes_exported_and_bound():
    from frankenpaxos_b200 import _lib
    L = _lib.lib()
    assert len(check_bound(L, HEADER)) >= 20
    assert L.fpx_abi_version() == 1


def test_test_aids_exported_and_bound():
    """The fpx_debug_* aids are declared in fpx_debug.h, not in include/fpx.h, and bound like the ABI."""
    from frankenpaxos_b200 import _lib
    names = check_bound(_lib.lib(), DEBUG_HEADER)
    assert len(names) == 9 and all(n.startswith("fpx_debug_") for n in names)
    assert not set(names) & set(declared_symbols())


def test_struct_layouts_match_header():
    from frankenpaxos_b200 import _lib, engine
    assert ctypes.sizeof(_lib.Config) == 15 * 4
    assert ctypes.sizeof(_lib.SyncResult) == 32
    assert ctypes.sizeof(_lib.ReadsSyncResult) == 32
    assert ctypes.sizeof(_lib.EpaxosConfig) == 6 * 4
    assert engine.P2A.itemsize == 16 and engine.P2B.itemsize == 16
    assert engine.CHOSEN.itemsize == 8 and engine.NACK.itemsize == 8


def test_no_cpu_fallback_without_device():
    """Constructing an engine without a CUDA device must fail loudly."""
    import torch
    import pytest
    from frankenpaxos_b200 import Engine, FpxError
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(FpxError) as ei:
        Engine(1, 1, 3)
    assert ei.value.status == -10


def test_config_validation_is_checked_before_device():
    """Config.checkValid (multipaxos/Config.scala:32-147) clauses -> FPX_ERR_CONFIG."""
    from frankenpaxos_b200 import Engine, FpxError
    import pytest
    bad = [
        dict(f=0, num_acceptor_groups=1, acceptors_per_group=1),               # f >= 1
        dict(f=1, num_acceptor_groups=1, acceptors_per_group=4),               # 2f+1 per group
        dict(f=1, num_acceptor_groups=1, acceptors_per_group=3, num_leaders=1),  # >= f+1 leaders
        dict(f=1, num_acceptor_groups=1, acceptors_per_group=3, num_replicas=1),
        dict(f=2, num_acceptor_groups=2, acceptors_per_group=3, flexible=True),  # min(2,3)-1 < 2
    ]
    for kw in bad:
        with pytest.raises(FpxError) as ei:
            Engine(**kw)
        assert ei.value.status == -2, kw


def test_jni_symbols_exported():
    """Every `@native def` of INTEGRATION.md's Native.scala is an exported Java_frankenpaxos_gpu_Native_* symbol
    (frankenpaxos_b200/csrc/fpx_jni.c by hand, fpx_jni_gen.c generated from include/fpx.h), and every entry
    point of include/fpx.h is reachable from the JVM side."""
    from frankenpaxos_b200 import build
    L = ctypes.CDLL(build.build())
    md = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    methods = re.findall(r"@native def ([A-Za-z0-9_]+)\(", md)
    assert len(methods) >= 80 and len(set(methods)) == len(methods)
    missing = [m for m in methods if not hasattr(L, "Java_frankenpaxos_gpu_Native_" + m)]
    assert not missing, missing
    # coverage of the C ABI: every fpx_* function is called by some JNI stub
    jni = open(os.path.join(ROOT, "frankenpaxos_b200", "csrc", "fpx_jni.c")).read() + \
        open(os.path.join(ROOT, "frankenpaxos_b200", "csrc", "fpx_jni_gen.c")).read()
    called = set(re.findall(r"\b(fpx_[a-z0-9_]+)\s*\(", jni))
    assert not [s for s in declared_symbols() if s not in called]


def test_generated_jni_is_up_to_date():
    """fpx_jni_gen.c and the GENERATED block of INTEGRATION.md are what gen_jni.py produces from the header."""
    import subprocess
    import sys
    gen = os.path.join(ROOT, "frankenpaxos_b200", "csrc", "fpx_jni_gen.c")
    before_c, before_md = open(gen).read(), open(os.path.join(ROOT, "INTEGRATION.md")).read()
    subprocess.check_call([sys.executable, os.path.join(ROOT, "frankenpaxos_b200", "csrc", "gen_jni.py")])
    assert open(gen).read() == before_c and open(os.path.join(ROOT, "INTEGRATION.md")).read() == before_md
