"""In-tree build of libfpx.so (sm_90a only).  `python -m frankenpaxos_b200.build`."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "lib", "libfpx.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC,-Wall,-Wextra,-Wno-unused-parameter",
    "-shared", "-cudart", "static",
]


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".c", ".cc")))


def deps():
    d = [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    d.append(os.path.join(ROOT, "include", "fpx.h"))
    return d


def have_nvcc():
    return os.path.exists(os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc"))


def stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(p) > t for p in deps())


def build(force=False, verbose=False):
    """Compile frankenpaxos_b200/csrc/*.cu -> frankenpaxos_b200/lib/libfpx.so."""
    if not force and not stale():
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    os.makedirs(os.path.dirname(LIB), exist_ok=True)
    cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + \
        ["-I", os.path.join(ROOT, "include"), "-o", LIB] + sources()
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("nvcc failed building libfpx.so")
    if verbose:
        sys.stderr.write(r.stderr)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
