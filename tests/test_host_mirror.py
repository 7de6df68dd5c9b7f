"""The C++ host mirror (frankenpaxos_b200/host/frankenpaxos_host.hpp: Actor / Transport /
Chan / FakeTransport / GpuProxyLeader / GpuAcceptor) above the C ABI."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def bin_dir(tmp_path_factory):
    """The host binaries are compiled outside the source tree, which may be read-only."""
    return str(tmp_path_factory.mktemp("host"))


def _compile(name, opt, out_dir):
    from frankenpaxos_b200 import build as B
    from oracle import fpx_oracle_py as O
    lib = B.build()
    O.build()
    src = os.path.join(ROOT, "tests", "host", name + ".cc")
    out = os.path.join(out_dir, name)
    cmd = ["g++", "-std=c++17", opt, "-Wall", "-Wextra", src, "-o", out,
           "-L" + os.path.dirname(lib), "-lfpx", "-L" + os.path.join(ROOT, "oracle"), "-lfpx_oracle",
           "-Wl,-rpath," + os.path.dirname(lib), "-Wl,-rpath," + os.path.join(ROOT, "oracle")]
    subprocess.check_call(cmd)
    return out


def build(out_dir):
    return _compile("fake_transport_parity", "-O1", out_dir)


def build_simulation(out_dir):
    return _compile("simulation", "-O2", out_dir)


def test_randomized_simulation_of_the_batching_shim_on_the_oracle_backend(bin_dir):
    """No GPU: the reference's randomized simulation (T/multipaxos/MultiPaxosTest.scala) over the host mirror,
    per-message handling vs one flush per step, both on the oracle backend; 60 runs x 250 steps per shape."""
    r = subprocess.run([build_simulation(bin_dir), "60", "250", "cpu"], capture_output=True, text=True, timeout=900)
    print(r.stdout, r.stderr)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.count("SIMULATION OK") == 4


@pytest.mark.gpu
def test_randomized_simulation_gpu_backend_matches_per_message_oracle(bin_dir):
    """The reference's own way of testing its handlers, on the product: 500 runs x 250 random steps (writes,
    random deliveries, leader changes through Phase 1) for f in {1, 2} x {majority, grid}, invariants of
    T/multipaxos/MultiPaxos.scala:291-320 after every step, and the batched CUDA backend byte-identical to the
    per-message oracle backend on everything replicas and leaders receive and on the final acceptor state."""
    r = subprocess.run([build_simulation(bin_dir), "500", "250"], capture_output=True, text=True, timeout=3000)
    print(r.stdout[-3000:], r.stderr[-2000:])
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert r.stdout.count("SIMULATION OK") == 4


def test_host_mirror_compiles_and_links(bin_dir):
    assert os.path.exists(build(bin_dir))


def test_batching_shim_on_the_oracle_backend(bin_dir):
    """No GPU: the host logic alone (GpuProxyLeader / GpuAcceptor buffering a delivery burst, one flush,
    replies routed back in order) against one-handler-per-message, both over the oracle backend --
    BASELINE cfg1 on FakeTransport with a leader change, three seeds."""
    r = subprocess.run([build(bin_dir), "128", "cpu"], capture_output=True, text=True, timeout=600)
    print(r.stdout, r.stderr)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.count("PARITY OK") == 3


@pytest.mark.gpu
def test_fake_transport_run_cfg1_parity(bin_dir):
    """BASELINE cfg1 (MultiPaxos f=1, 3 acceptors, 128 slots on FakeTransport) with a
    leader change: batched GPU actors vs per-message oracle actors, identical transcripts."""
    r = subprocess.run([build(bin_dir), "128"], capture_output=True, text=True, timeout=600)
    print(r.stdout, r.stderr)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.count("PARITY OK") == 3
