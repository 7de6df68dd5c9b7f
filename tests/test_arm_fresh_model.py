"""The CPU model of the arm's fresh-key certificate and fresh frontier (arm_fresh_model.py): hand cases for every
condition of the certificate and every rule of the frontier, and a guard that the model's pass-1 geometry is the
kernel's, read from fpx_arm.cuh.  No GPU."""
import os
import re

import numpy as np

import arm_fresh_model as M
from frankenpaxos_b200 import P2A_RANGE, P2B
from frankenpaxos_b200 import traces as T

ARM_CUH = os.path.join(os.path.dirname(__file__), "..", "frankenpaxos_b200", "csrc", "fpx_arm.cuh")
FPX_H = os.path.join(os.path.dirname(__file__), "..", "include", "fpx.h")


def constant(text, name):
    m = re.search(r"constexpr\s+int\s+" + name + r"\s*=\s*(\d+)\s*;", text)
    assert m, f"{name} not found in fpx_arm.cuh"
    return int(m.group(1))


def test_geometry_matches_the_kernel():
    """A retune of the arm kernel moves the edge positions the GPU tests place their violations at: the model's
    constants must follow it."""
    with open(ARM_CUH) as f:
        text = f.read()
    assert constant(text, "kArmThreads") == M.THREADS
    assert constant(text, "kArmCertUnroll") == M.CERT_UNROLL
    assert constant(text, "kArmUnroll") == M.UNROLL
    assert constant(text, "kArmUnrollCertified") == M.FALLBACK_UNROLL
    with open(FPX_H) as f:
        m = re.search(r"#define FPX_MAX_ROUND (0x[0-9a-fA-F]+)", f.read())
    assert int(m.group(1), 16) == M.MAX_ROUND
    assert (M.WARP_GROUP, M.CERT_CTA, M.GRID_CTA) == (128, 4096, 8192)


def test_grid_and_strides():
    assert M.arm_blocks(1, 132) == 1 and M.arm_blocks(8192, 132) == 1 and M.arm_blocks(8193, 132) == 2
    assert M.arm_blocks(132 * 8192 + 4097, 132) == 132
    n = 3 * 8192 + 1013
    assert M.arm_blocks(n, 132) == 4 and M.cert_stride(n, 132) == 16384
    # every batch above 4096 records needs a second stride of pass 1
    for n in (4097, 8192, 8193, 1 << 20):
        assert M.cert_stride(n, 132) < n


def test_local_ordinal():
    g = M.Geometry(capacity=1000)
    assert M.local_ordinal([-1, 0, 999, 1000, 1 << 30], g).tolist() == [-1, 0, 999, -1, -1]
    g.retire_below(300)
    assert g.base_local == 300 and g.slot_capacity == 1300
    assert M.local_ordinal([0, 299, 300, 1299, 1300], g).tolist() == [M.RETIRED, M.RETIRED, 300, 1299, -1]
    g.retire_below(100)        # the window never slides back
    assert g.base_local == 300
    # shard 1 of 3: capacity 1000 -> 333 local slots (ordinals of slots 1, 4, ..., 997)
    s = M.Geometry(capacity=1000, shard_index=1, shard_count=3)
    assert s.local_slots == 333
    assert M.local_ordinal([1, 2, 3, 4, 997, 998, 1000], s).tolist() == [0, -1, -1, 1, 332, -1, -1]
    s.retire_below(5)          # first ordinal whose slot is >= 5: slot 7, ordinal 2
    assert s.base_local == 2 and s.slot_capacity == 1006
    assert M.local_ordinal([1, 4, 7, 1003, 1006], s).tolist() == [M.RETIRED, M.RETIRED, 2, 334, -1]


def arms(slots, rnd=0):
    return T.arms(np.asarray(slots, dtype=np.int32), rnd)


def test_certificate_conditions():
    g = M.Geometry(capacity=1 << 12)
    ok = arms(np.arange(10, 100))
    assert M.certified(ok, g, 0) and M.certified(ok, g, 10)
    assert not M.certified(arms([]), g, 0)                              # n > 0
    assert not M.certified(ok, g, 11)                                   # the first ordinal below the frontier
    for i in (0, 45, 88):
        b = ok.copy()
        b["slot"][i + 1] = b["slot"][i]                                  # a repeated key, either value
        assert not M.certified(b, g, 0)
        b["round"][i + 1] = 1                                            # a second round of the slot
        assert not M.certified(b, g, 0)
        b = ok.copy()
        b[[i, i + 1]] = b[[i + 1, i]]                                    # two neighbours swapped
        assert not M.certified(b, g, 0)
    for bad_round in (-1, M.MAX_ROUND + 1, -(1 << 31)):
        b = ok.copy()
        b["round"][-1] = bad_round
        assert not M.certified(b, g, 0)
    b = ok.copy()
    b["round"][:] = M.MAX_ROUND
    assert M.certified(b, g, 0)
    assert not M.certified(arms([4094, 4095, 4096]), g, 0)              # the last one beyond the window
    assert M.certified(arms([0, 5, 4095]), g, 0)                        # gaps are fine
    # signed order: a negative slot is out of the window anyway
    assert not M.certified(arms([-5, 3]), g, 0)
    g.retire_below(64)
    assert not M.certified(arms(np.arange(63, 80)), g, 0)               # a retired slot
    assert M.certified(arms(np.arange(64, 80)), g, 0)
    s = M.Geometry(capacity=3000, shard_index=1, shard_count=3)
    assert M.certified(arms([1, 4, 7, 10]), s, 0)
    assert not M.certified(arms([1, 4, 8, 10]), s, 0)                   # a slot of shard 2


def test_frontier_rules():
    g = M.Geometry(capacity=100)
    fr = M.Frontier(M.MULTIPAXOS, g)
    assert fr.arm(arms(np.arange(10))) == "fresh" and fr.value == 10
    assert fr.arm(arms(np.arange(5, 20))) == "cas" and fr.value == 20          # re-arms below the frontier
    assert fr.arm(arms([20, 25])) == "fresh" and fr.value == 26
    # an empty call launches nothing: the last path stands and the frontier stays
    assert fr.arm(arms([])) == "fresh" and fr.value == 26
    # a refused batch still raises the frontier, over every record of the live window, the bad round's too
    b = arms([30, 40, 120])
    b["round"][1] = M.MAX_ROUND + 1
    assert fr.arm(b) == "cas" and fr.value == 41
    # a tally raises it to one past its largest live vote; votes outside the window do not count
    v = np.zeros(3, dtype=P2B)
    v["slot"] = [50, 60, 500]
    fr.tally(v)
    assert fr.value == 61
    fr.tally(np.zeros(0, dtype=P2B))
    assert fr.value == 61
    # retire_below leaves it alone, and the recycled ordinals enter above it
    fr.retire_below(80)
    assert fr.value == 61 and g.slot_capacity == 180
    assert fr.arm(arms([79, 100])) == "cas" and fr.value == 101                 # a retired slot
    assert fr.arm(arms(np.arange(101, 180))) == "fresh" and fr.value == 180
    assert fr.arm(arms([180])) == "cas" and fr.value == 180                     # beyond the window
    fr.reset()
    assert (fr.value, fr.last_path, g.base_local) == (0, "none", 0)
    assert fr.arm(arms(np.arange(10))) == "fresh"


def test_paths_per_engine_kind():
    g = M.Geometry(capacity=100)
    van = M.Frontier(M.VANILLA, g)
    assert van.arm(arms(np.arange(10))) == "cas" and van.value == 0           # the plain kernel leaves it alone
    men = M.Frontier(M.MENCIUS, M.Geometry(capacity=100))
    assert men.arm(arms([0, 2, 4])) == "fresh"
    men.arm_range(np.array([(6, 20, 0, -1)], dtype=P2A_RANGE))
    assert men.arm(arms([21, 23])) == "fresh" and men.value == 24
    men.arm_range(np.array([(30, 40, 0, -1), (41, 42, 0, -1)], dtype=P2A_RANGE))   # a one-slot range: sticky
    assert men.arm(arms([50, 52])) == "cas" and men.value == 24
    assert men.arm(arms([60])) == "cas"
    men.reset()
    assert men.arm(arms([0, 2])) == "fresh"


def test_pair_positions_of_the_test_batch():
    """The seams the GPU test places its violations at, derived from the geometry."""
    n = 3 * M.GRID_CTA + 1013
    stride = M.cert_stride(n, 132)
    seams = {0, 30, M.CHUNK - 1, M.WARP_GROUP - 1, M.CERT_CTA - 1, stride - 1, n - 2}
    assert seams == {0, 30, 31, 127, 4095, 16383, n - 2}
    assert n % M.CHUNK != 0 and (n - 2) // M.CHUNK == (n - 1) // M.CHUNK      # the last pair inside the ragged chunk
    # the pair (i, i + 1) crosses a chunk for 31, a warp for 127, a CTA for 4095, a stride for 16383
    for i, unit in ((31, M.CHUNK), (127, M.WARP_GROUP), (4095, M.CERT_CTA), (16383, stride)):
        assert i // unit != (i + 1) // unit
    assert 30 // M.CHUNK == 31 // M.CHUNK
