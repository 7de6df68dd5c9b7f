"""Executing EPaxos commits on the GPU with dense prefix dependencies (fpx_epaxos_graph_*, DESIGN §6b).

  cfg4     the 2^20 Commit rows replica 0 receives at BASELINE cfg4 (the `com` buffer of bench_epaxos_cfg4.py),
           committed with commit_dev from that device buffer, then one executeByComponent: its device time
           (CUDA events around its kernels, without the two host read-backs), best of `--reps` fresh handles
  chain    a reverse chain of 2^18 instances (x depends on x - 1, committed last to first): as prefix vectors in
           fpx_epaxos_graph (one column, watermark x) and as explicit x -> x - 1 edges in fpx_depgraph; both give
           the same components in the same order.  Host clock around each execute call, and the new handle's
           device time
  conflict ConflictIndex.batch (QUERY_THEN_PUT) at the size of test_conflict_index_many_tiles_matches_the_oracle:
           2^17 commands of 8 leaders on one of two hot keys (segments over ~90 and ~40 tiles of the segmented
           scan).  Host clock around the C call (its copies, kernels and status read-back) from prebuilt arrays,
           median and best of 20 calls per fresh handle, `--reps` handles

Prints the card name and power limit first, then one JSON line.
    python profiles/bench_epaxos_graph.py [--reps 3]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from frankenpaxos_b200 import traces as T  # noqa: E402
from frankenpaxos_b200.epaxos import ConflictIndex, DependencyGraph, EpaxosGraph  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def cfg4(reps, N=1 << 20, f=2):
    n = 2 * f + 1
    _, pa, _ = T.epaxos_cfg4(0, f=f, n_instances=N, me=0)
    com = np.concatenate([pa[:, 0:2], pa[:, 4:6], pa[:, 6 + n:6 + 2 * n]], axis=1)
    d_com = torch.from_numpy(np.ascontiguousarray(com, dtype=np.int32)).to("cuda")
    torch.cuda.synchronize()
    best, wall, res = 1e9, 1e9, None
    for _ in range(reps):
        g = EpaxosGraph(n, N // n + 2, max_batch=len(com))
        g.commit_dev(d_com.data_ptr(), len(com))
        g.sync()
        t = time.perf_counter()
        out, heads, bl = g.execute_raw()
        wall = min(wall, time.perf_counter() - t)
        best = min(best, g.last_kernel_ms())
        res = {"executed": len(out), "components": int(heads.sum()), "largest_component":
               int(np.diff(np.append(np.nonzero(heads)[0], len(out))).max()) if len(out) else 0,
               "blockers": int(bl.sum())}
        g.close()
    return {"rows": len(com), **res, "execute_kernel_ms": best, "execute_call_ms": wall * 1e3}


def chain(reps, L=1 << 18):
    rows = np.zeros((L, 5), np.int32)
    rows[:, 1] = np.arange(L)
    rows[:, 4] = np.arange(L)                      # x names [0, x): x - 1 and everything below it
    rows = rows[::-1].copy()
    keys = list(range(L - 1, -1, -1))
    deps = [[k - 1] if k else [] for k in keys]
    prefix_ms, prefix_wall, edge_wall = 1e9, 1e9, 1e9
    for _ in range(reps):
        g = EpaxosGraph(1, L, max_batch=L)
        g.commit(rows)
        t = time.perf_counter()
        out, heads, _ = g.execute_raw()
        prefix_wall = min(prefix_wall, time.perf_counter() - t)
        prefix_ms = min(prefix_ms, g.last_kernel_ms())
        g.close()
        dg = DependencyGraph(key_capacity=L, dep_pool_capacity=L, max_batch=L)
        dg.commit(keys, [0] * L, deps)
        t = time.perf_counter()
        comps, _ = dg.execute_by_component()
        edge_wall = min(edge_wall, time.perf_counter() - t)
        dg.close()
        assert heads.all() and out[:, 1].tolist() == list(range(L))
        assert comps == [[k] for k in range(L)]
    return {"instances": L, "same_components_same_order": True,
            "prefix_execute_kernel_ms": prefix_ms, "prefix_execute_call_ms": prefix_wall * 1e3,
            "edges_execute_call_ms": edge_wall * 1e3}


def conflict(reps, n=1 << 17, n_leaders=8, calls=20):
    g = np.random.default_rng(7)
    pool = g.choice(np.arange(1 << 24), size=2, replace=False).astype(np.int32)
    keys = g.choice(pool, size=n, p=[0.7, 0.3]).astype(np.int32)   # one key per command
    off = np.arange(n + 1, dtype=np.int32)
    lead = g.integers(0, n_leaders, n).astype(np.int32)
    ids = np.arange(n, dtype=np.int32)
    sets = (g.random(n) < 0.4).astype(np.uint8)
    out = np.zeros((n, n_leaders), np.int32)
    times = []
    for _ in range(reps):
        ci = ConflictIndex(n_leaders, key_capacity=1 << 12, max_commands=n, max_keys=n)
        for c in range(calls + 2):                 # the first two calls warm up
            t = time.perf_counter()
            ci._host_call(ci._L.fpx_conflict_index_batch, lead.ctypes.data, ids.ctypes.data, sets.ctypes.data,
                          off.ctypes.data, keys.ctypes.data, n, ConflictIndex.QUERY_THEN_PUT, out.ctypes.data)
            if c >= 2:
                times.append(time.perf_counter() - t)
        ci.close()
    return {"commands": n, "leaders": n_leaders, "batch_call_ms_median": float(np.median(times)) * 1e3,
            "batch_call_ms_best": min(times) * 1e3}


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    print("card, power limit:", card(), flush=True)
    print(json.dumps({"cfg4": cfg4(a.reps), "chain": chain(a.reps), "conflict": conflict(a.reps)}))
