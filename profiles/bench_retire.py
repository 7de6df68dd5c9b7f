"""Cost of fpx_retire_below at cfg2 size (2^20 slots per window, 5 acceptors), on one GPU.

  steady     retire one executed window while the next 2^20 slots are in flight; no secondary key was ever
             armed, so the call is one recycle_kernel launch
  rebuild    the same after a leader change re-armed 2^19 of the in-flight slots in a new round: 2^20 secondary
             keys in a 2^21-entry overflow table, all of them live, so the rebuild keeps every one
  drop       the next retire, which drops those 2^20 keys (their slots are now retired)

Each time is a host clock around retire_below and the stream synchronise after it (the call itself starts with
one), the median of `--reps` engines.  Prints the card name and power limit first, then one JSON line.
    python profiles/bench_retire.py [--reps 5]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

W = 1 << 20


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def window(e, T, cfg, k, round_=0):
    a, p, b = T.workload(900 + k, cfg, W, slot0=k * W, round_=round_)
    e.proxyleader_arm(a)
    ob, _ = e.acceptor_phase2a(p)
    e.replica_chosen(e.proxyleader_phase2b(ob[np.random.default_rng(k).permutation(len(ob))]))
    assert e.chosen_watermark() == (k + 1) * W          # retire_below checks against the published watermark


def timed_retire(e, slot):
    t0 = time.perf_counter()
    e.retire_below(slot)
    e.sync()
    return (time.perf_counter() - t0) * 1e6


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch
    from frankenpaxos_b200 import Engine
    from frankenpaxos_b200 import traces as T
    if not torch.cuda.is_available():
        sys.exit("bench_retire.py: no CUDA device")
    print("card, power limit:", card(), flush=True)
    cfg, _ = T.config_by_name("cfg2")
    res = {"steady_us": [], "rebuild_us": [], "drop_us": [], "launches": []}
    for rep in range(args.reps):
        e = Engine(slot_capacity=2 * W, overflow_capacity=2 * W, max_batch=3 * W, **cfg)
        window(e, T, cfg, 0)
        window(e, T, cfg, 1)
        c0 = e.launch_count
        res["steady_us"].append(timed_retire(e, W))                   # window 0 goes, window 1 stays
        steady_launches = e.launch_count - c0
        window(e, T, cfg, 2)
        half = T.arms(np.arange(2 * W, 2 * W + W // 2, dtype=np.int32), 1, np.arange(W // 2, dtype=np.int32))
        e.proxyleader_arm(half)                                        # leader change: 2^20 keys in the table
        c0 = e.launch_count
        res["rebuild_us"].append(timed_retire(e, 2 * W))              # window 1 goes, the keys stay
        rebuild_launches = e.launch_count - c0
        window(e, T, cfg, 3)
        res["drop_us"].append(timed_retire(e, 3 * W))                 # window 2 and its keys go
        res["launches"].append((steady_launches, rebuild_launches))
        e.close()
    med = {k: float(np.median(v)) for k, v in res.items() if k != "launches"}
    print(json.dumps({"card": card(), "median_us": med, "all_us": {k: v for k, v in res.items() if k != "launches"},
                      "launches_steady_rebuild": res["launches"][0]}))


if __name__ == "__main__":
    main()
