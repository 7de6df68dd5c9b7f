"""A/B of the device-resident cfg2 step inside one process: kernel order, tally path,
per-kernel CUDA-event times and the in-kernel phase marks of the last step.

  python profiles/exp_step.py [--steps 12] [--variants default,acc_first,exact,...]
"""
import argparse
import ctypes
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=12)
ap.add_argument("--variants", default="default,acc_first,exact,default,acc_first")
ap.add_argument("--out", default="")
ap.add_argument("--old-lib", action="store_true", help="time the round-1 build (profiles/_r1/libfpx.so) instead")
ap.add_argument("--lib", default="", help="time another build of libfpx.so (tuning variants under profiles/_var/)")
args = ap.parse_args()
if args.old_lib:
    os.environ["FPX_LIB_OVERRIDE"] = os.path.join(ROOT, "profiles", "_r1", "libfpx.so")
if args.lib:
    os.environ["FPX_LIB_OVERRIDE"] = os.path.join(ROOT, args.lib)

import bench  # noqa: E402
from frankenpaxos_b200 import Engine, traces as T  # noqa: E402

cfg = bench.CFG
n = 1 << 20
S = args.steps + 3
dev = torch.device("cuda")


def td(x):
    return torch.from_numpy(x.view(np.int32).reshape(len(x), -1)).to(dev)


base = [T.workload(b, cfg, n) for b in range(4)]
outp = torch.empty((3 * n, 4), dtype=torch.int32, device=dev)
outn = torch.empty((3 * n, 2), dtype=torch.int32, device=dev)
outc = torch.empty((3 * n, 2), dtype=torch.int32, device=dev)
wm = torch.zeros(1, dtype=torch.int32, device=dev)
results = {}
for variant in args.variants.split(","):
    eng = Engine(slot_capacity=S * n, max_batch=3 * n, overflow_capacity=1 << 10, **cfg)
    L = eng._L
    L.fpx_debug_phase_times.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    ext = torch.cuda.ExternalStream(eng.stream, device=dev)
    if not args.old_lib:
        eng._check(L.fpx_debug_set_tally_path(eng.h, sum(bit for tok, bit in (("exact", 2), ("nored", 4)) if tok in variant.split("_"))))
    for tok in variant.split("_"):
        if tok.startswith("seg"):      # segN: every acceptor launch cut into N pipelined segments (default: from the L2 size)
            eng.set_acceptor_segments(int(tok[3:]))
    flush = torch.empty(1 << 28, dtype=torch.uint8, device=dev) if "flush" in variant else None
    ins = []
    for s in range(S):
        a, p, b = base[s % 4]
        def rb(r):
            o = r.copy(); o["slot"] = o["slot"] + s * n; return o
        ins.append((td(rb(a)), td(rb(p)), td(rb(b))))
    torch.cuda.synchronize()
    names = ["arm", "acceptor", "tally", "replica", "watermark"]
    order = ["acceptor", "arm", "tally", "replica", "watermark"] if "accfirst" in variant.split("_") else names
    evs = [[torch.cuda.Event(enable_timing=True) for _ in range(6)] for _ in range(S)]

    def run(which, s):
        da, dp, db = ins[s]
        if which == "arm": eng.proxyleader_arm_dev(da.data_ptr(), n)
        elif which == "acceptor": eng.acceptor_phase2a_dev(dp.data_ptr(), 3 * n, outp.data_ptr(), outn.data_ptr())
        elif which == "tally":
            if flush is not None:      # read 256 MB: every dirty line of the earlier kernels is written back first
                with torch.cuda.stream(ext):
                    flush.view(torch.int64).sum()
                evs[s][order.index("tally")].record(ext)
            eng.proxyleader_phase2b_dev(db.data_ptr(), 3 * n, outc.data_ptr())
        elif which == "replica": eng.replica_chosen_last_dev(outc.data_ptr())
        else: eng.chosen_watermark_dev(wm.data_ptr())

    fused = "step" in variant.split("_")
    noev = "noev" in variant.split("_")
    import time
    t_host0 = time.perf_counter()
    for s in range(S):
        if s == 3 or not noev:
            evs[s][0].record(ext)
        if fused and noev:
            da, dp, db = ins[s]
            eng.step_dev(da.data_ptr(), n, dp.data_ptr(), 3 * n, outp.data_ptr(), outn.data_ptr(), db.data_ptr(), 3 * n,
                         outc.data_ptr(), wm.data_ptr(), ring_slot=-1)
            if s == S - 1:
                evs[s][5].record(ext)
            continue
        if fused:                      # fpx_step_dev: acceptor, arm, tally + replica + watermark in one kernel
            da, dp, db = ins[s]
            eng.step_dev(da.data_ptr(), n, dp.data_ptr(), 3 * n, outp.data_ptr(), outn.data_ptr(), db.data_ptr(), 3 * n,
                         outc.data_ptr(), wm.data_ptr(), ring_slot=s)
            for j in range(5):
                evs[s][j + 1].record(ext)
            continue
        for j, which in enumerate(order):
            run(which, s)
            evs[s][j + 1].record(ext)
    t_host = (time.perf_counter() - t_host0) / S * 1e6
    r = eng.sync()
    if "nored" not in variant:
        assert r.status == 0 and r.n_chosen == n and r.watermark == S * n, (r.status, r.n_chosen, r.watermark)
    step = evs[3][0].elapsed_time(evs[S - 1][5]) * 1e3 / (S - 3)
    per = {} if noev else {which: float(np.mean([evs[s][j].elapsed_time(evs[s][j + 1]) for s in range(3, S)])) * 1e3
                           for j, which in enumerate(order)}
    if noev:
        per = {}
    elif fused:
        ms = np.array([eng.step_kernel_ms(s) for s in range(3, S)])
        per = {"acceptor": float(ms[:, 0].mean()) * 1e3, "tally+replica+wm": float(ms[:, 1].mean()) * 1e3}
        per["arm"] = step - sum(per.values())
    ta = (ctypes.c_ulonglong * 8)(); tt = (ctypes.c_ulonglong * 8)()
    L.fpx_debug_phase_times(eng.h, ta, tt)
    tt = np.array(tt[:8], dtype=np.int64)
    ta = np.array(ta[:6], dtype=np.int64)
    res = {"step_us": step, "host_enqueue_us_per_step": t_host, "kernels_us": per, "sum_kernels_us": sum(per.values()),
           "tally_path": "r1" if args.old_lib else eng.last_tally_path,
           "tally_phases_us(A,bar,B,bar,C,bar,D)": (np.diff(tt) / 1e3).round(1).tolist(),
           "acceptor_phases_us(p1,bar,carry,p2,bar)": (np.diff(ta) / 1e3).round(1).tolist()}
    print(variant, json.dumps(res), flush=True)
    results.setdefault(variant, []).append(res)
    eng.close()
    del ins
    torch.cuda.empty_cache()
if args.out:
    json.dump(results, open(args.out, "w"), indent=1)
