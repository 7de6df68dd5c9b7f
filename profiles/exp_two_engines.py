"""Experiment: E slot-residue shard engines on ONE GPU, each on its own stream, the cooperative
kernels capped at k CTAs/SM so that kernels of different engines co-reside (the tally is bound by
L1TEX wavefronts, the acceptor by the memory system: complementary).  Prints slots/s per (E, k).
    python profiles/exp_two_engines.py"""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from frankenpaxos_b200 import Engine  # noqa: E402
from frankenpaxos_b200 import traces as T  # noqa: E402

CFG = dict(f=2, num_acceptor_groups=1, acceptors_per_group=5, flexible=False, num_leaders=3, num_replicas=3)
Q = 3
TOTAL = 1 << 20
K, W = 20, 4
dev = torch.device("cuda", 0)


def run(E, cap, stagger):
    per = TOTAL // E
    nrec = Q * per
    S = K + W
    engs = [Engine(slot_capacity=S * per * E, max_batch=nrec, overflow_capacity=1 << 10, shard_index=j, shard_count=E,
                   **CFG) for j in range(E)]
    for e in engs:
        e.set_coop_ctas_per_sm(cap)
    exts = [torch.cuda.ExternalStream(e.stream, device=dev) for e in engs]
    base = [T.workload(77 + j, CFG, per) for j in range(E)]
    ins = []
    for j in range(E):
        a, p, b = base[j]
        steps = []
        for s in range(S):
            def rb(rec):
                out = rec.copy()
                out["slot"] = ((out["slot"].astype(np.int64) + s * per) * E + j).astype(np.int32)
                return torch.from_numpy(out.view(np.int32).reshape(len(out), -1)).to(dev)
            steps.append((rb(a), rb(p), rb(b)))
        ins.append(steps)
    outs = [(torch.empty((nrec, 4), dtype=torch.int32, device=dev), torch.empty((nrec, 2), dtype=torch.int32, device=dev),
             torch.empty((nrec, 2), dtype=torch.int32, device=dev), torch.zeros(1, dtype=torch.int32, device=dev))
            for _ in range(E)]
    torch.cuda.synchronize()

    def stage(j, s, which):
        e = engs[j]; a, p, b = ins[j][s]; o = outs[j]
        if which == 0: e.proxyleader_arm_dev(a.data_ptr(), per)
        elif which == 1: e.acceptor_phase2a_dev(p.data_ptr(), nrec, o[0].data_ptr(), o[1].data_ptr())
        elif which == 2: e.proxyleader_phase2b_dev(b.data_ptr(), nrec, o[2].data_ptr())
        else:
            e.replica_chosen_last_dev(o[2].data_ptr()); e.chosen_watermark_dev(o[3].data_ptr())

    def step(s):
        if stagger:
            # engine j runs stage (t - j): while engine 0 tallies, engine 1 is in its acceptor pass
            for t in range(4 + E - 1):
                for j in range(E):
                    if 0 <= t - j < 4:
                        stage(j, s, t - j)
        else:
            for which in range(4):
                for j in range(E):
                    stage(j, s, which)

    for s in range(W):
        step(s)
    for e in engs:
        r = e.sync(); assert r.n_chosen == per and r.n_nack == 0
    master = torch.cuda.current_stream()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record(master)
    for x in exts: x.wait_event(e0)
    for k in range(K):
        step(W + k)
    for x in exts:
        ev = torch.cuda.Event(); ev.record(x); master.wait_event(ev)
    e1.record(master)
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    for j, e in enumerate(engs):
        r = e.sync(); assert r.status == 0 and r.n_chosen == per and r.watermark == S * per * E + j, (r.watermark,)
        e.close()
    return K * TOTAL / (ms * 1e-3), ms / K * 1e3


res = []
for E, cap, stagger in [(1, 0, False), (2, 0, False), (2, 2, False), (2, 2, True), (2, 1, True), (2, 3, True), (4, 1, True), (4, 2, True), (3, 2, True)]:
    if TOTAL % E:
        continue
    v, us = run(E, cap, stagger)
    res.append({"engines": E, "ctas_per_sm": cap, "staggered": stagger, "slots_per_s": v, "us_per_step": us})
    print(json.dumps(res[-1]), flush=True)
