"""Throughput of BASELINE cfg4's dep-set union kernel (dense, n=5 replicas, R=4 sets per
instance, 2^22 instances per launch so that inputs exceed L2): algorithmic bytes
4n(R+1) = 100 B/instance against the HBM peak of bench.py.
    python profiles/bench_depset_union.py"""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import peaks  # noqa: E402
from frankenpaxos_b200.epaxos import depset_union_dense_dev  # noqa: E402

G, R, n = 1 << 22, 4, 5
bufs = [torch.randint(0, 1 << 20, (G, R, n), dtype=torch.int32, device="cuda") for _ in range(3)]
out = torch.empty((G, n), dtype=torch.int32, device="cuda")
for b in bufs:
    depset_union_dense_dev(b.data_ptr(), G, R, n, out.data_ptr())
torch.cuda.synchronize()
ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
K = 30
ev[0].record()
for k in range(K):
    depset_union_dense_dev(bufs[k % 3].data_ptr(), G, R, n, out.data_ptr())
ev[1].record()
torch.cuda.synchronize()
ms = ev[0].elapsed_time(ev[1]) / K
peak, _ = peaks()
gbs = G * 4 * n * (R + 1) / (ms * 1e-3) / 1e9
print(json.dumps({"kernel": "depset_union_dense_kernel", "instances_per_launch": G, "ms": ms,
                  "instances_per_s": G / (ms * 1e-3), "GB/s": gbs, "frac_of_hbm_peak": gbs / peak}))
