"""BASELINE cfg4 (EPaxos, 5 replicas, 20 % conflicts, 2^20 instances) as seen by replica 0: device time of
each handler batch on DEVICE-resident rows (fpx_epaxos_*_dev, CUDA events on the handle's stream, best of 3
fresh replicas), with the algorithmic bytes per message next to it.
    python profiles/bench_epaxos_cfg4.py"""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import peaks  # noqa: E402
from frankenpaxos_b200 import traces as T  # noqa: E402
from frankenpaxos_b200.epaxos import EpaxosReplica  # noqa: E402


def run(N=1 << 20, f=2, reps=3):
    n = 2 * f + 1
    lead, pa, ok = T.epaxos_cfg4(0, f=f, n_instances=N, me=0)
    dev = torch.device("cuda", 0)
    td = lambda x: torch.from_numpy(np.ascontiguousarray(x, dtype=np.int32)).to(dev)
    d_lead, d_pa, d_ok = td(lead), td(pa), td(ok)
    d_rep = torch.zeros((len(pa), 4 + n), dtype=torch.int32, device=dev)
    d_ev = torch.zeros((len(ok), 2 + n), dtype=torch.int32, device=dev)
    best = {}
    ev_counts = None
    for _ in range(reps):
        eng = EpaxosReplica(f, 0, N // n + 2, max_batch=1 << 20)
        ext = torch.cuda.ExternalStream(eng.stream, device=dev)
        e = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        e[0].record(ext); eng.lead_dev(d_lead.data_ptr(), len(lead))
        e[1].record(ext); eng.preaccept_dev(d_pa.data_ptr(), len(pa), d_rep.data_ptr())
        e[2].record(ext); eng.preacceptok_dev(d_ok.data_ptr(), len(ok), d_ev.data_ptr())
        e[3].record(ext)
        eng.sync()
        for name, j in (("lead", 0), ("preaccept", 1), ("preacceptok", 2)):
            ms = e[j].elapsed_time(e[j + 1])
            best[name] = min(best.get(name, 1e9), ms)
        ev = d_ev.cpu().numpy()
        ev_counts = (int((ev[:, 0] == 1).sum()), int((ev[:, 0] == 2).sum()))
        eng.close()
    msgs = {"lead": len(lead), "preaccept": len(pa), "preacceptok": len(ok)}
    # algorithmic bytes per message: input row + reply row + cmdLog row read+write (+ leader row for lead / responses)
    alg = {"lead": 4 * (8 + n) + 64 + 512, "preaccept": 4 * (6 + 2 * n) + 4 * (4 + n) + 2 * 64,
           "preacceptok": 4 * (6 + n) + 4 * (2 + n) + 4 * 10 + 64}
    peak, _ = peaks()
    return {"config": "cfg4: EPaxos n=5 f=2, 2^20 instances, BernoulliSingleKeyWorkload(0.2), replica 0's view, device-resident rows",
            "fast_commits": ev_counts[0], "slow_paths": ev_counts[1],
            "calls": {k: {"messages": msgs[k], "kernel_ms": best[k], "messages_per_s": msgs[k] / (best[k] * 1e-3),
                          "algorithmic_bytes_per_message": alg[k],
                          "GB/s": alg[k] * msgs[k] / (best[k] * 1e-3) / 1e9,
                          "frac_of_hbm_peak": alg[k] * msgs[k] / (best[k] * 1e-3) / 1e9 / peak} for k in best}}


if __name__ == "__main__":
    print(json.dumps(run()))
