"""Device time of the MultiPaxos read path (fpx_reads_*) at cfg2 size (f = 2, 5 acceptors), on one GPU.

  tally      3 x 2^20 shuffled MaxSlotReplies (3 acceptors of 5 per read) completing 2^20 Client reads
  replica    one batch of 2^20 read requests, every one deferred (slots ahead of W)
  advance    the advance that releases those 2^20 reads

Each is the _dev form between two CUDA events on the engine's stream, median of `--reps` runs; inputs and
outputs stay on the device, nothing is copied.  The reads are re-opened (tally) or the handle is fresh
(replica, advance) before each run, outside the timed window.  Prints the card name and power limit first,
then one JSON line.
    python profiles/bench_reads.py [--reps 10]"""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from profiles.bench_retire import card  # noqa: E402

N = 1 << 20


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    import torch
    from frankenpaxos_b200 import Engine, Reads, READS_CLIENT, MAX_SLOT_REPLY, READ_REQUEST
    from frankenpaxos_b200 import traces as T
    if not torch.cuda.is_available():
        sys.exit("bench_reads.py: no CUDA device")
    print("card, power limit:", card(), flush=True)
    cfg, _ = T.config_by_name("cfg2")
    dev = torch.device("cuda", 0)
    g = np.random.default_rng(1)
    rec = np.zeros(3 * N, MAX_SLOT_REPLY)
    rec["key"] = np.repeat(np.arange(N), 3)
    rec["id"] = 1
    acc = np.argsort(g.random((N, 5)), axis=1)[:, :3].reshape(-1)
    rec["voter"] = acc
    rec["slot"] = g.integers(0, 1 << 24, 3 * N)
    rec = rec[g.permutation(3 * N)]
    req = np.zeros(N, READ_REQUEST)
    req["slot"] = g.integers(0, 1 << 20, N)
    req["handle"] = np.arange(N)
    d_rec = torch.from_numpy(rec.view(np.int32).reshape(-1, 4).copy()).to(dev)
    d_req = torch.from_numpy(req.view(np.int32).reshape(-1, 2).copy()).to(dev)
    d_out = torch.zeros((3 * N, 4), dtype=torch.int32, device=dev)
    d_w = torch.full((1,), 1 << 20, dtype=torch.int32, device=dev)
    keys, ids = np.arange(N, dtype=np.int32), np.ones(N, np.int32)

    e = Engine(slot_capacity=1 << 12, max_batch=1 << 12, **cfg)
    stream = torch.cuda.ExternalStream(e.stream)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

    def timed(fn):
        ev[0].record(stream)
        fn()
        ev[1].record(stream)
        ev[1].synchronize()
        return ev[0].elapsed_time(ev[1]) * 1e3

    res = {"tally_us": [], "replica_us": [], "advance_us": []}
    counts = {}
    r = Reads(e, READS_CLIENT, key_capacity=N, pending_capacity=N, max_batch=3 * N)
    for rep in range(args.reps + 1):                    # run 0 warms every kernel up
        ids += 1
        r.open(keys, ids)
        d_rec[:, 1] = int(ids[0])
        torch.cuda.synchronize()
        t = timed(lambda: r.max_slot_replies_dev(d_rec.data_ptr(), 3 * N, d_out.data_ptr()))
        counts["completed"] = r.sync().n_slots
        if rep:
            res["tally_us"].append(t)
    r.close()
    for rep in range(args.reps + 1):
        r = Reads(e, READS_CLIENT, key_capacity=1, pending_capacity=N, max_batch=N)
        t1 = timed(lambda: r.replica_dev(d_req.data_ptr(), N, d_out.data_ptr()))
        s = r.sync()
        t2 = timed(lambda: r.advance_dev(d_w.data_ptr(), d_out.data_ptr()))
        s2 = r.sync()
        counts["pending"], counts["released"] = s.n_pending, s2.n_released
        if rep:
            res["replica_us"].append(t1); res["advance_us"].append(t2)
        r.close()
    e.close()
    med = {k: float(np.median(v)) for k, v in res.items()}
    print(json.dumps({"card": card(), "median_us": med, "all_us": res, "counts": counts}))


if __name__ == "__main__":
    main()
