"""Device time of a MultiPaxos leader change from bytes at cfg2 (f = 2, one group of five, 2^20 slots in flight):
  acceptors  5 Phase1a -> 5 Phase1b of about 0.9 * 2^20 infos each, values of 0-200 bytes (fpx_acceptor_phase1a_wire;
             the call reads its info count back once, so its time is a host clock around work that ends in a sync);
  leader     3 of those Phase1bs -> the 2^20 re-proposed records (fpx_leader_phase1b_wire), and its entry walk
             (p1_walk_kernel) on its own from a torch.profiler pass run separately;
  phase2a    the 2^20 ProxyLeaderInbound{phase2a} messages (fpx_wire_encode_phase2a).
CUDA events on the engine's stream, inputs resident in HBM, L2 flushed by a 256 MB read between rounds, 2 warm-up +
5 timed rounds (mean).  The single-threaded CPU oracle (tests/wire_phase1_oracle.cc) is timed on the same inputs as
a CPU baseline.  The card's name and power limit are read in the same run.
    python profiles/bench_wire_phase1.py"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import wire_phase1_oracle as O  # noqa: E402
from frankenpaxos_b200 import VALUE_NOOP, WIRE_ACCEPTOR_INBOUND, Engine, dst  # noqa: E402

assert torch.cuda.is_available(), "this measurement needs the GPU"
dev = torch.device("cuda", 0)
S = 1 << 20
g = np.random.Generator(np.random.PCG64(0))
eng = Engine(2, 1, 5, slot_capacity=1 << 21, max_batch=1 << 23)
ext = torch.cuda.ExternalStream(eng.stream, device=dev)
flush = torch.zeros(256 << 20, dtype=torch.uint8, device=dev)
flush_sink = torch.zeros((), dtype=torch.int64, device=dev)


def timed(fn, rounds=5, warm=2, host=False):
    ms = []
    for r in range(warm + rounds):
        flush_sink.copy_(flush.view(torch.int32).sum())
        torch.cuda.synchronize()
        if host:
            t = time.perf_counter(); fn(); eng.sync(); ms_r = (time.perf_counter() - t) * 1e3
        else:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(ext); fn(); e1.record(ext)
            torch.cuda.synchronize()
            ms_r = e0.elapsed_time(e1)
        if r >= warm:
            ms.append(ms_r)
    return {"ms": float(np.mean(ms)), "ms_std": float(np.std(ms))}


# votes of all five acceptors, 90% of the slots each, values 0-200 bytes
lens = g.integers(0, 201, 4096)
voffs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
arena = g.integers(0, 256, int(voffs[-1]), dtype=np.uint8)
for c in range(5):
    voted = np.nonzero(g.random(S) < 0.9)[0].astype(np.int32)
    p = np.zeros(len(voted), O.P2A)
    p["slot"], p["round"], p["dst"] = voted, g.integers(0, 7, len(voted)), dst(0, c)
    p["value_id"] = np.where(g.random(len(voted)) < 0.05, VALUE_NOOP, g.integers(0, 4096, len(voted)))
    eng.acceptor_phase2a(p)
body = b"\x08\x07\x10\x00"
req, roffs = O.pack([b"\x0a\x04" + body] * 5)
kind, recs = eng.wire_decode_inbound(WIRE_ACCEPTOR_INBOUND, req, roffs)
recs = recs.copy()
recs["a"] = dst(0, np.arange(5))
p1b, p1offs = eng.acceptor_phase1a_wire(req, kind, recs, arena, voffs)     # rounds -> 7; the timed calls repeat it
res = {"phase1b_bytes": int(p1offs[5])}
t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
d_req, d_kind, d_recs = t(req), t(kind), t(recs.view(np.int32).reshape(-1, 4))
d_arena, d_voffs = t(np.concatenate([arena, np.zeros(64, np.uint8)])), t(voffs)
cap = int(p1offs[5]) + 64
d_p1b, d_p1offs = torch.zeros(cap, dtype=torch.uint8, device=dev), torch.zeros(6, dtype=torch.int32, device=dev)
torch.cuda.synchronize()
res["acceptors_phase1b_encode_5"] = timed(lambda: eng.acceptor_phase1a_wire_dev(
    d_req.data_ptr(), len(req), d_kind.data_ptr(), d_recs.data_ptr(), 5, d_arena.data_ptr(), d_voffs.data_ptr(),
    len(voffs) - 1, d_p1b.data_ptr(), cap, d_p1offs.data_ptr()), host=True)
# the leader: the first three Phase1bs
n3 = int(p1offs[3])
d_buf = torch.cat([d_p1b[:n3], torch.zeros(64, dtype=torch.uint8, device=dev)]).contiguous()
d_offs = t(p1offs[:4])
d_out, d_sp, d_res = (torch.zeros(s, dtype=torch.int32, device=dev) for s in ((S, 4), (S, 2), (3,)))
torch.cuda.synchronize()
lead = lambda: eng.leader_phase1b_wire_dev(7, 0, d_buf.data_ptr(), n3, d_offs.data_ptr(), 3, 0, d_out.data_ptr(),
                                           d_sp.data_ptr(), S, d_res.data_ptr())
res["leader_phase1b_3"] = timed(lead)
eng.sync()
complete, max_slot, n_out = d_res.cpu().tolist()
assert complete == 2 and n_out == max_slot + 1
with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    for _ in range(3):
        lead(); eng.sync()
walk = [e for e in prof.key_averages() if "p1_walk_kernel" in e.key]
res["leader_entry_walk"] = {"ms": walk[0].device_time / 1e3 if walk else None, "source": "torch.profiler, mean of 3"}
out_cap = int(n3 + 32 * n_out) + 64
d_p2a, d_p2offs = torch.zeros(out_cap, dtype=torch.uint8, device=dev), torch.zeros(n_out + 1, dtype=torch.int32, device=dev)
torch.cuda.synchronize()
res["phase2a_encode"] = timed(lambda: eng.wire_encode_phase2a_dev(
    d_out.data_ptr(), n_out, d_buf.data_ptr(), n3, d_sp.data_ptr(), n_out, 0, d_p2a.data_ptr(), out_cap,
    d_p2offs.data_ptr()))
eng.sync()
res["phase2a_bytes"] = int(d_p2offs[n_out].item())
# CPU baseline: the single-threaded oracle on the same bytes
buf3, offs3 = O.pack(O.split(p1b, p1offs)[:3])
t0 = time.perf_counter()
o = O.leader_phase1b(2, 1, 5, 0, 7, 0, buf3, offs3, 0, S)
res["cpu_baseline_oracle_leader_phase1b_3_ms"] = (time.perf_counter() - t0) * 1e3
t0 = time.perf_counter()
O.encode_phase2a(o[4], buf3, o[5], 0)
res["cpu_baseline_oracle_phase2a_encode_ms"] = (time.perf_counter() - t0) * 1e3
res["cpu_baseline_note"] = "single-threaded C++ oracle (test infrastructure), not the reference JVM"
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                   text=True).stdout.strip()
res["card"] = q
print(json.dumps(res, indent=1))
