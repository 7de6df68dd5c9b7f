"""Device time of a compartmentalized Mencius leader change from bytes (f = 2, LG = 3 leader groups of AG = 2 acceptor
groups of five; the failing leader group 1 holds 2^20 slots in flight, values of 0-200 bytes):
  acceptors  the f+1 x AG = 6 Phase1a -> 6 Phase1bs of about 0.9 * 2^19 infos each, half of them noop-range votes
             (fpx_mencius_acceptor_phase1a_wire; the call reads its info count back once, so its time is a host clock
             around work that ends in a sync);
  leader     those 6 Phase1bs -> the 2^20 re-proposed records of leader group 1 (fpx_mencius_leader_phase1b_wire);
  phase2a    the 2^20 ProxyLeaderInbound{phase2a = 2} messages (fpx_wire_encode_mencius_phase2a).
CUDA events on the engine's stream, inputs resident in HBM, L2 flushed by a 256 MB read between rounds, 2 warm-up +
5 timed rounds (mean).  The single-threaded CPU oracle (tests/wire_mencius_phase1_oracle.cc) is timed on the same
inputs as a CPU baseline.  The card's name and power limit are read in the same run.
    python profiles/bench_wire_mencius_phase1.py"""
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
import wire_mencius_phase1_oracle as O  # noqa: E402
from frankenpaxos_b200 import MENCIUS, VALUE_NOOP, WIRE_MENCIUS_ACCEPTOR_INBOUND, Engine, dst  # noqa: E402

assert torch.cuda.is_available(), "this measurement needs the GPU"
dev = torch.device("cuda", 0)
F, LG, AG, LEADER = 2, 3, 2, 1
N = 1 << 20                                   # slots of leader group 1 in flight
S = LG * N
g = np.random.Generator(np.random.PCG64(0))
eng = Engine(F, AG, 2 * F + 1, protocol=MENCIUS, num_leader_groups=LG, slot_capacity=S, max_batch=1 << 23)
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


# leader group 1's slots: Phase2a votes of acceptors 0-2 on 90% of the lower half, noop ranges over the upper half
lens = g.integers(0, 201, 4096)
voffs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
arena = g.integers(0, 256, int(voffs[-1]), dtype=np.uint8)
mine = np.arange(LEADER, S // 2, LG, dtype=np.int32)
for c in range(F + 1):
    voted = mine[g.random(len(mine)) < 0.9]
    p = np.zeros(len(voted), O.P2A)
    p["slot"], p["round"] = voted, g.integers(0, 7, len(voted))
    p["dst"] = dst(LEADER * AG + (voted // LG) % AG, c)
    p["value_id"] = np.where(g.random(len(voted)) < 0.05, VALUE_NOOP, g.integers(0, 4096, len(voted)))
    eng.acceptor_phase2a(p)
ranges = np.array([(s, s + 3 * 4096, 6, int(dst(LEADER * AG + ag, c))) for s in range(S // 2 + LEADER - 1, S - 3 * 4096, 3 * 4096)
                   for ag in range(AG) for c in range(F + 1)], O.P2A_RANGE)
ranges["slot_start"] += (LEADER - ranges["slot_start"] % LG) % LG
eng.mencius_acceptor_noop_range(ranges)
raw = b"\x0a\x04\x08\x07\x10\x00"                 # AcceptorInbound{phase1a{round 7, chosen_watermark 0}}
req, roffs = O.pack([raw] * (AG * (F + 1)))
kind, recs = eng.wire_decode_inbound(WIRE_MENCIUS_ACCEPTOR_INBOUND, req, roffs)
recs = recs.copy()
recs["a"] = dst(LEADER * AG + np.repeat(np.arange(AG), F + 1), np.tile(np.arange(F + 1), AG))
n_msgs = len(recs)
p1b, p1offs = eng.mencius_acceptor_phase1a_wire(req, kind, recs, arena, voffs)   # rounds -> 7; timed calls repeat it
res = {"phase1b_bytes": int(p1offs[n_msgs])}
t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
d_req, d_kind, d_recs = t(req), t(kind), t(recs.view(np.int32).reshape(-1, 4))
d_arena, d_voffs = t(np.concatenate([arena, np.zeros(64, np.uint8)])), t(voffs)
cap = int(p1offs[n_msgs]) + 64
d_p1b, d_p1offs = torch.zeros(cap, dtype=torch.uint8, device=dev), torch.zeros(n_msgs + 1, dtype=torch.int32, device=dev)
torch.cuda.synchronize()
res["acceptors_phase1b_encode_6"] = timed(lambda: eng.mencius_acceptor_phase1a_wire_dev(
    d_req.data_ptr(), len(req), d_kind.data_ptr(), d_recs.data_ptr(), n_msgs, d_arena.data_ptr(), d_voffs.data_ptr(),
    len(voffs) - 1, d_p1b.data_ptr(), cap, d_p1offs.data_ptr()), host=True)
nb = int(p1offs[n_msgs])
d_buf = torch.cat([d_p1b[:nb], torch.zeros(64, dtype=torch.uint8, device=dev)]).contiguous()
d_offs = t(p1offs)
d_out, d_sp, d_res = (torch.zeros(s, dtype=torch.int32, device=dev) for s in ((N, 4), (N, 2), (4,)))
torch.cuda.synchronize()
res["leader_phase1b_6"] = timed(lambda: eng.mencius_leader_phase1b_wire_dev(
    LEADER, 7, 0, -1, d_buf.data_ptr(), nb, d_offs.data_ptr(), n_msgs, 0, d_out.data_ptr(), d_sp.data_ptr(), N,
    d_res.data_ptr()))
eng.sync()
complete, max_slot, n_out, next_slot = d_res.cpu().tolist()
assert complete == n_msgs - 1 and n_out > 0.99 * N and next_slot == max_slot + LG
res["records"] = n_out
out_cap = int(nb + 32 * n_out) + 64
d_p2a, d_p2offs = torch.zeros(out_cap, dtype=torch.uint8, device=dev), torch.zeros(n_out + 1, dtype=torch.int32, device=dev)
torch.cuda.synchronize()
res["phase2a_encode"] = timed(lambda: eng.wire_encode_mencius_phase2a_dev(
    d_out.data_ptr(), n_out, d_buf.data_ptr(), nb, d_sp.data_ptr(), n_out, 0, d_p2a.data_ptr(), out_cap,
    d_p2offs.data_ptr()))
eng.sync()
res["phase2a_bytes"] = int(d_p2offs[n_out].item())
# CPU baseline: the single-threaded oracle on the same bytes
buf, offs = O.pack(O.split(p1b, p1offs))
t0 = time.perf_counter()
o = O.leader_phase1b(F, LG, AG, 2 * F + 1, LEADER, 7, 0, buf, offs, -1, 0, N)
res["cpu_baseline_oracle_leader_phase1b_6_ms"] = (time.perf_counter() - t0) * 1e3
assert o[0] == 0 and len(o[5]) == n_out
res["cpu_baseline_note"] = "single-threaded C++ oracle (test infrastructure), not the reference JVM"
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                   text=True).stdout.strip()
res["card"] = q
print(json.dumps(res, indent=1))
