"""Device time of Compartmentalized Mencius' replica path from protobuf bytes, and of its noop-range encoders.
  mixed     2^20 ReplicaInbound messages, about 1 % ChosenNoopRange (20 slots each) interleaved with the Chosens: decoded by
            fpx_wire_decode_mencius_replica_inbound_dev, then applied in one fpx_mencius_replica_inbound_dev call.
  per_type  the same batch the way it went before: decoded, then cut at every change of message type, the Chosen runs
            through fpx_replica_chosen_dev and the ranges through fpx_mencius_replica_chosen_range (host records, one
            host round trip per run).
  encode    65535 Phase2bNoopRange and 65535 ChosenNoopRange records (one range call's worth) into bytes.
CUDA events on the engine's stream, a fresh log per round, L2 flushed by a 256 MB read between rounds, 3 warm-up +
10 timed rounds (mean).  The card's name and power limit are read in the same run.
    python profiles/bench_wire_mencius.py"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from frankenpaxos_b200 import CHOSEN_RANGE, MENCIUS, P2B_RANGE, Engine  # noqa: E402

assert torch.cuda.is_available(), "this measurement needs the GPU"
dev = torch.device("cuda", 0)
LG, N = 3, 1 << 20
eng = Engine(1, 1, 3, num_leaders=2, num_replicas=2, slot_capacity=1 << 22, max_batch=N, protocol=MENCIUS,
             num_leader_groups=LG)
ext = torch.cuda.ExternalStream(eng.stream, device=dev)
g = np.random.default_rng(1)


def varint(v):
    out = bytearray()
    v &= (1 << 64) - 1
    while v >= 0x80:
        out.append((v & 0x7f) | 0x80); v >>= 7
    out.append(v)
    return bytes(out)


# slots 0 .. N-1 in a random order, a range every ~100 messages standing for 20 slots of a lagging leader group.  The
# ranges start in distinct 64-slot blocks, so no two of them overlap and one mixed call takes the whole batch.
is_range = g.random(N) < 0.01
slots = g.permutation(N).astype(np.int64)
blocks = g.permutation(N // 64)[:int(is_range.sum())]
slots[is_range] = blocks * 64 + g.integers(0, LG, size=len(blocks))
msgs = []
for i in range(N):
    s = int(slots[i])
    if is_range[i]:
        body = b"\x08" + varint(s) + b"\x10" + varint(s + 20 * LG)
        msgs.append(b"\x12" + varint(len(body)) + body)            # ReplicaInbound{chosen_noop_range}
    else:
        body = b"\x08" + varint(s) + b"\x12\x02\x12\x00"           # Chosen{slot, CommandBatchOrNoop{noop}}
        msgs.append(b"\x0a" + varint(len(body)) + body)
offs = np.zeros(N + 1, dtype=np.int32)
offs[1:] = np.cumsum([len(m) for m in msgs])
buf = np.frombuffer(b"".join(msgs) + b"\0" * 64, dtype=np.uint8)
d_buf = torch.from_numpy(buf.copy()).to(dev)
d_offs = torch.from_numpy(offs).to(dev)
d_kind = torch.empty(N, dtype=torch.int32, device=dev)
d_recs = torch.empty((N, 4), dtype=torch.int32, device=dev)
d_vals = torch.empty((N, 2), dtype=torch.int32, device=dev)
d_split = torch.empty(1, dtype=torch.int32, device=dev)
flush = torch.zeros(256 << 20, dtype=torch.uint8, device=dev)
flush_sink = torch.zeros((), dtype=torch.int64, device=dev)


def timed(fn, rounds=10, warm=3, fresh=True):
    ms = []
    for r in range(warm + rounds):
        if fresh:
            eng.reset()
        flush_sink.copy_(flush.view(torch.int32).sum())   # evict L2 by reading: no dirty lines billed to the kernel
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(ext); fn(); e1.record(ext)
        torch.cuda.synchronize()
        if r >= warm:
            ms.append(e0.elapsed_time(e1))
    return float(np.mean(ms)), float(np.std(ms))


def decode():
    eng.wire_decode_mencius_replica_inbound_dev(d_buf.data_ptr(), d_offs.data_ptr(), N, 0, d_kind.data_ptr(),
                                                d_recs.data_ptr(), d_vals.data_ptr())


def mixed():
    decode()
    eng.mencius_replica_inbound_dev(d_recs.data_ptr(), N, d_split.data_ptr())


dec_ms, dec_sd = timed(decode)
mix_ms, mix_sd = timed(mixed)
eng.sync()
assert int(d_split.item()) == N
log_mixed = eng.snapshot_log(0, N + 40 * LG)
wm_mixed = eng.chosen_watermark()

# the per-type path: runs of equal kind, in delivery order
kind = d_kind.cpu().numpy()
recs = d_recs.cpu().numpy()
cut = np.flatnonzero(np.diff(kind)) + 1
runs = list(zip(np.r_[0, cut], np.r_[cut, N]))
d_chosen = torch.from_numpy(np.ascontiguousarray(recs[:, [0, 2]])).to(dev)      # fpx_chosen {slot, value_id}
host_ranges = np.ascontiguousarray(recs[:, :2]).view(CHOSEN_RANGE).ravel()


def per_type():
    decode()
    for a, b in runs:
        if kind[a] == 1:
            eng.replica_chosen_dev(d_chosen[a].data_ptr(), int(b - a))
        else:
            eng.mencius_replica_chosen_range(host_ranges[a:b])


pt_ms, pt_sd = timed(per_type, rounds=3, warm=1)
eng.sync()
assert np.array_equal(eng.snapshot_log(0, N + 40 * LG), log_mixed) and eng.chosen_watermark() == wm_mixed

# encoders: one range call's worth of records
K = 65535
p = np.zeros(K, dtype=P2B_RANGE)
p["dst"] = g.integers(0, 3, size=K); p["slot_start"] = g.integers(0, 1 << 22, size=K)
p["slot_end"] = p["slot_start"] + 30 * LG; p["round"] = g.integers(0, 100, size=K)
c = np.zeros(K, dtype=CHOSEN_RANGE)
c["slot_start"], c["slot_end"] = p["slot_start"], p["slot_end"]
d_p = torch.from_numpy(p.view(np.int32).reshape(K, 4)).to(dev)
d_c = torch.from_numpy(c.view(np.int32).reshape(K, 2)).to(dev)
d_out = torch.empty(64 * K + 64, dtype=torch.uint8, device=dev)
d_eoffs = torch.empty(K + 1, dtype=torch.int32, device=dev)
p2b_ms, p2b_sd = timed(lambda: eng.wire_encode_mencius_phase2b_range_dev(d_p.data_ptr(), K, d_out.data_ptr(), 64 * K,
                                                                          d_eoffs.data_ptr()), fresh=False)
eng.sync()
p2b_total = int(d_eoffs[K].item())
cr_ms, cr_sd = timed(lambda: eng.wire_encode_mencius_chosen_range_dev(d_c.data_ptr(), K, d_out.data_ptr(), 64 * K,
                                                                       d_eoffs.data_ptr()), fresh=False)
eng.sync()
cr_total = int(d_eoffs[K].item())
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
print(json.dumps({
    "workload": f"2^20 ReplicaInbound, {int(is_range.sum())} ChosenNoopRange of 20 slots interleaved, LG = {LG}",
    "wire_bytes": int(offs[-1]), "type_runs": len(runs),
    "decode": {"ms": dec_ms, "ms_std": dec_sd, "messages_per_s": N / (dec_ms * 1e-3)},
    "decode_and_mixed_apply": {"ms": mix_ms, "ms_std": mix_sd, "messages_per_s": N / (mix_ms * 1e-3),
                               "calls": "decode + fpx_mencius_replica_inbound_dev"},
    "decode_and_per_type_apply": {"ms": pt_ms, "ms_std": pt_sd, "messages_per_s": N / (pt_ms * 1e-3),
                                  "calls": "decode + one fpx_replica_chosen_dev / fpx_mencius_replica_chosen_range per run",
                                  "rounds": 3},
    "encode_phase2b_noop_range": {"records": K, "bytes": p2b_total, "ms": p2b_ms, "ms_std": p2b_sd},
    "encode_chosen_noop_range": {"records": K, "bytes": cr_total, "ms": cr_ms, "ms_std": cr_sd},
    "device": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip(), "l2": "256 MB buffer read between rounds"}))
eng.close()
