"""Device time of the vanilla Mencius wire codec on BASELINE cfg5's Phase2 traffic (n = 7 servers, 2^20 slots, so
6 * 2^20 Phase2as and as many replies): encode the dense reply stream of fpx_vm_phase2a (all Phase2b in a fresh log)
into ServerInbound bytes, and decode 6 * 2^20 ServerInbound{phase2b} messages back into records.  CUDA events on the
engine's stream, inputs resident in HBM, L2 flushed by a 256 MB read between rounds, 3 warm-up + 10 timed rounds.
The card's name and power limit are read in the same run.
    python profiles/bench_wire_vm.py"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from frankenpaxos_b200 import P2B, VANILLA_MENCIUS, Engine  # noqa: E402
from frankenpaxos_b200 import traces as T  # noqa: E402

assert torch.cuda.is_available(), "this measurement needs the GPU"
dev = torch.device("cuda", 0)
cfg, n_slots = T.config_by_name("cfg5")
servers = cfg["acceptors_per_group"]
eng = Engine(slot_capacity=n_slots, max_batch=(servers - 1) * n_slots, protocol=VANILLA_MENCIUS, **cfg)
ext = torch.cuda.ExternalStream(eng.stream, device=dev)
_, p, _ = T.vanilla_cfg5(0, cfg["f"], n_slots)
n = len(p)
rep = np.zeros(n, dtype=P2B)                      # what fpx_vm_phase2a answers in a fresh log: kind 0 = Phase2b
rep["acceptor"] = p["dst"]; rep["slot"] = p["slot"]; rep["round"] = p["round"]


def varint_len(v):
    v = v.astype(np.int64)
    out = np.ones(len(v), dtype=np.int64)
    for k in range(1, 5):
        out += (v >= (1 << (7 * k)))
    return np.where(v < 0, 10, out)


# ServerInbound{phase2b = 5 {server_index = 1, slot = 2, round = 3}}: outer tag + length, three tagged int32
msg_len = 2 + 3 + varint_len(rep["acceptor"]) + varint_len(rep["slot"]) + varint_len(rep["round"])
total = int(msg_len.sum())
d_rec = torch.from_numpy(rep.view(np.int32).reshape(n, 4)).to(dev)
cap = 48 * n
d_bytes = torch.empty(cap + 64, dtype=torch.uint8, device=dev)
d_offs = torch.empty(n + 1, dtype=torch.int32, device=dev)
d_kind = torch.empty(n, dtype=torch.int32, device=dev)
d_out = torch.empty((n, 4), dtype=torch.int32, device=dev)
d_sender = torch.empty(n, dtype=torch.int32, device=dev)
d_voffs = torch.zeros(1, dtype=torch.int32, device=dev)     # no values: every reply is a Phase2b
flush = torch.zeros(256 << 20, dtype=torch.uint8, device=dev)
flush_sink = torch.zeros((), dtype=torch.int64, device=dev)


def timed(fn, rounds=10, warm=3):
    ms = []
    for r in range(warm + rounds):
        flush_sink.copy_(flush.view(torch.int32).sum())   # evict L2 by reading: no dirty lines billed to the kernel
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(ext); fn(); e1.record(ext)
        torch.cuda.synchronize()
        if r >= warm:
            ms.append(e0.elapsed_time(e1))
    return float(np.mean(ms)), float(np.std(ms))


enc_ms, enc_sd = timed(lambda: eng.wire_encode_vm_replies_dev(d_rec.data_ptr(), n, 0, d_voffs.data_ptr(), 0,
                                                               d_bytes.data_ptr(), cap, d_offs.data_ptr()))
eng.sync()
assert int(d_offs[n].item()) == total
assert np.array_equal(np.diff(d_offs.cpu().numpy()), msg_len)
dec_ms, dec_sd = timed(lambda: eng.wire_decode_vm_server_inbound_dev(d_bytes.data_ptr(), d_offs.data_ptr(), n,
                                                                     d_kind.data_ptr(), d_out.data_ptr(),
                                                                     d_sender.data_ptr()))
eng.sync()
assert torch.equal(d_out, d_rec) and bool((d_kind == 5).all()) and torch.equal(d_sender, d_rec[:, 1])
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
enc_bytes = 16 * n + total + 4 * (n + 1)                  # records in, bytes + offsets out
dec_bytes = total + 4 * (n + 1) + 16 * n + 4 * n + 4 * n  # bytes + offsets in, records + kinds + senders out
print(json.dumps({
    "workload": "cfg5 Phase2 replies: 6*2^20 ServerInbound{phase2b}, slots < 2^20, round 0", "messages": n,
    "wire_bytes": total, "bytes_per_message": total / n,
    "encode": {"ms": enc_ms, "ms_std": enc_sd, "messages_per_s": n / (enc_ms * 1e-3), "algorithmic_bytes": enc_bytes,
               "GB/s": enc_bytes / (enc_ms * 1e-3) / 1e9,
               "kernels": "wire_size_kernel<WireKindCodec<kWireVmReply>> + tile_offsets_kernel + "
                          "wire_gather_emit_kernel<WireKindCodec<kWireVmReply>>"},
    "decode": {"ms": dec_ms, "ms_std": dec_sd, "messages_per_s": n / (dec_ms * 1e-3), "algorithmic_bytes": dec_bytes,
               "GB/s": dec_bytes / (dec_ms * 1e-3) / 1e9, "kernels": "wire_decode_kernel"},
    "device": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip(), "l2": "256 MB buffer read between rounds"}))
eng.close()
