"""Device time of the wire codec on the cfg2 step's Phase2b traffic (3 * 2^20 messages):
encode the acceptor's replies into ProxyLeaderInbound bytes, decode them back into records.
CUDA events on the engine's stream, inputs resident in HBM, 3 warm-up + 10 timed rounds.
    python profiles/bench_wire.py"""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from frankenpaxos_b200 import Engine  # noqa: E402
from frankenpaxos_b200 import traces as T  # noqa: E402

dev = torch.device("cuda", 0)
n_slots = 1 << 20
cfg = bench.CFG
eng = Engine(slot_capacity=n_slots, max_batch=3 * n_slots, **cfg)
ext = torch.cuda.ExternalStream(eng.stream, device=dev)
_, p, b = T.workload(0, cfg, n_slots)
n = len(b)
d_rec = torch.from_numpy(b.view(np.int32).reshape(n, 4)).to(dev)
cap = 46 * n
d_bytes = torch.empty(cap + 64, dtype=torch.uint8, device=dev)
d_offs = torch.empty(n + 1, dtype=torch.int32, device=dev)
d_kind = torch.empty(n, dtype=torch.int32, device=dev)
d_out = torch.empty((n, 4), dtype=torch.int32, device=dev)
flush = torch.zeros(256 << 20, dtype=torch.uint8, device=dev)
flush_sink = torch.zeros((), dtype=torch.int64, device=dev)


def timed(fn, rounds=10, warm=3):
    ms = []
    for r in range(warm + rounds):
        flush_sink.copy_(flush.view(torch.int32).sum())   # evict L2 between rounds by READING 256 MB: lines stay clean
                                                            # (a written flush buffer leaves a whole L2 of dirty lines whose
                                                            # write-back would be billed to the timed kernel)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(ext); fn(); e1.record(ext)
        torch.cuda.synchronize()
        if r >= warm:
            ms.append(e0.elapsed_time(e1))
    return float(np.mean(ms))


enc_ms = timed(lambda: eng.wire_encode_phase2b_dev(d_rec.data_ptr(), n, d_bytes.data_ptr(), cap, d_offs.data_ptr()))
eng.sync()
total = int(d_offs[n].item())
dec_ms = timed(lambda: eng.wire_decode_inbound_dev(0, d_bytes.data_ptr(), d_offs.data_ptr(), n, d_kind.data_ptr(),
                                                   d_out.data_ptr()))
eng.sync()
assert torch.equal(d_out, d_rec) and bool((d_kind == 2).all())
peak, src = bench.peaks()
enc_bytes = 16 * n + total + 4 * (n + 1)          # records in, bytes + offsets out
dec_bytes = total + 4 * (n + 1) + 16 * n + 4 * n  # bytes + offsets in, records + kinds out
print(json.dumps({
    "workload": "cfg2 step: 3*2^20 Phase2b, slots < 2^20, round 0", "messages": n, "wire_bytes": total,
    "bytes_per_message": total / n,
    "encode": {"ms": enc_ms, "messages_per_s": n / (enc_ms * 1e-3), "algorithmic_bytes": enc_bytes,
               "GB/s": enc_bytes / (enc_ms * 1e-3) / 1e9, "frac_of_hbm_peak": enc_bytes / (enc_ms * 1e-3) / 1e9 / peak,
               "kernels": "wire_size_kernel + wire_emit_small_kernel"},
    "decode": {"ms": dec_ms, "messages_per_s": n / (dec_ms * 1e-3), "algorithmic_bytes": dec_bytes,
               "GB/s": dec_bytes / (dec_ms * 1e-3) / 1e9, "frac_of_hbm_peak": dec_bytes / (dec_ms * 1e-3) / 1e9 / peak,
               "kernels": "wire_decode_kernel"},
    "hbm_peak_GB/s": peak, "peak_source": src, "l2": "256 MB buffer read between rounds"}))
