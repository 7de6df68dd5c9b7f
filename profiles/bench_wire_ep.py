"""Device time of the EPaxos wire codec on BASELINE cfg4's traffic (f = 2, n = 5 replicas, 2^20 instances led round
robin): decode the 838 860 PreAccepts replica 0 receives and pack them into fpx_epaxos_preaccept rows, encode its
handlePreAccept replies (the PreAcceptOks it sends back), and decode the PreAcceptOks replica 0 receives as a leader
and pack them into fpx_epaxos_preacceptok rows.  The bytes are written by
Google's Python protobuf runtime (tests/golden/make_wire_ep_golden.py's descriptor pool), the decoded rows checked
against the trace.  CUDA events on the handle's stream, inputs resident in HBM, L2 flushed by a 256 MB read between
rounds, 3 warm-up + 10 timed rounds.  The card's name and power limit are read in the same run.
    python profiles/bench_wire_ep.py"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from frankenpaxos_b200 import traces as T  # noqa: E402
from frankenpaxos_b200.epaxos import CALL_PREACCEPT, CALL_PREACCEPTOK, REPLY_OK, EpaxosReplica  # noqa: E402
import wire_ep_oracle as W  # noqa: E402

assert torch.cuda.is_available(), "this measurement needs the GPU"
dev = torch.device("cuda", 0)
f, N = 2, 1 << 20
n = 2 * f + 1
lead, pa, ok = T.epaxos_cfg4(0, f=f, n_instances=N, me=0)
G = W.golden_module()
eng = EpaxosReplica(f, 0, N // n + 2, max_batch=max(len(pa), len(ok)))
ext = torch.cuda.ExternalStream(eng.stream, device=dev)
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


def measure(name, raws, call, expect, local_deps=None):
    buf, offs = W.pack(raws)
    m = len(raws)
    d_buf, d_offs = torch.from_numpy(buf).to(dev), torch.from_numpy(offs).to(dev)
    d_kind = torch.empty(m, dtype=torch.int32, device=dev)
    d_rows = torch.empty((m, 12 + n), dtype=torch.int32, device=dev)
    d_values = torch.empty((m, 2), dtype=torch.int32, device=dev)
    d_out = torch.empty((m, expect.shape[1]), dtype=torch.int32, device=dev)
    d_ld = None if local_deps is None else torch.from_numpy(np.ascontiguousarray(local_deps)).to(dev)

    def dec():
        eng.wire_decode_dev(d_buf.data_ptr(), d_offs.data_ptr(), m, 0, d_kind.data_ptr(), d_rows.data_ptr(),
                            d_values.data_ptr())

    def pk():
        eng.wire_pack_dev(call, d_kind.data_ptr(), d_rows.data_ptr(), 0, m, 0 if d_ld is None else d_ld.data_ptr(),
                          d_out.data_ptr())

    dec_ms, dec_sd = timed(dec)
    pack_ms, pack_sd = timed(pk)
    eng.sync()
    got = d_out.cpu().numpy()
    if call == CALL_PREACCEPT:
        got[:, 4] = expect[:, 4]                          # value ids: the decoder's are batch positions
    assert np.array_equal(got, expect), name
    total = int(offs[-1])
    dec_bytes = total + 4 * (m + 1) + 4 * m * (13 + n) + 8 * m   # bytes + offsets in, kinds + rows + spans out
    return {"messages": m, "wire_bytes": total, "bytes_per_message": total / m,
            "decode": {"ms": dec_ms, "ms_std": dec_sd, "messages_per_s": m / (dec_ms * 1e-3),
                       "algorithmic_bytes": dec_bytes, "GB/s": dec_bytes / (dec_ms * 1e-3) / 1e9,
                       "kernels": "ep_wire_decode_kernel"},
            "pack": {"ms": pack_ms, "ms_std": pack_sd, "kernels": "ep_wire_pack_kernel"}}, d_out


res = {"workload": "cfg4 (f = 2, 2^20 instances): replica 0's PreAccepts and PreAcceptOks"}
res["preaccept"], pa_rows = measure("PreAccept", W.preaccept_messages(G, pa, n), CALL_PREACCEPT, pa, pa[:, 6:6 + n])
res["preacceptok"], _ = measure("PreAcceptOk", W.preacceptok_messages(G, ok, n), CALL_PREACCEPTOK, ok)


def measure_encode(d_in, m):
    """handlePreAccept on the packed rows once, then its m replies to bytes (fpx_epaxos_wire_encode_dev)"""
    d_reply = torch.empty((m, 4 + n), dtype=torch.int32, device=dev)
    eng.preaccept_dev(d_in.data_ptr(), m, d_reply.data_ptr())
    eng.sync()
    arena, voffs = W.value_arena(m + 1)                    # the decoder's value ids: batch positions
    d_arena, d_voffs = torch.from_numpy(arena).to(dev), torch.from_numpy(voffs.astype(np.int32)).to(dev)
    cap = m * (128 + 14 * n) + 16
    d_bytes = torch.empty(cap, dtype=torch.uint8, device=dev)
    d_offs = torch.empty(m + 1, dtype=torch.int32, device=dev)

    def enc():
        eng.wire_encode_dev(CALL_PREACCEPT, d_in.data_ptr(), d_reply.data_ptr(), m, d_arena.data_ptr(),
                            d_voffs.data_ptr(), len(voffs) - 1, d_bytes.data_ptr(), cap, d_offs.data_ptr())

    enc_ms, enc_sd = timed(enc)
    eng.sync()
    lens = np.diff(d_offs.cpu().numpy())
    kinds = d_reply[:, 0].cpu().numpy()
    assert bool((kinds == REPLY_OK).all()) and bool((lens > 0).all())   # a PreAcceptOk for every PreAccept
    total = int(lens.sum())
    enc_bytes = 4 * m * (6 + 2 * n) + 4 * m * (4 + n) + total + 4 * (m + 1)   # rows in, bytes + offsets out
    return {"messages": m, "wire_bytes": total, "bytes_per_message": total / m, "ms": enc_ms, "ms_std": enc_sd,
            "messages_per_s": m / (enc_ms * 1e-3), "algorithmic_bytes": enc_bytes,
            "GB/s": enc_bytes / (enc_ms * 1e-3) / 1e9,
            "kernels": "wire_size_kernel<EpWireCodec> + tile_offsets_kernel + wire_gather_emit_kernel<EpWireCodec>"}


res["encode"] = {"preacceptok_replies": measure_encode(pa_rows, len(pa))}
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
res.update({"device": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip(),
            "l2": "256 MB buffer read between rounds"})
print(json.dumps(res))
eng.close()
