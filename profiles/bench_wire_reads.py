"""Device time of the MultiPaxos replica / read-path wire codec at the sizes of a cfg2 step (f = 2, 2^20 slots):
  encode  3 * 2^20 MaxSlotReplies from decoded AcceptorInbound{max_slot_request} records (fpx_wire_encode_max_slot_replies),
          2^20 ReadRequests and 2^14 ReadRequestBatches of 64 Commands (fpx_reads_wire_encode_read_requests);
  decode  those 3 * 2^20 ClientInbound{max_slot_reply} messages (fpx_reads_wire_decode), and on the replica
          (fpx_wire_decode_replica_inbound) the 2^20 Chosen messages fpx_wire_encode_chosen writes for a cfg2 step
          and the ReadRequests and ReadRequestBatches above.
CUDA events on the engine's stream, inputs resident in HBM, L2 flushed by a 256 MB read between rounds, 3 warm-up +
10 timed rounds (mean).  The card's name and power limit are read in the same run.
    python profiles/bench_wire_reads.py"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from frankenpaxos_b200 import (CHOSEN, READS_CLIENT, READS_READ_BATCHER, WIRE_ACCEPTOR_INBOUND, Engine,  # noqa: E402
                               Reads)
from frankenpaxos_b200 import traces as T  # noqa: E402

assert torch.cuda.is_available(), "this measurement needs the GPU"
dev = torch.device("cuda", 0)
cfg, n_slots = T.config_by_name("cfg2")
N = 3 * n_slots                                   # f + 1 = 3 MaxSlotReplies per linearizable read
eng = Engine(slot_capacity=n_slots, max_batch=n_slots, **cfg)
ext = torch.cuda.ExternalStream(eng.stream, device=dev)
client = Reads(eng, READS_CLIENT, key_capacity=1 << 10, pending_capacity=1 << 10, max_batch=1 << 10)
batcher = Reads(eng, READS_READ_BATCHER, key_capacity=1 << 10, pending_capacity=1 << 10, max_batch=1 << 10)
flush = torch.zeros(256 << 20, dtype=torch.uint8, device=dev)
flush_sink = torch.zeros((), dtype=torch.int64, device=dev)
i32 = lambda *s: torch.zeros(s, dtype=torch.int32, device=dev)
u8 = lambda n: torch.zeros(n + 64, dtype=torch.uint8, device=dev)


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
    return {"ms": float(np.mean(ms)), "ms_std": float(np.std(ms))}


def offsets_of(lengths):
    return torch.from_numpy(np.concatenate([[0], np.cumsum(lengths)]).astype(np.int32)).to(dev)


res = {}
# -- the acceptor: AcceptorInbound{max_slot_request{command_id{client_address (16 B), pseudonym, id}}}
cid = bytes([0x0a, 16]) + bytes(range(16)) + bytes([0x10, 0xc8, 0x01, 0x18, 0x90, 0x4e])
body = bytes([0x0a, len(cid)]) + cid
req = bytes([0x1a, len(body)]) + body
d_req = torch.from_numpy(np.tile(np.frombuffer(req, np.uint8), N)).to(dev)
d_req = torch.cat([d_req, torch.zeros(64, dtype=torch.uint8, device=dev)])
d_req_offs = offsets_of(np.full(N, len(req)))
d_kind, d_rec = i32(N), i32(N, 4)
torch.cuda.synchronize()                          # the inputs are written on torch's stream, the codec runs on the engine's
eng.wire_decode_inbound_dev(WIRE_ACCEPTOR_INBOUND, d_req.data_ptr(), d_req_offs.data_ptr(), N, d_kind.data_ptr(),
                            d_rec.data_ptr())
eng.sync()
acc = torch.arange(N, device=dev, dtype=torch.int32) % 5
d_rec[:, 0] = acc; d_rec[:, 1] = torch.arange(N, device=dev, dtype=torch.int32) // 3
cap = 64 * N
d_rep, d_rep_offs = u8(cap), i32(N + 1)
res["encode_max_slot_replies"] = timed(lambda: eng.wire_encode_max_slot_replies_dev(
    d_req.data_ptr(), len(req) * N, d_kind.data_ptr(), d_rec.data_ptr(), N, d_rep.data_ptr(), cap, d_rep_offs.data_ptr()))
eng.sync()
rep_bytes = int(d_rep_offs[N].item())
# -- the Client: the 3 * 2^20 ClientInbound{max_slot_reply}
d_k2, d_o2, d_s2 = i32(N), i32(N, 4), i32(N, 2)
res["decode_client_max_slot_replies"] = timed(lambda: client.wire_decode_dev(
    d_rep.data_ptr(), d_rep_offs.data_ptr(), N, d_k2.data_ptr(), d_o2.data_ptr(), d_s2.data_ptr()))
client.sync()
assert bool((d_k2 == 4).all()) and bool((d_o2[:, 2] == acc).all()) and bool((d_o2[:, 0] == 200).all())
# -- the replica: the Chosen stream of a cfg2 step, Noop values
chosen = np.zeros(n_slots, CHOSEN)
chosen["slot"] = np.random.default_rng(0).permutation(n_slots); chosen["value_id"] = np.arange(n_slots)
arena = np.tile(np.frombuffer(b"\x12\x00", np.uint8), n_slots)
wbuf, woffs = eng.wire_encode_chosen(chosen, arena, np.arange(0, 2 * n_slots + 1, 2, dtype=np.int32))
d_ch_bytes = torch.from_numpy(np.concatenate([wbuf, np.zeros(64, np.uint8)])).to(dev)
d_ch_offs = torch.from_numpy(woffs).to(dev)
d_kind3, d_ch, d_cv, d_rd, d_rc, d_cnt = i32(n_slots), i32(n_slots, 2), i32(n_slots, 2), i32(1 << 20, 2), \
    i32(1 << 20, 2), i32(3)
torch.cuda.synchronize()


def replica_decode(d_bytes, d_offs, n, cap):
    return lambda: eng.wire_decode_replica_inbound_dev(d_bytes.data_ptr(), d_offs.data_ptr(), n, 0, 0, cap,
                                                       d_kind3.data_ptr(), d_ch.data_ptr(), d_cv.data_ptr(),
                                                       d_rd.data_ptr(), d_rc.data_ptr(), d_cnt.data_ptr())


res["decode_replica_chosen"] = timed(replica_decode(d_ch_bytes, d_ch_offs, n_slots, 0))
eng.sync()
assert d_cnt.cpu().tolist() == [n_slots, 0, n_slots]
# -- completed reads: 2^20 ReadRequests (Client) and 2^14 ReadRequestBatches of 64 (ReadBatcher)
cmd = bytes([0x0a, len(cid)]) + cid + bytes([0x12, 8]) + bytes(8)               # Command{command_id, 8 B}
entry = bytes([0x12, len(cmd)]) + cmd
for name, h, n, per in (("read_request", client, n_slots, 1), ("read_request_batch", batcher, 1 << 14, 64)):
    recs = np.zeros((n, 4), np.int32)
    recs[:, 0] = np.arange(n); recs[:, 2] = np.arange(n) * 7
    d_in = torch.from_numpy(recs).to(dev)
    d_arena = torch.from_numpy(np.tile(np.frombuffer(entry * per, np.uint8), n)).to(dev)
    d_voffs = offsets_of(np.full(n, len(entry) * per))
    cap = (len(entry) * per + 16) * n
    d_out, d_offs = u8(cap), i32(n + 1)
    torch.cuda.synchronize()
    res[f"encode_{name}"] = timed(lambda: h.wire_encode_read_requests_dev(
        d_in.data_ptr(), n, d_arena.data_ptr(), d_voffs.data_ptr(), n, d_out.data_ptr(), cap, d_offs.data_ptr()))
    h.sync()
    res[f"decode_replica_{name}"] = timed(replica_decode(d_out, d_offs, n, 1 << 20))
    eng.sync()
    assert d_cnt.cpu().tolist() == [0, n * per, n]
    res[f"encode_{name}"]["messages"] = res[f"decode_replica_{name}"]["messages"] = n
    res[f"encode_{name}"]["wire_bytes"] = int(d_offs[n].item())
for k in ("encode_max_slot_replies", "decode_client_max_slot_replies"):
    res[k]["messages"] = N; res[k]["wire_bytes"] = rep_bytes
res["decode_replica_chosen"]["messages"] = n_slots; res["decode_replica_chosen"]["wire_bytes"] = int(woffs[-1])
for v in res.values():
    v["messages_per_s"] = v["messages"] / (v["ms"] * 1e-3)
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
print(json.dumps({"workload": "cfg2-sized read path and replica input", "results": res,
                  "device": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip(),
                  "l2": "256 MB buffer read between rounds"}))
client.close(); batcher.close(); eng.close()
