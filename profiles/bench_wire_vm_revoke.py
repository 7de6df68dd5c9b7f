"""Time of the servers' side of a vanilla Mencius revocation at cfg5 (n = 7, f = 3, 2^20 slots in flight): server 3
fails and its 2^17 slots of the range [3, 3 + 7 * 2^17) are revoked.  About a third of them hold a round-0 vote at
each survivor, with values of 0-200 bytes.
  phase1a   the f + 1 = 4 survivors' Phase1a -> 4 Phase1bs (fpx_vm_phase1a_wire_dev).  The call reads its walked-slot
            count back once, so its time is a host clock around work that ends in a sync.  Each round first restores
            the entries the previous round raised, outside the timed region.
  choose    the 2^17 Chosen{isRevocation = true} at one survivor (fpx_vm_choose_dev), CUDA events.
The single-threaded CPU model of Server.handlePhase1a (tests/vm_revoke_model.py) is timed on one survivor's Phase1a
for comparison.  The card's name and power limit are read in the same run.  2 warm-up + 5 timed rounds (mean).
    python profiles/bench_wire_vm_revoke.py"""
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
import wire_vm_oracle as V  # noqa: E402
from vm_revoke_model import Server  # noqa: E402
from frankenpaxos_b200 import P2A, P2B, VALUE_NOOP, VANILLA_MENCIUS, Engine  # noqa: E402

assert torch.cuda.is_available(), "this measurement needs the GPU"
dev = torch.device("cuda", 0)
N, F, CAP, WALKED, REVOKED = 7, 3, 1 << 20, 1 << 17, 3
SURVIVORS = [0, 1, 2, 4]
START, STOP = REVOKED, REVOKED + N * WALKED
ROUND = N + 1
g = np.random.Generator(np.random.PCG64(0))


def varint(v):
    out = bytearray()
    while True:
        b = v & 0x7f
        v >>= 7
        out.append(b | (0x80 if v else 0))
        if not v:
            return bytes(out)


def field(num, payload):
    return varint(num << 3 | 2) + varint(len(payload)) + payload


# CommandOrNoop{command {command_id {client_address, pseudonym, id}, command}} values of 0-200 command bytes
values = [field(1, field(1, field(1, b"c") + b"\x10\x01\x18" + varint(k)) + field(2, bytes(g.integers(0, 256, int(g.integers(0, 201))).astype(np.uint8))))
          for k in range(256)]
arena, voffs = V.pack(values)
slots = np.arange(START, STOP, N)
eng = Engine(F, 1, N, slot_capacity=CAP, max_batch=1 << 20, protocol=VANILLA_MENCIUS)
p2a = []
for s in SURVIVORS:
    hit = slots[g.random(len(slots)) < 0.3]
    p2a.append(np.rec.fromarrays([hit, np.zeros(len(hit)), g.integers(0, len(values), len(hit)), np.full(len(hit), s)],
                                 dtype=P2A).view(P2A))
p2a = np.concatenate(p2a)
phase1a = field(2, b"\x08" + varint(ROUND) + b"\x10" + varint(START) + b"\x18" + varint(STOP))
buf, offs = V.pack([phase1a] * len(SURVIVORS))
kind, rec, _ = eng.wire_decode_vm_server_inbound(buf, offs)
rec = rec.copy(); rec["a"] = SURVIVORS


def dev_of(x):
    return torch.from_numpy(np.ascontiguousarray(x).view(np.uint8).reshape(-1).copy()).to(dev)


d_buf, d_kind, d_rec = dev_of(np.frombuffer(bytes(buf) + b"\0", np.uint8)), dev_of(kind), dev_of(rec)
d_arena, d_voffs = dev_of(np.frombuffer(bytes(arena) + b"\0", np.uint8)), dev_of(voffs)
d_ns = dev_of(np.arange(N, dtype=np.int32) + N * (STOP // N + 1))
cap = 64 * len(SURVIVORS) + len(SURVIVORS) * WALKED * (48 + max(len(v) for v in values))
d_out = torch.zeros(cap, dtype=torch.uint8, device=dev)
d_offs = torch.zeros(len(SURVIVORS) + 1, dtype=torch.int32, device=dev)
d_skips = torch.zeros((len(SURVIVORS), 4), dtype=torch.int32, device=dev)
chosen = np.rec.fromarrays([np.ones(WALKED), np.zeros(WALKED), slots, g.integers(0, len(values), WALKED)],
                           dtype=P2B).view(P2B)
d_chosen = dev_of(chosen)


def run_phase1a():
    eng.vm_phase1a_wire_dev(d_buf.data_ptr(), len(buf), d_kind.data_ptr(), d_rec.data_ptr(), len(SURVIVORS),
                            d_arena.data_ptr(), d_voffs.data_ptr(), len(values), d_ns.data_ptr(), d_out.data_ptr(), cap,
                            d_offs.data_ptr(), d_skips.data_ptr())
    torch.cuda.synchronize()


ms_p1a, ms_choose = [], []
ext = torch.cuda.ExternalStream(eng.stream, device=dev)
for r in range(7):
    eng.reset()
    eng.vm_phase2a(p2a)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    run_phase1a()
    t1 = time.perf_counter()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(ext)
    eng.vm_choose_dev(d_chosen.data_ptr(), WALKED)
    b.record(ext)
    torch.cuda.synchronize()
    if r >= 2:
        ms_p1a.append((t1 - t0) * 1e3)
        ms_choose.append(a.elapsed_time(b))
reply_bytes = int(d_offs[-1].item())

model = Server(0, N, next_slot=int(N * (STOP // N + 1)))
for r in p2a[p2a["dst"] == 0]:
    model.phase2a(int(r["slot"]), 0, int(r["value_id"]))
t0 = time.perf_counter()
model.phase1a(ROUND, START, STOP)
cpu_ms = (time.perf_counter() - t0) * 1e3

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                      text=True).stdout.strip()
print(json.dumps({"card": card, "config": "cfg5: n = 7, f = 3, 2^20 slots, server 3's 2^17 slots revoked",
                  "phase1a_ms": float(np.mean(ms_p1a)), "phase1a_reply_bytes": reply_bytes,
                  "choose_ms": float(np.mean(ms_choose)),
                  "cpu_model_phase1a_one_server_ms": cpu_ms}))
