"""Batches and traces for compartmentalized Mencius' leader-change wire path tests
(tests/test_wire_mencius_phase1_*.py).  TEST INFRASTRUCTURE."""
import importlib.util
import json
import os

import numpy as np

import wire_mencius_phase1_oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = json.load(open(os.path.join(HERE, "golden", "wire_mencius_phase1.json")))

_mk = None


def runtime():
    """tests/golden/make_wire_mencius_phase1_golden.py: the protobuf runtime's classes and the Python transcriptions."""
    global _mk
    if _mk is None:
        spec = importlib.util.spec_from_file_location("mk_mencius_phase1",
                                                      os.path.join(HERE, "golden", "make_wire_mencius_phase1_golden.py"))
        _mk = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(_mk)
    return _mk


def arena(g, n_values, max_len=200):
    """CommandBatchOrNoop-like value bytes of 0 .. max_len bytes."""
    lens = g.integers(0, max_len + 1, size=n_values)
    voffs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    return g.integers(0, 256, size=int(voffs[-1]), dtype=np.uint8), voffs


# canonical CommandBatchOrNoops, which the runtime re-serializes unchanged: Noop, an empty batch, one command
_CMD_ID = b"\x0a\x01a\x10\x01\x18\x01"
_CMD = b"\x0a" + bytes([len(_CMD_ID)]) + _CMD_ID + b"\x12\x02xy"
_BATCH = b"\x0a" + bytes([len(_CMD)]) + _CMD
VALUES = [b"\x12\x00", b"\x0a\x00", b"\x0a" + bytes([len(_BATCH)]) + _BATCH]


def value_arena():
    a = np.frombuffer(b"".join(VALUES), np.uint8).copy()
    return a, np.concatenate([[0], np.cumsum([len(v) for v in VALUES])]).astype(np.int32)


def empty_phase1b(group, acceptor, round_):
    return O.encode_phase1b(group, acceptor, round_, [], [], [], np.zeros(0, np.uint8), np.zeros(1, np.int32))


def random_batch(g, lgroups, agroups, per_group, leader_group, round_, n_slots, n_msgs, arena_, voffs, extra=True):
    """Phase1bs of random acceptors of one leader group with votes on its slots (ascending, some duplicated), stale
    rounds and replacing duplicates; when extra, sometimes a slot of another leader group, a higher round or a
    non-member."""
    msgs = []
    for _ in range(n_msgs):
        gi, ai = int(g.integers(0, agroups)), int(g.integers(0, per_group))
        rnd = round_ - int(g.integers(0, 2)) if g.random() < 0.3 else round_
        k = int(g.integers(0, n_slots + 1))
        slots = leader_group + lgroups * np.sort(g.choice(n_slots, size=k, replace=False)) if k else np.zeros(0, int)
        slots = slots.astype(np.int32)
        if k > 2 and g.random() < 0.3:
            slots = np.sort(np.concatenate([slots, slots[:2]]))
        if extra and k and g.random() < 0.05:
            slots[-1] += 1                                      # another leader group's slot
        vr = g.integers(-1, round_ + 1, size=len(slots)).astype(np.int32)
        vid = g.integers(0, len(voffs) - 1, size=len(slots)).astype(np.int32)
        vid[g.random(len(slots)) < 0.2] = O.VALUE_NOOP
        msgs.append(O.encode_phase1b(gi, ai, rnd, slots, vr, vid, arena_, voffs))
    if extra and g.random() < 0.3:
        at = int(g.integers(0, len(msgs) + 1))
        bad = empty_phase1b(int(g.integers(0, agroups)), per_group, round_) if g.random() < 0.5 else \
            empty_phase1b(0, 0, round_ + 1)
        msgs.insert(at, bad)
    return msgs


def phase1a_batch(rounds_cws, acceptors):
    """AcceptorInbound{phase1a} per (round, chosen_watermark) -> (request bytes, kind, WIRE_REC records with a =
    acceptors[i]) as fpx_wire_decode_inbound(FPX_WIRE_MENCIUS_ACCEPTOR_INBOUND) writes them."""
    mk = runtime()
    body, kind, recs = b"", [], np.zeros(len(rounds_cws), O.WIRE_REC)
    for i, ((r, cw), a) in enumerate(zip(rounds_cws, acceptors)):
        m = mk.cls("AcceptorInbound")()
        m.phase1a.round, m.phase1a.chosen_watermark = r, cw
        inner = m.phase1a.SerializeToString()
        raw = m.SerializeToString()
        start = len(body) + len(raw) - len(inner)
        recs[i] = (a, 0, start, len(inner))
        kind.append(1)
        body += raw
    return np.frombuffer(body + b"\0" * 16, np.uint8).copy(), np.array(kind, np.int32), recs


def random_trace(g, f, lgroups, agroups, capacity, n_p2a, n_ranges, max_round, n_values):
    """Phase2a records (dst = engine group << 16 | acceptor, the slot's group) and Phase2aNoopRange records over
    capacity slots, in the order a test delivers them: ranges after the Phase2as they cover, so that noop-range votes
    lie above every Phase2a vote of some acceptors."""
    per_group = 2 * f + 1
    p2a = np.zeros(n_p2a, O.P2A)
    slots = g.integers(0, capacity // 2, size=n_p2a)
    p2a["slot"] = slots
    p2a["round"] = g.integers(0, max_round + 1, size=n_p2a)
    p2a["value_id"] = g.integers(0, n_values, size=n_p2a)
    p2a["value_id"][g.random(n_p2a) < 0.1] = O.VALUE_NOOP
    grp = (slots % lgroups) * agroups + (slots // lgroups) % agroups
    p2a["dst"] = (grp << 16) | g.integers(0, per_group, size=n_p2a)
    rng = np.zeros(n_ranges, O.P2A_RANGE)
    for i in range(n_ranges):
        start = int(g.integers(capacity // 4, capacity - 1))
        end = int(g.integers(start + 1, min(capacity, start + 40) + 1))
        lg = start % lgroups
        rng[i] = (start, end, int(g.integers(0, max_round + 1)),
                  ((lg * agroups + int(g.integers(0, agroups))) << 16) | int(g.integers(0, per_group)))
    return p2a, rng
