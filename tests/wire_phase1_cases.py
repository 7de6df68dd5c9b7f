"""Phase1b batches for the leader's Phase-1 wire path tests (tests/test_wire_phase1_*.py).  TEST INFRASTRUCTURE."""
import json
import os

import numpy as np

import wire_phase1_oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = json.load(open(os.path.join(HERE, "golden", "wire_phase1.json")))
F, GROUPS, PER_GROUP = 1, 2, 3          # the golden batches' config: two groups of 2f+1


def empty_phase1b(group, acceptor, round_):
    return O.encode_phase1b(group, acceptor, round_, [], [], [], np.zeros(0, np.uint8), np.zeros(1, np.int32))


def golden_batch(case):
    """The golden message first, then empty Phase1bs of its round from two other acceptors of every group: the batch
    completes at its last message whatever the golden message is."""
    v = case["verdict"]
    round_ = v.get("round", 0)
    mine = (v.get("group_index"), v.get("acceptor_index")) if v.get("kind") == 1 else None
    msgs = [bytes.fromhex(case["hex"])]
    for g in range(GROUPS):
        others = [a for a in range(PER_GROUP) if (g, a) != mine][:2]
        msgs += [empty_phase1b(g, a, round_) for a in others]
    return msgs, round_


def golden_expectation(case, buf, offs):
    """(status, complete, max_slot, [(slot, value bytes or None)]) from the runtime's parse of the golden message."""
    v = case["verdict"]
    if "error" in v:
        return -15, -1, -1, []
    n = len(offs) - 1
    info = v.get("info", []) if v.get("kind") == 1 else []
    held = v.get("kind") == 1 and v["group_index"] < GROUPS and v["acceptor_index"] < PER_GROUP
    slots = [s for s, _, _ in info] if held else []
    max_slot = max(slots) if slots else -1
    out = []
    for s in range(0, max_slot + 1):
        first = next(((vr, val) for sl, vr, val in info if sl == s), None)
        out.append((s, bytes.fromhex(first[1]) if first and s % GROUPS == v["group_index"] else None))
    keys = [(v["group_index"], v["acceptor_index"])] if held else []
    for g in range(GROUPS):
        keys += [(g, a) for a in range(PER_GROUP) if (g, a) != (keys[0] if held else None)][:2]
    have, complete = set(), -1
    for i, k in enumerate([None] * (0 if held else 1) + keys):
        if k is not None:
            have.add(k)
        if all(sum(1 for h in have if h[0] == g) >= F + 1 for g in range(GROUPS)):
            complete = i
            break
    assert complete == n - 1 or held
    return 0, complete, max_slot, out


def random_phase1b_batch(g, groups, per_group, round_, n_slots, n_msgs, arena, voffs, extra=True):
    """Phase1bs of random acceptors with random votes (slots ascending, some duplicated); stale rounds, replacing
    duplicates and, when extra, a higher round or a non-member somewhere."""
    msgs = []
    for _ in range(n_msgs):
        gi, ai = int(g.integers(0, groups)), int(g.integers(0, per_group))
        rnd = round_ - int(g.integers(0, 2)) if g.random() < 0.3 else round_
        k = int(g.integers(0, n_slots + 1))
        slots = np.sort(g.choice(n_slots, size=k, replace=False)).astype(np.int32) if k else np.zeros(0, np.int32)
        if k > 2 and g.random() < 0.3:
            slots = np.sort(np.concatenate([slots, slots[:2]]))
        vr = g.integers(-1, round_ + 1, size=len(slots)).astype(np.int32)
        vid = g.integers(0, len(voffs) - 1, size=len(slots)).astype(np.int32)
        vid[g.random(len(slots)) < 0.2] = O.VALUE_NOOP
        msgs.append(O.encode_phase1b(gi, ai, rnd, slots, vr, vid, arena, voffs))
    if extra and g.random() < 0.3:
        at = int(g.integers(0, len(msgs) + 1))
        bad = empty_phase1b(int(g.integers(0, groups)), per_group, round_) if g.random() < 0.5 else \
            empty_phase1b(0, 0, round_ + 1)
        msgs.insert(at, bad)
    return msgs


def arena(g, n_values, max_len=200):
    """CommandBatchOrNoop-like value bytes of 0 .. max_len bytes."""
    lens = g.integers(0, max_len + 1, size=n_values)
    voffs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    return g.integers(0, 256, size=int(voffs[-1]), dtype=np.uint8), voffs
