"""Golden vectors for the servers' side of a vanilla Mencius revocation: tests/golden/wire_vm_revoke.json.

Each case starts from an empty engine of n = 3 servers and applies `setup` (Phase2a records {slot, round, value,
server}, Chosen records {is_revocation, server, slot, value}), then delivers one ServerInbound batch to
fpx_vm_phase1a_wire with `next_slot`.  The expected replies come from tests/vm_revoke_model.py (a transcription of
Server.handlePhase1a, S/vanillamencius/Server.scala:831-911) serialised by Google's Python protobuf runtime, with the
message shapes of make_wire_vm_golden.py; `entries` are every server's fpx_vm_entries rows of slots [0, 24) after
the batch.  Values: value id v is the CommandOrNoop `values_hex[v]`.

    python tests/golden/make_wire_vm_revoke_golden.py      # rewrites tests/golden/wire_vm_revoke.json
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import make_wire_vm_golden as G  # noqa: E402
from vm_revoke_model import NOOP, Server  # noqa: E402

N, SLOTS = 3, 24


def cmd_or_noop(vals, v):
    if v == NOOP:
        c = G.vcls("CommandOrNoop")()
        c.noop.SetInParent()
        return c
    return vals[v]


def reply_bytes(vals, server, reply):
    si = G.vcls("ServerInbound")()
    if reply[0] == "nack":
        _, start, stop, rnd = reply
        si.phase1_nack.start_slot_inclusive, si.phase1_nack.stop_slot_exclusive, si.phase1_nack.round = start, stop, rnd
        return si.SerializeToString()
    _, rnd, start, stop, infos = reply
    p = si.phase1b
    p.server_index, p.round, p.start_slot_inclusive, p.stop_slot_exclusive = server, rnd, start, stop
    for slot, kind, a, b in infos:
        info = p.info.add()
        info.slot = slot
        if kind == "pending":
            info.pending_slot_info.vote_round = a
            info.pending_slot_info.vote_value.CopyFrom(cmd_or_noop(vals, b))
        else:
            info.chosen_slot_info.value.CopyFrom(cmd_or_noop(vals, a))
            info.chosen_slot_info.is_revocation = bool(b)
    return si.SerializeToString()


def phase1a(round_, start, stop):
    si = G.vcls("ServerInbound")()
    si.phase1a.round, si.phase1a.start_slot_inclusive, si.phase1a.stop_slot_exclusive = round_, start, stop
    return si.SerializeToString()


def case(name, vals, p2a, chosen, batch, next_slot=(0, 1, 2)):
    """batch: [(receiving server, ServerInbound bytes)]"""
    model = [Server(s, N, next_slot[s]) for s in range(N)]
    for slot, rnd, v, s in p2a:
        model[s].phase2a(slot, rnd, v)
    for rev, s, slot, v in chosen:
        model[s].choose(slot, v, rev)
    replies, skips = [], []
    for s, msg in batch:
        si = G.vcls("ServerInbound")(); si.ParseFromString(msg)
        if si.WhichOneof("request") != "phase1a":
            replies.append(""); skips.append(None)
            continue
        rep, skip = model[s].phase1a(si.phase1a.round, si.phase1a.start_slot_inclusive, si.phase1a.stop_slot_exclusive)
        replies.append(reply_bytes(vals, s, rep).hex()); skips.append(list(skip) if skip else None)
    return {"name": name, "setup_phase2a": [list(x) for x in p2a], "setup_chosen": [list(x) for x in chosen],
            "next_slot": list(next_slot), "batch": [[s, m.hex()] for s, m in batch], "replies": replies,
            "skips": skips, "next_slot_after": [m.next_slot for m in model],
            "entries": [[list(m.entry_row(x)) for x in range(SLOTS)] for m in model]}


def cases():
    g = np.random.Generator(np.random.PCG64(7))
    vals = [G.vvalue(g, k) for k in (0, 5, 30, 200)]
    votes = [(0, 0, 0, 1), (3, 2, 1, 1), (6, 0, 2, 1), (9, 1, NOOP, 1), (12, 0, 3, 1)]
    out = [
        # a Nack at the first, a middle and the last walked slot of [0, 15): the slots before it stay raised
        case("nack_first_slot", vals, votes + [(0, 9, 1, 2)], [], [(2, phase1a(4, 0, 15))]),
        case("nack_middle_slot", vals, votes + [(6, 9, 1, 2)], [], [(2, phase1a(4, 0, 15)), (1, phase1a(4, 0, 15))]),
        case("nack_last_slot", vals, votes + [(12, 9, 1, 1)], [], [(1, phase1a(4, 0, 15))]),
        case("empty_range", vals, votes, [], [(1, phase1a(3, 6, 6)), (2, phase1a(3, 9, 2))]),
        # server 0 revoked while alive: its log fill first, then the walk
        case("self_revocation_fill", vals, [(0, 0, 1, 0), (3, 0, 2, 0)], [], [(0, phase1a(3, 0, 19))],
             next_slot=(6, 1, 2)),
        case("chosen_with_revocation", vals, votes, [(1, 1, 3, 2), (0, 1, 6, NOOP), (1, 2, 9, 1), (0, 2, 9, 1)],
             [(1, phase1a(5, 0, 12)), (2, phase1a(5, 0, 12))]),
        # two Phase1a of one server in one batch: the second, lower one meets the first's raise
        case("raise_then_lower_round", vals, votes, [], [(1, phase1a(6, 0, 9)), (1, phase1a(4, 0, 9)),
                                                          (1, phase1a(7, 3, 12))]),
        case("other_members_get_nothing", vals, votes, [],
             [(0, G.vcls("ServerInbound")(phase2b=G.vcls("Phase2b")(server_index=0, slot=1, round=0)).SerializeToString()),
              (1, phase1a(3, 1, 8))]),
    ]
    return [v.SerializeToString().hex() for v in vals], out


def main():
    values, cs = cases()
    with open(os.path.join(HERE, "wire_vm_revoke.json"), "w") as f:
        json.dump({"n": N, "slots": SLOTS, "values_hex": values, "cases": cs}, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
