"""Golden wire vectors of compartmentalized Mencius' leader change: LeaderInbound batches for the new leader's
Phase1b handling and the Phase2a re-proposals.

Produced, like make_wire_mencius_golden.py, by Google's Python protobuf runtime (an implementation independent of
the codec) over the shapes of shared/src/main/scala/frankenpaxos/mencius/Mencius.proto: Phase1a :104-118,
Phase1bSlotInfo :120-127, Phase1b :129-137, Phase2a :151-157, Nack :266-271, Recover :288-296, LeaderInbound :322-338,
ProxyLeaderInbound :339-350, AcceptorInbound :352-361.  The LeaderInbound members this path does not parse (2-6, 8)
and the other ProxyLeaderInbound / AcceptorInbound members are transcribed as messages without fields: their bodies
are skipped by length.  Each case is a batch, the leader group's state and what `leader` (a transcription of
Leader.handlePhase1b, S/mencius/Leader.scala:582-659, over the runtime's parse) makes of it; each Phase2a case the
canonical ProxyLeaderInbound bytes of one record.  `acceptor` transcribes Acceptor.handlePhase1a
(S/mencius/Acceptor.scala:166-200) the same way; the CPU tests use both.

    python tests/golden/make_wire_mencius_phase1_golden.py      # rewrites tests/golden/wire_mencius_phase1.json
"""
import json
import os
import sys

import numpy as np
from google.protobuf import descriptor_pb2, descriptor_pool, message_factory

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_wire_mencius_golden as base  # noqa: E402

F = descriptor_pb2.FieldDescriptorProto
MPKG = "frankenpaxos.mencius.phase1"
# the golden batches' config: f = 1, three leader groups of two acceptor groups of 2f+1
FC, LG, AG, PER_GROUP = 1, 3, 2, 3


def build_pool():
    fdp = descriptor_pb2.FileDescriptorProto()
    fdp.name = "MenciusPhase1.proto"; fdp.package = MPKG; fdp.syntax = "proto2"

    def msg(name, fields, oneof=None):
        m = fdp.message_type.add(); m.name = name
        if oneof:
            m.oneof_decl.add().name = oneof
        for (fname, num, ftype, label, tname) in fields:
            f = m.field.add(); f.name = fname; f.number = num; f.type = ftype; f.label = label
            if tname:
                f.type_name = f".{MPKG}.{tname}"
            if oneof:
                f.oneof_index = 0

    REQ, OPT, REP = F.LABEL_REQUIRED, F.LABEL_OPTIONAL, F.LABEL_REPEATED
    I32, BYT, MSG = F.TYPE_INT32, F.TYPE_BYTES, F.TYPE_MESSAGE
    msg("Noop", [])
    msg("Opaque", [])
    msg("CommandId", [("client_address", 1, BYT, REQ, None), ("client_pseudonym", 2, I32, REQ, None),
                      ("client_id", 3, I32, REQ, None)])
    msg("Command", [("command_id", 1, MSG, REQ, "CommandId"), ("command", 2, BYT, REQ, None)])
    msg("CommandBatch", [("command", 1, MSG, REP, "Command")])
    msg("CommandBatchOrNoop", [("command_batch", 1, MSG, OPT, "CommandBatch"), ("noop", 2, MSG, OPT, "Noop")], "value")
    msg("Phase1a", [("round", 1, I32, REQ, None), ("chosen_watermark", 2, I32, REQ, None)])
    msg("Phase1bSlotInfo", [("slot", 1, I32, REQ, None), ("vote_round", 2, I32, REQ, None),
                            ("vote_value", 3, MSG, REQ, "CommandBatchOrNoop")])
    msg("Phase1b", [("group_index", 1, I32, REQ, None), ("acceptor_index", 2, I32, REQ, None),
                    ("round", 3, I32, REQ, None), ("info", 4, MSG, REP, "Phase1bSlotInfo")])
    msg("Phase2a", [("slot", 1, I32, REQ, None), ("round", 2, I32, REQ, None),
                    ("command_batch_or_noop", 3, MSG, REQ, "CommandBatchOrNoop")])
    msg("Nack", [("round", 1, I32, REQ, None)])
    msg("Recover", [("slot", 1, I32, REQ, None)])
    msg("LeaderInbound", [("phase1b", 1, MSG, OPT, "Phase1b"), ("client_request", 2, MSG, OPT, "Opaque"),
                          ("client_request_batch", 3, MSG, OPT, "Opaque"), ("high_watermark", 4, MSG, OPT, "Opaque"),
                          ("leader_info_request_client", 5, MSG, OPT, "Opaque"),
                          ("leader_info_request_batcher", 6, MSG, OPT, "Opaque"), ("nack", 7, MSG, OPT, "Nack"),
                          ("chosen_watermark", 8, MSG, OPT, "Opaque"), ("recover", 9, MSG, OPT, "Recover")], "request")
    msg("ProxyLeaderInbound", [("high_watermark", 1, MSG, OPT, "Opaque"), ("phase2a", 2, MSG, OPT, "Phase2a"),
                               ("phase2a_noop_range", 3, MSG, OPT, "Opaque"), ("phase2b", 4, MSG, OPT, "Opaque"),
                               ("phase2b_noop_range", 5, MSG, OPT, "Opaque")], "request")
    msg("AcceptorInbound", [("phase1a", 1, MSG, OPT, "Phase1a"), ("phase2a", 2, MSG, OPT, "Opaque"),
                            ("phase2a_noop_range", 3, MSG, OPT, "Opaque")], "request")
    pool = descriptor_pool.DescriptorPool()
    pool.Add(fdp)
    return pool


POOL = build_pool()


def cls(name):
    return message_factory.GetMessageClass(POOL.FindMessageTypeByName(f"{MPKG}.{name}"))


def payload(g, n_cmds, cmd_len):
    v = cls("CommandBatchOrNoop")()
    v.ParseFromString(base.payload(g, n_cmds, cmd_len).SerializeToString())
    return v


def phase1b(g, group, acceptor, round_, infos):
    """LeaderInbound{phase1b}; infos: (slot, vote_round, (n_cmds, cmd_len)) or (slot, vote_round, value bytes)"""
    m = cls("LeaderInbound")()
    p = m.phase1b
    p.group_index, p.acceptor_index, p.round = group, acceptor, round_
    for slot, vr, shape in infos:
        i = p.info.add()
        i.slot, i.vote_round = slot, vr
        if isinstance(shape, bytes):
            i.vote_value.ParseFromString(shape)
        else:
            i.vote_value.CopyFrom(payload(g, *shape))
    return m.SerializeToString()


def member(name, **fields):
    m = cls("LeaderInbound")()
    getattr(m, name).SetInParent()
    for k, v in fields.items():
        setattr(getattr(m, name), k, v)
    return m.SerializeToString()


def next_classic_round(n, leader, round_):
    """ClassicRoundRobin(n).nextClassicRound (RoundSystem.scala:66-80)"""
    if round_ < 0:
        return leader
    smallest = n * (round_ // n)
    return smallest + leader % n if smallest + leader % n > round_ else smallest + n + leader % n


def leader(msgs, f, lgroups, agroups, per_group, leader_group, round_, cw, recover_slot):
    """Leader.handlePhase1b over runtime-parsed LeaderInbounds, one at a time -> (status, index, result) with result
    (max_slot, next_slot, [(slot, vote value bytes or None)]) at completion, else None."""
    held = [dict() for _ in range(agroups)]
    for i, raw in enumerate(msgs):
        m = cls("LeaderInbound")()
        try:
            m.ParseFromString(raw)
        except Exception:
            return -15, i, None
        if not m.IsInitialized():
            return -15, i, None
        if m.WhichOneof("request") != "phase1b":
            continue
        p = m.phase1b
        if p.round != round_:
            if p.round > round_:
                return -14, i, None               # logger.checkLt
            continue
        if not (0 <= p.group_index < agroups and 0 <= p.acceptor_index < per_group):
            return -5, i, None
        held[p.group_index][p.acceptor_index] = p
        if any(len(h) < f + 1 for h in held):
            continue
        mx = max(max(max((x.slot for x in p1.info), default=-1) for p1 in h.values()) for h in held)
        mx = max(mx, recover_slot)
        if mx != -1 and mx % lgroups != leader_group:
            return -14, i, None                   # logger.check
        nxt = next_classic_round(lgroups, leader_group, mx)
        if nxt > (1 << 31) - 1:
            return -6, i, None
        out = []
        for s in range(next_classic_round(lgroups, leader_group, cw - 1), mx + 1, lgroups):
            group = held[(s // lgroups) % agroups]
            best = None
            for a in sorted(group):
                x = next((x for x in group[a].info if x.slot == s), None)
                if x is not None and (best is None or x.vote_round > best.vote_round):
                    best = x
            out.append((s, None if best is None else best.vote_value.SerializeToString()))
        return 0, i, (mx, nxt, out)
    return 0, -1, None


def acceptor(states, acc_round, engine_group, index, agroups, raw_phase1a):
    """Acceptor.handlePhase1a: states {slot: (vote_round, value bytes)} -> (new round, LeaderInbound bytes)"""
    p = cls("Phase1a")()
    p.ParseFromString(raw_phase1a)
    m = cls("LeaderInbound")()
    if p.round < acc_round:
        m.nack.round = acc_round
        return acc_round, m.SerializeToString()
    b = m.phase1b
    b.group_index, b.acceptor_index, b.round = engine_group % agroups, index, p.round
    for s in sorted(states):
        if s >= p.chosen_watermark:
            x = b.info.add()
            x.slot, x.vote_round = s, states[s][0]
            x.vote_value.ParseFromString(states[s][1])
    return p.round, m.SerializeToString()


def cases():
    g = np.random.Generator(np.random.PCG64(20261019))

    def quorum(round_, skip=()):
        """empty Phase1bs from acceptors 1 and 2 of both acceptor groups (not those in skip)"""
        return [phase1b(g, ag, a, round_, []) for ag in range(AG) for a in (1, 2) if (ag, a) not in skip]

    out = []

    def add(name, msgs, leader_group=1, round_=7, cw=0, recover_slot=-1):
        st, idx, res = leader(msgs, FC, LG, AG, PER_GROUP, leader_group, round_, cw, recover_slot)
        c = {"name": name, "msgs": [m.hex() for m in msgs], "leader_group": leader_group, "round": round_,
             "chosen_watermark": cw, "recover_slot": recover_slot, "status": st, "index": idx}
        if res is not None:
            c.update(max_slot=res[0], next_slot=res[1],
                     records=[[s, None if v is None else v.hex()] for s, v in res[2]])
        out.append(c)

    add("empty phase1bs", quorum(7))
    add("empty phase1bs, leader group 0, a watermark", quorum(7), leader_group=0, cw=5)
    votes = [(1, 3, (1, 10)), (4, 2, (-1, 0)), (7, 6, (2, 20)), (13, 1, (1, 5))]
    add("votes of both acceptor groups", [phase1b(g, 0, 0, 7, votes[:2] + votes[3:]), phase1b(g, 1, 0, 7, votes[2:3])]
        + quorum(7, skip={(0, 2), (1, 2)}))
    add("a nack parsed as field 7", [member("nack", round=9)] + quorum(7))
    add("a recover member replacing a phase1b", [phase1b(g, 0, 0, 7, [(1, 1, (1, 3))]) + member("recover", slot=4)]
        + quorum(7))
    add("a chosen_watermark member replacing a phase1b",
        [phase1b(g, 0, 0, 7, [(1, 1, (1, 3))]) + member("chosen_watermark")] + quorum(7))
    add("two phase1b members merging", [phase1b(g, 0, 0, 6, [(1, 4, (1, 8))]) + phase1b(g, 0, 0, 7, [(7, 4, (2, 3))])]
        + quorum(7, skip={(0, 2)}))
    add("a stale round is ignored", [phase1b(g, 0, 0, 5, [(19, 1, (1, 3))])] + quorum(7))
    add("a higher round", [phase1b(g, 0, 0, 8, [])] + quorum(7))
    add("an acceptor group outside the leader group", [phase1b(g, AG, 0, 7, [])] + quorum(7))
    add("an info slot of another leader group", [phase1b(g, 0, 0, 7, [(1, 1, (1, 3)), (5, 1, (1, 3))])] + quorum(7))
    add("an info slot of another leader group below the max", [phase1b(g, 0, 0, 7, [(2, 1, (1, 3)), (13, 1, (1, 3))])]
        + quorum(7))
    add("a recover_slot beyond every info", [phase1b(g, 0, 0, 7, [(1, 2, (1, 6))])] + quorum(7), recover_slot=19)
    add("a recover_slot of another group", quorum(7), recover_slot=18)
    add("a recover_slot and no votes", quorum(7), leader_group=2, recover_slot=2)
    add("ties go to the lowest acceptor index", [phase1b(g, 0, 2, 7, [(1, 3, (1, 4))]), phase1b(g, 0, 1, 7, [(1, 3, (1, 5))])]
        + quorum(7, skip={(0, 1), (0, 2)}))
    add("the first info of a slot", [phase1b(g, 0, 0, 7, [(1, 3, (1, 4)), (1, 5, (1, 9))])] + quorum(7))
    add("incomplete", quorum(7)[:-1])
    add("malformed", quorum(7)[:1] + [b"\x0a\x05\x08"])
    return out


def main():
    g = np.random.Generator(np.random.PCG64(20261020))
    leader_cases = cases()
    enc = []
    for slot, rnd, shape in [(0, 0, (-1, 0)), (4, 2, (1, 10)), (127, 128, (2, 60)), ((1 << 31) - 1, -1, (1, 200)),
                             (301, 16384, (0, 0))]:
        v = payload(g, *shape)
        m = cls("ProxyLeaderInbound")(phase2a=cls("Phase2a")(slot=slot, round=rnd, command_batch_or_noop=v))
        enc.append({"slot": slot, "round": rnd, "noop": shape[0] < 0, "payload_hex": v.SerializeToString().hex(),
                    "hex": m.SerializeToString().hex()})
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "wire_mencius_phase1.json")
    json.dump({"generator": "tests/golden/make_wire_mencius_phase1_golden.py (python protobuf runtime "
                            + __import__("google.protobuf").protobuf.__version__ + ")",
               "config": {"f": FC, "lgroups": LG, "agroups": AG, "per_group": PER_GROUP},
               "leader": leader_cases, "phase2a": enc}, open(out, "w"), indent=0)
    print(len(leader_cases), "+", len(enc), "cases ->", out)


if __name__ == "__main__":
    main()
