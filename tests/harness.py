"""Differential harness: drive the CUDA engine (through the C ABI) and the CPU
oracle with the same delivery trace and compare every observable bit-exactly."""
import numpy as np

from frankenpaxos_b200 import CHOSEN, NACK, P2A, P2B, Engine, FpxError
from frankenpaxos_b200 import traces as T
from oracle import fpx_oracle_py as O

# Quorum systems on both sides of every proxy-leader row size.  A row is {round, value, one stamp per
# voter} padded to 8, 16 or 32 words, i.e. at most 6, 14 or 30 voters per slot (fpx_create).
WIDE_SHAPES = {
    # 7 voters: the smallest 16-word row
    "maj7": dict(f=3, num_acceptor_groups=1, acceptors_per_group=7, flexible=False, num_leaders=4, num_replicas=4),
    # 14 voters: a full 16-word row
    "grid2x7": dict(f=1, num_acceptor_groups=2, acceptors_per_group=7, flexible=True, num_leaders=2, num_replicas=2),
    # 15 voters: the smallest 32-word row
    "maj15": dict(f=7, num_acceptor_groups=1, acceptors_per_group=15, flexible=False, num_leaders=8, num_replicas=8),
    # 15 voters per slot in two groups: 30 acceptors, 32-word rows
    "groups2x15": dict(f=7, num_acceptor_groups=2, acceptors_per_group=15, flexible=False, num_leaders=8,
                       num_replicas=8),
    # 29 voters, 32-word rows
    "maj29": dict(f=14, num_acceptor_groups=1, acceptors_per_group=29, flexible=False, num_leaders=15,
                  num_replicas=15),
    # 30 voters: a full 32-word row
    "grid5x6": dict(f=1, num_acceptor_groups=5, acceptors_per_group=6, flexible=True, num_leaders=2, num_replicas=2),
}


def voters(cfg):
    return cfg["num_acceptor_groups"] * cfg["acceptors_per_group"] if cfg["flexible"] else cfg["acceptors_per_group"]


def row_words(cfg):
    v = voters(cfg)
    return 8 if v <= 6 else (16 if v <= 14 else 32)


def make_pair(cfg, slot_capacity, max_batch=1 << 16, overflow_capacity=1 << 8, tally_max_sub=0, **kw):
    """tally_max_sub > 0: the engine cuts every tally call into launches of at most that many votes."""
    eng = Engine(slot_capacity=slot_capacity, max_batch=max_batch, overflow_capacity=overflow_capacity,
                 **cfg, **kw)
    if tally_max_sub:
        eng.set_tally_max_sub(tally_max_sub)
    ora = O.MultiPaxos(cfg["f"], cfg["num_acceptor_groups"], cfg["acceptors_per_group"],
                       cfg.get("flexible", False), cfg.get("num_leaders"), cfg.get("num_replicas"))
    return eng, ora


def same(a, b, what):
    assert a.dtype == b.dtype, what
    assert len(a) == len(b), f"{what}: lengths {len(a)} != {len(b)}"
    if len(a) and not np.array_equal(a, b):
        bad = np.nonzero(a != b)[0]
        raise AssertionError(f"{what}: first mismatch at {bad[0]}: engine {a[bad[0]]} oracle {b[bad[0]]} "
                             f"({len(bad)} of {len(a)} differ)")


def arm(eng, ora, recs):
    st, idx = ora.arm(recs)
    try:
        eng.proxyleader_arm(recs)
        est, eidx = 0, -1
    except FpxError as e:
        est, eidx = e.status, e.index
    assert (est, eidx) == (st, idx), f"arm status: engine {(est, eidx)} oracle {(st, idx)}"
    return st


def phase2a(eng, ora, recs):
    st, idx, ob, on = ora.acceptor_phase2a(recs)
    try:
        eb, en = eng.acceptor_phase2a(recs)
        est, eidx = 0, -1
    except FpxError as e:
        est, eidx = e.status, e.index
        eb = en = None
    assert (est, eidx) == (st, idx), f"phase2a status: engine {(est, eidx)} oracle {(st, idx)}"
    if st == 0:
        same(eb, ob, "Phase2b stream")
        same(en, on, "Nack stream")
    return ob, on


def phase2b(eng, ora, recs):
    st, idx, oc = ora.proxyleader_phase2b(recs)
    try:
        ec = eng.proxyleader_phase2b(recs)
        est, eidx = 0, -1
    except FpxError as e:
        est, eidx = e.status, e.index
        ec = None
    assert (est, eidx) == (st, idx), f"phase2b status: engine {(est, eidx)} oracle {(st, idx)}"
    if st == 0:
        same(ec, oc, "Chosen stream")
    return st, oc


def replica(eng, ora, chosen):
    ora.replica_chosen(chosen)
    eng.replica_chosen(chosen)
    assert eng.chosen_watermark() == ora.executed_watermark()


def compare_acceptors(eng, ora, cfg, first_slot, n_slots):
    for g in range(cfg["num_acceptor_groups"]):
        for a in range(cfg["acceptors_per_group"]):
            er, em, evr, evv = eng.snapshot_acceptor(g, a, first_slot, n_slots)
            orr, om, ovr, ovv = ora.snapshot_acceptor(g, a, first_slot, n_slots)
            assert (er, em) == (orr, om), f"acceptor ({g},{a}) round/maxVotedSlot {(er, em)} vs {(orr, om)}"
            same(evr, ovr, f"acceptor ({g},{a}) voteRound")
            same(evv, ovv, f"acceptor ({g},{a}) voteValue")


def compare_log(eng, ora, first_slot, n_slots):
    same(eng.snapshot_log(first_slot, n_slots), ora.snapshot_log(first_slot, n_slots), "replica log")


def adversarial(cfg, seed, n_slots, kmax, coop_ctas_per_sm=0, max_batch=1 << 16, tally_max_sub=0):
    """Random rounds (stale and fresh), duplicate deliveries, late votes, several live rounds per slot (so
    armed rows move to the overflow table), non-thrifty fan-out, many small and large batches; every
    acceptor and the replica log compared after each phase."""
    g = T.rng(seed)
    eng, ora = make_pair(cfg, n_slots, max_batch=max_batch, overflow_capacity=1 << 13 if n_slots <= 3000 else 1 << 20,
                         tally_max_sub=tally_max_sub)
    eng.set_coop_ctas_per_sm(coop_ctas_per_sm)
    for phase in range(4):
        k = int(g.integers(1, kmax))
        slots = g.integers(0, n_slots, size=k).astype(np.int32)
        rounds = g.integers(0, 4, size=k).astype(np.int32) if phase else np.zeros(k, dtype=np.int32)
        values = (slots * 8 + rounds).astype(np.int32)   # one value per (slot, round)
        a = T.arms(slots, 0, values)
        a["round"] = rounds
        arm(eng, ora, a)
        p = T.phase2as(g, slots, cfg["f"], cfg["num_acceptor_groups"], cfg["acceptors_per_group"],
                       cfg["flexible"], rounds, values, thrifty=bool(g.integers(0, 2)))
        p = p[g.permutation(len(p))]
        dup = p[g.integers(0, len(p), size=len(p) // 10)]
        p = np.concatenate([p, dup])[g.permutation(len(p) + len(dup))]
        votes = []
        for chunk in np.array_split(p, int(g.integers(1, 4))):
            ob, on = phase2a(eng, ora, chunk)
            votes.append(ob)
        compare_acceptors(eng, ora, cfg, 0, n_slots)
        v = np.concatenate(votes)
        v = np.concatenate([v, v[g.integers(0, max(len(v), 1), size=len(v) // 5)]]) if len(v) else v
        v = v[g.permutation(len(v))]
        for chunk in np.array_split(v, int(g.integers(1, 6))):
            st, c = phase2b(eng, ora, chunk)
            assert st == 0
            replica(eng, ora, c)
    compare_log(eng, ora, 0, n_slots)
    eng.close()
