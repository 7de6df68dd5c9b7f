"""The arm's fresh-key certificate at the seams of its pass-1 geometry, and the fresh frontier through every engine
call, against the CPU model (arm_fresh_model.py) and the oracle.

Pass 1 of arm_kernel<true> compares every adjacent pair of the batch by a warp shuffle inside a 32-record chunk,
by lane 31's look-ahead load across chunks, warps' unroll groups, CTAs and grid strides; a batch it wrongly
certifies does not fault but silently arms the wrong state.  So every violation is placed at each kind of seam,
every arm asserts the path the model predicts (Engine.last_arm_path), and every batch's keys are voted afterwards
and the Chosen stream and the replica log compared with the oracle's, on both tally paths.  Marked gpu."""
import numpy as np
import pytest

import arm_fresh_model as M
import harness as H
from frankenpaxos_b200 import CHOSEN, MENCIUS, P2A, P2A_RANGE, P2B, P2B_RANGE, VANILLA_MENCIUS, Engine, FpxError
from frankenpaxos_b200 import traces as T
from oracle import fpx_oracle_py as O

pytestmark = pytest.mark.gpu

ERR_SLOT_RANGE, ERR_ROUND_RANGE = -6, -7


@pytest.fixture(autouse=True, params=["auto", "exact"])
def tally_path(request, monkeypatch):
    monkeypatch.setenv("FPX_TALLY_PATH", request.param)
    return request.param


CFG2 = T.config_by_name("cfg2")[0]
N_EDGE = 3 * M.GRID_CTA + 1013          # 4 CTAs, a first pass-1 stride of 16 384 records, n % 32 != 0
PAIR_AT = (0, 30, M.CHUNK - 1, M.WARP_GROUP - 1, M.CERT_CTA - 1, 4 * M.CERT_CTA - 1, N_EDGE - 2)
ONE_AT = (0, M.CHUNK - 1, M.CHUNK, M.CERT_CTA, 4 * M.CERT_CTA, N_EDGE - 1)


def grid(cfg):
    return cfg["f"], cfg["num_acceptor_groups"], cfg["acceptors_per_group"], cfg["flexible"]


def oracle(cfg):
    return O.MultiPaxos(*grid(cfg), cfg["num_leaders"], cfg["num_replicas"])


def num_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def arm(eng, ora, fr, recs, want=None):
    """One arm call: its status is the oracle's and its path the model's (and `want`, when given)."""
    H.arm(eng, ora, recs)
    path = fr.arm(recs)
    assert eng.last_arm_path == path, f"arm of {len(recs)} records took {eng.last_arm_path}, model {path}"
    if want is not None:
        assert path == want
    return path


def arm_fails(eng, fr, recs, status, index):
    """An arm the engine refuses with (status, index) on the per-record path; the engine is reset afterwards
    (a failed call is fatal)."""
    with pytest.raises(FpxError) as ei:
        eng.proxyleader_arm(recs)
    assert (ei.value.status, ei.value.index) == (status, index)
    assert fr.arm(recs) == "cas" and eng.last_arm_path == "cas"
    eng.reset()
    fr.reset()


def key_votes(cfg, g, slots, rounds):
    """a full quorum of Phase2bs for every key (slot, round)"""
    return T.votes_of(T.phase2as(g, slots, *grid(cfg), np.asarray(rounds, dtype=np.int32), values=slots))


def probe(eng, ora, fr, cfg, g, slots, rounds=0, first=None, count=None, max_sub=0):
    """Votes a full quorum for every key (slot, round), shuffled, through the tally (cut into launches of at most
    max_sub votes), the Chosen stream to the replica; Chosen stream, watermark and log against the oracle."""
    slots = np.asarray(slots, dtype=np.int32)
    rounds = np.broadcast_to(np.asarray(rounds, dtype=np.int32), slots.shape)
    v = T.shuffled(g, key_votes(cfg, g, slots, rounds))
    eng.set_tally_max_sub(max_sub)
    st, c = H.phase2b(eng, ora, v)
    assert st == 0
    fr.tally(v)
    H.replica(eng, ora, c)
    lo = int(slots.min()) if first is None else first
    H.compare_log(eng, ora, lo, (int(slots.max()) + 1 - lo) if count is None else count)
    return c


def ordered(slots, rnd=0):
    slots = np.asarray(slots, dtype=np.int32)
    return T.arms(slots, rnd, slots * 3 + 1)


# --------------------------------------------------------------------------- a. pair violations at every seam
def pair_case(kind, base, i):
    """base with the pair (i, i + 1) broken; -> (batch, keys to vote as (slots, rounds))"""
    b = base.copy()
    if kind == "same_value":
        b[i + 1] = b[i]
    elif kind == "other_value":
        b[i + 1] = b[i]
        b["value_id"][i + 1] = b["value_id"][i] + 7          # first in delivery order wins
    elif kind == "second_round":
        b[i + 1] = b[i]
        b["round"][i + 1] = 1
        b["value_id"][i + 1] = b["value_id"][i] + 5
    else:
        b[[i, i + 1]] = b[[i + 1, i]]
    keys = np.unique(b[["slot", "round"]])
    return b, keys["slot"].astype(np.int32), keys["round"].astype(np.int32)


@pytest.mark.parametrize("kind", ["same_value", "other_value", "second_round", "swapped"])
def test_pair_violation_at_every_seam(kind):
    """A ragged batch of 3 * 8192 + 1013 records (4 CTAs, two pass-1 strides) with one broken pair at each seam:
    inside a chunk, lane 31's look-ahead, warp 0's unroll group to warp 1, CTA 0 to CTA 1, the first grid stride
    to the second, the last pair of the partial chunk.  Its twin without the violation takes the fast path, the
    broken batch the CAS; then every key of the batch (both rounds of a second-round slot) gets a full quorum."""
    cfg = CFG2
    n = N_EDGE
    assert M.cert_stride(n, num_sms()) == 4 * M.CERT_CTA
    eng = Engine(slot_capacity=1 << 15, max_batch=1 << 17, overflow_capacity=1 << 8, **cfg)
    fr = M.Frontier(M.MULTIPAXOS, M.Geometry(1 << 15))
    g = T.rng(100 + len(kind))
    base = ordered(np.arange(n))
    for i in PAIR_AT:
        ora = oracle(cfg)
        arm(eng, ora, fr, base, "fresh")
        eng.reset(); fr.reset()
        ora = oracle(cfg)
        b, slots, rounds = pair_case(kind, base, i)
        assert arm(eng, ora, fr, b) == "cas", f"pair ({i}, {i + 1})"
        c = probe(eng, ora, fr, cfg, g, slots, rounds, first=0, count=n)
        if kind == "other_value":
            assert c[c["slot"] == i]["value_id"].tolist() == [b["value_id"][i]]
        eng.reset(); fr.reset()
    eng.close()


# --------------------------------------------------------------------------- b. single-record violations
def test_single_record_errors_at_every_seam():
    """A round above FPX_MAX_ROUND at record i; a slot beyond the window as the last record i of a batch; on a
    3-shard engine a slot of another shard at record i of an ordered batch.  Each is refused with its error at
    index i by the CAS path, and the engine is reset."""
    cfg = CFG2
    n = N_EDGE
    cap = 1 << 15
    eng = Engine(slot_capacity=cap, max_batch=1 << 17, overflow_capacity=1 << 8, **cfg)
    fr = M.Frontier(M.MULTIPAXOS, M.Geometry(cap))
    base = ordered(np.arange(n))
    for i in ONE_AT:
        b = base.copy()
        b["round"][i] = M.MAX_ROUND + 1
        arm_fails(eng, fr, b, ERR_ROUND_RANGE, i)
        b = base[: i + 1].copy()
        b["slot"][i] = cap
        arm_fails(eng, fr, b, ERR_SLOT_RANGE, i)
    eng.close()
    eng = Engine(slot_capacity=3 * cap, max_batch=1 << 17, overflow_capacity=1 << 8, shard_index=1, shard_count=3,
                 **cfg)
    fr = M.Frontier(M.MULTIPAXOS, M.Geometry(3 * cap, 1, 3))
    base = ordered(3 * np.arange(n) + 1)
    ora = oracle(cfg)
    arm(eng, ora, fr, base, "fresh")
    eng.reset(); fr.reset()
    for i in ONE_AT:
        b = base.copy()
        b["slot"][i] += 1                     # shard 2's slot, still in order
        arm_fails(eng, fr, b, ERR_SLOT_RANGE, i)
    eng.close()


@pytest.mark.parametrize("k", [1, M.CHUNK, M.CERT_CTA + 1])
def test_prefix_below_the_frontier_or_retired(k):
    """An ordered batch whose first k records lie below the fresh frontier (keys armed by an earlier batch), and
    one whose first k records are retired slots: no error, the CAS path, and every key votes as in the oracle."""
    cfg = CFG2
    n = N_EDGE
    cap = 1 << 15
    g = T.rng(200 + k)
    eng = Engine(slot_capacity=cap, max_batch=1 << 17, overflow_capacity=1 << 8, **cfg)
    fr = M.Frontier(M.MULTIPAXOS, M.Geometry(cap))
    ora = oracle(cfg)
    arm(eng, ora, fr, ordered(np.arange(k)), "fresh")
    assert arm(eng, ora, fr, ordered(np.arange(n))) == "cas"
    probe(eng, ora, fr, cfg, g, np.arange(n))
    eng.reset(); fr.reset()
    ora = oracle(cfg)
    W = 5000
    arm(eng, ora, fr, ordered(np.arange(W)), "fresh")
    probe(eng, ora, fr, cfg, g, np.arange(W))
    eng.retire_below(W); fr.retire_below(W)
    s = np.arange(W - k, W - k + n)
    assert arm(eng, ora, fr, ordered(s)) == "cas"
    probe(eng, ora, fr, cfg, g, s[k:], first=W, count=n - k)
    eng.close()


# --------------------------------------------------------------------------- c. full size and the SM cap
def test_million_keys_in_order_then_shuffled_with_repeats_and_second_rounds():
    """2^20 records in slot order: the fast path over 128 CTAs.  Then, on the reset engine, the same number of
    records shuffled, about 1 % of them a repeated key and 1 % a second round of a slot: the certifying kernel's
    6-deep CAS fallback over 128 CTAs.  1000 of the repeats carry another value: one batch may hold at most
    kMaxConflicts (1024) of those (FPX_ERR_CONFLICT beyond).  Both bit-exact against the oracle after every key
    is voted."""
    cfg = CFG2
    N = 1 << 20
    g = T.rng(300)
    assert M.arm_blocks(N, num_sms()) == 128
    eng = Engine(slot_capacity=N, max_batch=1 << 22, overflow_capacity=1 << 16, **cfg)
    fr = M.Frontier(M.MULTIPAXOS, M.Geometry(N))
    ora = oracle(cfg)
    arm(eng, ora, fr, ordered(np.arange(N)), "fresh")
    probe(eng, ora, fr, cfg, g, np.arange(N))
    eng.reset(); fr.reset()
    ora = oracle(cfg)
    m = N // 100
    keys = np.arange(N - 2 * m, dtype=np.int32)
    rep = g.choice(keys, size=m, replace=False)
    sec = g.choice(keys, size=m, replace=False)
    other = np.arange(m) < 1000
    b = np.concatenate([ordered(keys), T.arms(rep, 0, rep * 3 + 1 + other), T.arms(sec, 1, sec * 3 + 9)])
    b = b[g.permutation(N)]
    assert len(b) == N
    arm(eng, ora, fr, b, "cas")
    c = probe(eng, ora, fr, cfg, g, np.concatenate([keys, sec]), np.concatenate([np.zeros(len(keys)), np.ones(m)]),
              first=0, count=len(keys))
    assert len(c) == len(keys) + m
    eng.close()


def test_batch_past_the_sm_cap():
    """num_sms * 8192 + 4097 records: the grid is capped at the SM count, so both passes and the fallback run
    grid-stride loops.  In order: the fast path; with one swapped pair at the end of pass 1's first stride and
    one as the last pair: the CAS path.  Every key voted, bit-exact."""
    cfg = CFG2
    sms = num_sms()
    n = sms * M.GRID_CTA + 4097
    assert M.arm_blocks(n, sms) == sms
    g = T.rng(400)
    cap = 1 << 21
    eng = Engine(slot_capacity=cap, max_batch=1 << 22, overflow_capacity=1 << 8, **cfg)
    fr = M.Frontier(M.MULTIPAXOS, M.Geometry(cap))
    base = ordered(np.arange(n))
    ora = oracle(cfg)
    arm(eng, ora, fr, base, "fresh")
    probe(eng, ora, fr, cfg, g, np.arange(n))
    eng.reset(); fr.reset()
    ora = oracle(cfg)
    b = base.copy()
    for i in (sms * M.CERT_CTA - 1, n - 2):
        b[[i, i + 1]] = b[[i + 1, i]]
    arm(eng, ora, fr, b, "cas")
    probe(eng, ora, fr, cfg, g, np.arange(n))
    eng.close()


# --------------------------------------------------------------------------- d. the frontier through every call
SEQ_SHAPES = {
    "cfg2": (CFG2, 0, 1),
    "cfg2_shard1of2": (CFG2, 1, 2),
    "grid5x6": (H.WIDE_SHAPES["grid5x6"], 0, 1),       # 30 voters, 32-word rows
}


class Sequence:
    """One engine, its oracle and its model under a random sequence of calls.  Slots are handled as this shard's
    ordinals u (slot = u * shard_count + shard_index); the value of key (u, r) is u * 8 + r."""

    def __init__(self, cfg, idx, cnt, local_slots, g):
        self.cfg, self.idx, self.cnt, self.g = cfg, idx, cnt, g
        cap = local_slots * cnt
        self.eng = Engine(slot_capacity=cap, max_batch=1 << 15, overflow_capacity=1 << 13, shard_index=idx,
                          shard_count=cnt, **cfg)
        self.geo = M.Geometry(cap, idx, cnt)
        self.fr = M.Frontier(M.MULTIPAXOS, self.geo)
        assert self.geo.local_slots == local_slots
        self.fresh()

    def fresh(self):
        self.ora = oracle(self.cfg)
        self.round = {}              # ordinal -> its largest armed round
        self.open = set()            # keys (ordinal, round) armed and not voted yet
        self.next = 0                # one past the largest ordinal ever armed

    @property
    def base(self):
        return self.geo.base_local

    @property
    def end(self):
        return self.geo.base_local + self.geo.local_slots

    def slot(self, u):
        return (np.asarray(u, dtype=np.int64) * self.cnt + self.idx).astype(np.int32)

    def arm(self, us, rounds):
        us = np.asarray(us, dtype=np.int64)
        rounds = np.broadcast_to(np.asarray(rounds, dtype=np.int32), us.shape)
        recs = T.arms(self.slot(us), 0, (us * 8 + rounds).astype(np.int32))
        recs["round"] = rounds
        path = arm(self.eng, self.ora, self.fr, recs)
        for u, r in zip(us.tolist(), rounds.tolist()):
            if r > self.round.get(u, -1):
                self.round[u] = r
                self.open.add((u, r))
        self.next = max(self.next, int(us.max()) + 1)
        return path

    def vote(self, frac, max_sub):
        keys = sorted(self.open)
        if not keys:
            return
        take = [keys[j] for j in np.nonzero(self.g.random(len(keys)) < frac)[0]] or keys[:1]
        us = np.array([k[0] for k in take])
        rs = np.array([k[1] for k in take], dtype=np.int32)
        v = T.shuffled(self.g, key_votes(self.cfg, self.g, self.slot(us), rs))
        if self.g.random() < 0.3:                                        # re-deliveries
            v = np.concatenate([v, v[self.g.integers(0, len(v), size=len(v) // 4)]])
        self.eng.set_tally_max_sub(max_sub)
        st, c = H.phase2b(self.eng, self.ora, v)
        assert st == 0
        self.fr.tally(v)
        if self.cnt == 1:
            H.replica(self.eng, self.ora, c)
        else:                       # the oracle sees this shard's slots only: its watermark is not the shard's
            self.ora.replica_chosen(c)
            self.eng.replica_chosen(c)
        self.open.difference_update(take)

    def compare(self):
        first = int(self.slot(self.base))
        last = int(self.slot(max(self.base, self.next - 1)))
        H.compare_log(self.eng, self.ora, first, last - first + 1)


@pytest.mark.parametrize("shape", list(SEQ_SHAPES))
def test_frontier_through_random_call_sequences(shape):
    """300 random calls on a ring of 3007 rows (not a multiple of 32, so recycled windows wrap it in the middle
    of a chunk): ordered arms of new slots (some with gaps), ordered arms that straddle the frontier (filling the
    gaps), shuffled arms, second-round arms of live slots, vote batches (some cut into 1024-vote launches),
    retire_below up to the watermark, and reset.  Every arm's path is the model's; every vote and replica call
    matches the oracle, and the live log is compared before every retire and reset."""
    cfg, idx, cnt = SEQ_SHAPES[shape]
    g = T.rng(500 + len(shape) + idx)
    S = Sequence(cfg, idx, cnt, 3007, g)
    paths = {"fresh": 0, "cas": 0}
    retires = 0
    for _ in range(300):
        op = g.random()
        room = S.end - S.next
        if op < 0.25 and room > 0:                                       # ordered new slots, maybe with gaps
            us = S.next + np.arange(int(min(room, g.integers(1, 700))))
            if g.random() < 0.3 and len(us) > 4:
                us = np.sort(g.choice(us, size=len(us) // 2, replace=False))
            paths[S.arm(us, 0)] += 1
        elif op < 0.35 and S.next > S.base:                              # ordered across the frontier
            holes = [u for u in range(S.base, S.next) if u not in S.round]
            lo = holes[0] if holes and g.random() < 0.7 else max(S.base, S.fr.value - int(g.integers(1, 100)))
            hi = min(S.end, max(lo + 1, S.fr.value + int(g.integers(0, 300))))
            us = np.arange(lo, hi)
            paths[S.arm(us, [S.round.get(u, 0) for u in us.tolist()])] += 1
        elif op < 0.45 and room > 1:                                     # shuffled new slots
            us = S.next + np.arange(int(min(room, g.integers(2, 500))))
            paths[S.arm(us[g.permutation(len(us))], 0)] += 1
        elif op < 0.50:                                                  # a leader change for some live slots
            live = [u for u in S.round if u >= S.base]
            if live:
                us = np.sort(g.choice(live, size=min(len(live), int(g.integers(1, 20))), replace=False))
                paths[S.arm(us, [S.round[u] + 1 for u in us.tolist()])] += 1
        elif op < 0.85:                                                  # votes
            S.vote(float(g.uniform(0.3, 1.0)), 1024 if g.random() < 0.4 else 0)
        elif op < 0.98:                                                  # slide the window behind the watermark
            wm = S.eng.chosen_watermark()
            if wm > int(S.slot(S.base)):
                S.compare()
                S.eng.retire_below(wm)
                S.fr.retire_below(wm)
                S.open = {(u, r) for (u, r) in S.open if u >= S.base}
                retires += 1
        else:
            S.compare()
            S.eng.reset()
            S.fr.reset()
            S.fresh()
    S.compare()
    S.eng.close()
    assert paths["fresh"] >= 10 and paths["cas"] >= 10 and retires >= 3, (paths, retires)


def mencius_votes(slots, f, LG, AG, per, g):
    b = np.zeros(len(slots) * (f + 1), dtype=P2B)
    b["group"] = np.repeat((slots % LG) * AG + (slots // LG) % AG, f + 1)
    b["acceptor"] = np.array([g.permutation(per)[: f + 1] for _ in slots]).reshape(-1)
    b["slot"] = np.repeat(slots, f + 1)
    return b[g.permutation(len(b))]


def test_mencius_paths_around_one_slot_ranges():
    """Compartmentalized Mencius: ordered arms take the fast path, also after a multi-slot noop range; after a
    one-slot range every arm takes the CAS path (it must look the key up in the range table) until reset.  A
    later Phase2a of the key the one-slot range holds is ignored, as in the oracle: the range's votes still
    choose it."""
    f, LG, AG, per, cap = 1, 2, 1, 3, 8192
    g = T.rng(600)
    eng = Engine(f, AG, per, num_leaders=2, num_replicas=2, slot_capacity=cap, max_batch=1 << 15, protocol=MENCIUS,
                 num_leader_groups=LG)
    ora = O.MultiPaxos(f, AG, per, False, 2, 2, mencius_leader_groups=LG)
    fr = M.Frontier(M.MENCIUS, M.Geometry(cap))

    def arm_range(recs):
        r = np.array(recs, dtype=P2A_RANGE)
        st, err = ora.arm_range(r, cap)
        assert st == 0
        eng.mencius_arm_range(r)
        fr.arm_range(r)

    def vote(slots):
        v = mencius_votes(np.asarray(slots, dtype=np.int32), f, LG, AG, per, g)
        st, c = H.phase2b(eng, ora, v)
        assert st == 0
        fr.tally(v)
        H.replica(eng, ora, c)

    arm(eng, ora, fr, ordered(np.arange(0, 1000)), "fresh")
    vote(np.arange(0, 1000))
    arm_range([(1000, 1100, 0, -1)])
    arm(eng, ora, fr, ordered(np.arange(1100, 2000)), "fresh")
    arm_range([(2000, 2001, 0, -1)])                                     # one slot: shares the key space
    arm(eng, ora, fr, ordered(np.arange(2002, 3000)), "cas")
    arm(eng, ora, fr, T.arms([2000], 0, [77]), "cas")                    # the range holds (2000, 0): ignored
    v = np.array([(0, 2000, 2001, 0), (1, 2000, 2001, 0)], dtype=P2B_RANGE)   # group 0: slot 2000 % LG
    st, err, oc = ora.range_phase2b(v)
    assert st == 0 and oc.tolist() == [(2000, 2001)]
    H.same(eng.mencius_range_phase2b(v), oc, "ChosenNoopRange")
    vote(np.concatenate([np.arange(1100, 2000), np.arange(2002, 3000)]))
    H.compare_log(eng, ora, 0, 3000)
    eng.reset(); fr.reset()
    ora = O.MultiPaxos(f, AG, per, False, 2, 2, mencius_leader_groups=LG)
    arm(eng, ora, fr, ordered(np.arange(0, 3000)), "fresh")
    vote(np.arange(0, 3000))
    H.compare_log(eng, ora, 0, 3000)
    eng.close()


def test_vanilla_mencius_arms_take_the_plain_kernel():
    """Vanilla Mencius' client requests run the plain per-record kernel, ordered or not."""
    f = 1
    n = 2 * f + 1
    eng = Engine(f, 1, n, num_leaders=f + 1, num_replicas=f + 1, slot_capacity=8192, max_batch=1 << 15,
                 protocol=VANILLA_MENCIUS)
    ora = O.VanillaMencius(f)
    fr = M.Frontier(M.VANILLA, M.Geometry(8192))
    for lo, hi in ((0, 3000), (3000, 6000)):
        req = np.array([(s, 0, s + 100, s % n) for s in range(lo, hi)], dtype=P2A)
        assert ora.client_request(req) == (0, -1)
        eng.vm_client_request(req)
        assert eng.last_arm_path == fr.arm(req) == "cas"
    eng.close()


# --------------------------------------------------------------------------- e. the step forms
def _td(x):
    import torch
    return torch.from_numpy(x.view(np.int32).reshape(len(x), -1).copy()).to(torch.device("cuda", 0))


def test_bench_shaped_step_on_rebased_windows():
    """fpx_step_dev as bench.py drives it -- acceptor batch, the window's arm batch in slot order, the shuffled
    votes -- on windows re-based one after another through a ring of 3 windows that is retired behind the
    watermark: every step's arm batch takes the fast path, and every stream and the log are the oracle's."""
    import torch
    cfg = CFG2
    W = 8192 + 77
    eng = Engine(slot_capacity=3 * W, max_batch=1 << 16, overflow_capacity=1 << 8, **cfg)
    ora = oracle(cfg)
    fr = M.Frontier(M.MULTIPAXOS, M.Geometry(3 * W))
    dev = torch.device("cuda", 0)
    for w in range(6):
        a, p, b = T.workload(700 + w % 2, cfg, W, slot0=w * W)
        n = len(p)
        o_b = torch.zeros((n, 4), dtype=torch.int32, device=dev)
        o_n = torch.zeros((n, 2), dtype=torch.int32, device=dev)
        o_c = torch.zeros((len(b), 2), dtype=torch.int32, device=dev)
        d_wm = torch.zeros(1, dtype=torch.int32, device=dev)
        d_a, d_p, d_b = _td(a), _td(p), _td(b)
        eng.step_dev(d_a.data_ptr(), len(a), d_p.data_ptr(), n, o_b.data_ptr(), o_n.data_ptr(), d_b.data_ptr(),
                     len(b), o_c.data_ptr(), d_wm.data_ptr())
        r = eng.sync()
        assert eng.last_arm_path == fr.arm(a) == "fresh"
        fr.tally(b)
        st, _, ob, on = ora.acceptor_phase2a(p)
        assert st == 0 and len(on) == 0
        H.same(o_b.cpu().numpy().view(P2B).reshape(-1)[: r.n_p2b], ob, "Phase2b stream")
        assert ora.arm(a) == (0, -1)
        st, _, oc = ora.proxyleader_phase2b(b)
        assert st == 0
        H.same(o_c[: r.n_chosen].cpu().numpy().view(CHOSEN).reshape(-1),
               oc, "Chosen stream")
        ora.replica_chosen(oc)
        assert int(d_wm.item()) == ora.executed_watermark() == (w + 1) * W
        H.compare_log(eng, ora, w * W, W)
        if w >= 1:
            eng.retire_below(w * W)
            fr.retire_below(w * W)
    eng.close()


@pytest.mark.parametrize("explicit", [True, False])
def test_step_submit_arm_paths(explicit):
    """fpx_step_submit with an explicit arm batch in slot order takes the fast path.  With arm = None the step
    arms from its Phase2a batch, which repeats every slot once per acceptor it goes to: a repeated key, so that
    batch takes the CAS path by design -- the same keys, the state the oracle has."""
    import torch
    cfg = CFG2
    W = 6000
    eng = Engine(slot_capacity=2 * W, max_batch=1 << 16, overflow_capacity=1 << 8, **cfg)
    ora = oracle(cfg)
    fr = M.Frontier(M.MULTIPAXOS, M.Geometry(2 * W))
    pin = lambda r: torch.from_numpy(r.view(np.int32).reshape(len(r), -1).copy()).pin_memory()
    for w in range(2):
        a, p, b = T.workload(800 + w, cfg, W, slot0=w * W)
        arm_recs = a if explicit else p
        ha, hp, hb = pin(a), pin(p), pin(b)
        ob = torch.zeros((len(p), 4), dtype=torch.int32).pin_memory()
        on = torch.zeros((len(p), 2), dtype=torch.int32).pin_memory()
        oc = torch.zeros((len(b), 2), dtype=torch.int32).pin_memory()
        eng.step_submit(ha.data_ptr() if explicit else None, len(a) if explicit else 0, hp.data_ptr(), len(p),
                        hb.data_ptr(), len(b), ob.data_ptr(), on.data_ptr(), oc.data_ptr())
        n_p2b, n_nack, n_chosen, wm = eng.step_wait()
        want = fr.arm(arm_recs)
        assert want == ("fresh" if explicit else "cas") and eng.last_arm_path == want
        fr.tally(b)
        assert ora.arm(arm_recs) == (0, -1)
        st, _, eb, en = ora.acceptor_phase2a(p)
        assert st == 0 and (n_p2b, n_nack) == (len(eb), len(en))
        st, _, ec = ora.proxyleader_phase2b(b)
        assert st == 0 and n_chosen == len(ec)
        H.same(oc.numpy().view(CHOSEN).reshape(-1)[:n_chosen], ec,
               "Chosen stream")
        ora.replica_chosen(ec)
        assert wm == ora.executed_watermark()
        H.compare_log(eng, ora, w * W, W)
    eng.close()


@pytest.mark.parametrize("max_sub", [0, 1024])
def test_stray_vote_raises_the_frontier_past_the_arms(max_sub):
    """A vote for a slot nobody armed is fatal, but the tally has stamped it into the unarmed row: the frontier
    moves past it, above every armed row, and an ordered arm over that row takes the CAS path.  The stray vote is
    the first slot past the armed ones or 5000 slots beyond, in the last launch of a call cut into 1024-vote
    launches or in a one-launch call."""
    cfg = CFG2
    cap, k = 1 << 14, 3000
    g = T.rng(900 + max_sub)
    eng = Engine(slot_capacity=cap, max_batch=1 << 15, overflow_capacity=1 << 8, **cfg)
    eng.set_tally_max_sub(max_sub)
    fr = M.Frontier(M.MULTIPAXOS, M.Geometry(cap))
    for stray_slot in (k, k + 5000):
        ora = oracle(cfg)
        arm(eng, ora, fr, ordered(np.arange(k)), "fresh")
        v = T.shuffled(g, key_votes(cfg, g, np.arange(k, dtype=np.int32), np.zeros(k)))
        stray = np.zeros(1, dtype=P2B)
        stray[0] = (0, 1, stray_slot, 0)
        v = np.concatenate([v, stray])
        st, _ = H.phase2b(eng, ora, v)
        assert st == -4
        fr.tally(v)
        assert fr.value == stray_slot + 1
        arm(eng, oracle(cfg), fr, ordered(np.arange(k, k + 6000)), "cas")
        eng.reset(); fr.reset()
    eng.close()
