"""EPaxos and its execution side past one tile and one grid stride, against the oracle.

The multi-block code of these kernels only runs at sizes the other EPaxos tests do not reach:
  dependency graph   `dg_execute_kernel` walks its vertices in grid-stride loops (stride = SMs x 1024): at
                     key_capacity = 2^18 every vertex past the first stride is handled in a later iteration
                     than the vertices that depend on it
  conflict index     carries between 1024-access tiles (`tile_carry_kernel`): hot keys over ~128 tiles, segments
                     that end exactly on, one past and one short of a tile boundary, 16 columns (8 leaders), a
                     near-full table, and over 1024 tiles (the carry kernel's chunk of tiles)
  EPaxos handlers    the Nack's largestBallot carried from earlier 1024-record tiles and earlier batches, and the
                     E1 / E2 batch-contract detection across CTAs
  cfg4 round         one PreAccept round at 2^20 instances
The CPU test at the end checks the oracle's Tarjan itself against scipy on the dependency-graph workload."""
import time

import numpy as np
import pytest

from frankenpaxos_b200 import traces as T
from oracle import fpx_oracle_py as O

I32_MIN, I32_MAX = -(1 << 31), (1 << 31) - 1
H100_STRIDE = 132 * 1024            # grid stride of dg_execute_kernel on a 132-SM H100


def _stride():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count * 1024


def _raises(fn, *a, **k):
    from frankenpaxos_b200 import FpxError
    with pytest.raises(FpxError) as ei:
        fn(*a, **k)
    return ei.value.status, ei.value.index


# =========================================================================== dependency graph workload
class DgPlan:
    """A dependency-graph workload over keys [0, cap): round 0 commits ~150k keys in 64-key blocks (batches of at
    most 2^15, keys repeated inside a batch), rounds 1-3 commit some of the blockers and mark others executed.

    Dependencies: mostly lower keys of the same block (chains stay shorter than a block), a few long-range ones,
    planted cycles of sizes 1, 2, ... 500 (one of them across the stride boundary), dependencies on executed keys,
    on keys outside [0, cap), and on absent keys in [stride, cap) from vertices in [0, stride) -- the blocker a
    vertex of the first stride records for a vertex of the second.  Sequence numbers: many ties, negatives,
    INT32_MIN and INT32_MAX."""

    BLOCK = 64

    def __init__(self, seed, cap, stride):
        assert cap > stride
        g = np.random.Generator(np.random.PCG64(seed))
        self.g, self.cap, self.stride = g, cap, stride
        nb = cap // self.BLOCK
        blocks = np.sort(g.choice(nb, size=int(nb * 0.58), replace=False))
        in_block = np.zeros(cap, bool)
        in_block[(blocks[:, None] * self.BLOCK + np.arange(self.BLOCK)).ravel()] = True
        keys = np.nonzero(in_block)[0]
        # 1 % of the block keys are executed before anything is committed
        ex0 = g.choice(keys, size=len(keys) // 100, replace=False)
        self.executed0 = np.sort(ex0)
        live = np.ones(cap, bool); live[ex0] = False
        self.commit_keys = keys[live[keys]]
        absent = np.nonzero(~in_block)[0]
        self.absent_hi = g.choice(absent[absent >= stride], size=1500, replace=False)   # referenced from [0, stride)
        self.absent_lo = g.choice(absent[absent < stride], size=300, replace=False)     # referenced from [stride, cap)
        self.deps = {int(k): [] for k in self.commit_keys}
        ck = self.commit_keys
        # near dependencies: lower keys of the same block (committed or executed; an absent one would be a block key)
        for k in ck.tolist():
            lo = k - k % self.BLOCK
            if k > lo:
                nd = int(g.integers(0, 4))
                if nd:
                    self.deps[k].extend(sorted(set(int(x) for x in g.integers(lo, k, size=nd))))
        # planted cycles: k_i -> k_(i+1) -> ... -> k_0; one across the stride boundary
        self.cycles = []
        for size in [1] * 12 + [2] * 12 + [3, 5, 17, 17, 64, 200, 500]:
            self.cycles.append(g.choice(ck, size=size, replace=False))
        near = ck[(ck > stride - 2000) & (ck < stride + 2000)]
        self.cycles.append(np.concatenate([np.sort(near[near < stride])[-150:], np.sort(near[near >= stride])[:150]]))
        for cyc in self.cycles:
            cyc = cyc.tolist()
            for i, k in enumerate(cyc):
                self.deps[k].append(cyc[(i + 1) % len(cyc)])
        # what follows can block a vertex: kept out of the blocks the cycles live in (all but one 17-cycle stay
        # executable in round 0)
        cyc_block = np.zeros(nb, bool)
        cyc_block[np.concatenate(self.cycles) // self.BLOCK] = True
        free = ck[~cyc_block[ck // self.BLOCK]]
        # long-range dependencies, either direction, across strides too
        for k in g.choice(free, size=len(ck) // 300, replace=False).tolist():
            self.deps[k].append(int(g.choice(ck)))
        # absent keys of the second stride referenced from the first, and the other way round
        lo_keys, hi_keys = free[free < stride], free[free >= stride]
        self.hi_refs = g.choice(lo_keys, size=len(self.absent_hi), replace=False)
        for k, w in zip(self.hi_refs.tolist(), self.absent_hi.tolist()):
            self.deps[k].append(w)
        for k, w in zip(g.choice(hi_keys, size=len(self.absent_lo), replace=False).tolist(), self.absent_lo.tolist()):
            self.deps[k].append(w)
        self.deps[int(self.cycles[27][3])].append(int(self.absent_lo[0]))      # a blocked cycle
        # dependencies on executed keys, and on keys outside [0, cap)
        for k in g.choice(ck, size=3000, replace=False).tolist():
            self.deps[k].append(int(g.choice(self.executed0)))
        for k, w in zip(g.choice(free, size=6, replace=False).tolist(), [cap, cap + 7, -1, -100, I32_MAX, I32_MIN]):
            self.deps[k].append(w)
        for k in self.deps:
            self.deps[k] = sorted(set(self.deps[k]))
        self.seq = self.seqs(ck)

    def seqs(self, keys):
        g = self.g
        s = g.integers(-20, 21, size=len(keys)).astype(np.int64)
        u = g.random(len(keys))
        s[u < 0.05] = I32_MIN
        s[(u >= 0.05) & (u < 0.10)] = I32_MAX
        wide = (u >= 0.10) & (u < 0.15)
        s[wide] = g.integers(I32_MIN, I32_MAX, size=int(wide.sum()), endpoint=True)
        return dict(zip(keys.tolist(), s.tolist()))

    def round0_batches(self, max_batch=1 << 15):
        """Delivery batches: every committed key once, plus repeats (other seq / deps) that must be ignored --
        inside the same batch after the first delivery, and in later batches."""
        g = self.g
        order = g.permutation(self.commit_keys)
        out = []
        step = max_batch - max_batch // 16
        for b0 in range(0, len(order), step):
            ks = order[b0:b0 + step]
            rep = g.choice(order[:b0 + len(ks)], size=max_batch // 16)
            # delivery position: the originals in order, a repeat anywhere after its key's first delivery
            first = np.searchsorted(np.arange(b0, b0 + len(ks)), np.nonzero(np.isin(order, rep))[0])
            where = dict(zip(order[np.isin(order, rep)].tolist(), first.tolist()))
            pos = np.concatenate([np.arange(len(ks), dtype=float),
                                  [where[k] + 0.5 + g.random() * (len(ks) - where[k]) for k in rep.tolist()]])
            entries = [(k, self.seq[k], self.deps[k]) for k in ks.tolist()] + \
                      [(k, int(g.integers(-5, 5)), [int(g.integers(0, self.cap))]) for k in rep.tolist()]
            out.append([entries[j] for j in np.argsort(pos, kind="stable")])
        return out


class DgModel:
    """Committed / executed state of the workload, for the checks."""

    def __init__(self, cap):
        self.cap = cap
        self.status = np.zeros(cap, np.int8)        # 0 absent, 1 committed, 2 executed
        self.seq = np.zeros(cap, np.int64)
        self.src, self.dst = [], []

    def commit(self, batch):
        for k, s, d in batch:
            if 0 <= k < self.cap and self.status[k] == 0:
                self.status[k] = 1
                self.seq[k] = s
                self.src.append(np.full(len(d), k, np.int64)); self.dst.append(np.asarray(d, np.int64))

    def edges(self):
        return np.concatenate(self.src), np.concatenate(self.dst)

    def blockers(self):
        s, d = self.edges()
        ok = (d >= 0) & (d < self.cap)
        s, d = s[ok], d[ok]
        return np.unique(d[(self.status[s] == 1) & (self.status[d] == 0)])

    def check_execution(self, comps, blockers, ocomps, oblockers):
        """As test_depgraph_random_graphs_match_the_oracle, vectorised: the oracle's components (as sets, with
        the same member order) in a dependency-respecting order, and exactly the blockers computed here."""
        cap = self.cap
        assert sorted(map(tuple, comps)) == sorted(map(tuple, ocomps)), "components differ from the oracle's"
        want = self.blockers()
        got = np.asarray(blockers, np.int64)
        if not np.array_equal(got, want):
            miss, extra = np.setdiff1d(want, got), np.setdiff1d(got, want)
            raise AssertionError(f"blockers: {len(miss)} missing (first {miss[:8].tolist()}), "
                                 f"{len(extra)} extra (first {extra[:8].tolist()})")
        assert set(b for b in oblockers if 0 <= b < cap) <= set(got.tolist())
        flat = np.asarray([k for c in comps for k in c], np.int64)
        cid = np.repeat(np.arange(len(comps)), [len(c) for c in comps])
        assert (self.status[flat] == 1).all() and len(np.unique(flat)) == len(flat)
        # members by (seq, key)
        same = cid[1:] == cid[:-1]
        a, b = flat[:-1][same], flat[1:][same]
        sa, sb = self.seq[a], self.seq[b]
        assert ((sa < sb) | ((sa == sb) & (a < b))).all(), "member order is not (sequence number, key)"
        # every dependency of a member: executed before, in an earlier component or in the same one
        pos = np.full(cap, -1, np.int64)
        pos[flat] = cid
        s, d = self.edges()
        ok = (d >= 0) & (d < cap) & (pos[s] >= 0)
        s, d = s[ok], d[ok]
        good = (self.status[d] == 2) | ((pos[d] >= 0) & (pos[d] <= pos[s]))
        assert good.all(), f"{int((~good).sum())} dependencies violated, first {s[~good][0]} -> {d[~good][0]}"
        self.status[flat] = 2
        return len(flat)


def _dg_round0(plan, dg, ora, model):
    dg.update_executed(plan.executed0); ora.update_executed(plan.executed0.tolist())
    model.status[plan.executed0] = 2
    for batch in plan.round0_batches():
        dg.commit([k for k, _, _ in batch], [s for _, s, _ in batch], [d for _, _, d in batch])
        for k, s, d in batch:
            ora.commit(k, s, d)
        model.commit(batch)


def _dg_later_round(plan, dg, ora, model, blockers):
    """Commit half of the blockers (dependencies on committed, executed or other absent keys) and mark a quarter
    executed."""
    g = plan.g
    bl = g.permutation(np.asarray(blockers, np.int64))
    com, ex = bl[:len(bl) // 2], bl[len(bl) // 2:len(bl) // 2 + len(bl) // 4]
    if len(ex):
        dg.update_executed(ex); ora.update_executed(ex.tolist())
        model.status[ex] = 2
    known = np.nonzero(model.status > 0)[0]
    absent = np.nonzero(model.status == 0)[0]
    seqs = plan.seqs(com)
    batch = []
    for k in com.tolist():
        d = [int(x) for x in g.choice(known, size=int(g.integers(0, 3)))]
        if g.random() < 0.2:
            d.append(int(g.choice(absent)))
        batch.append((k, seqs[k], sorted(set(d))))
    for b0 in range(0, len(batch), 1 << 15):
        part = batch[b0:b0 + (1 << 15)]
        dg.commit([k for k, _, _ in part], [s for _, s, _ in part], [d for _, _, d in part])
    for k, s, d in batch:
        ora.commit(k, s, d)
    model.commit(batch)


@pytest.mark.gpu
def test_depgraph_beyond_one_grid_stride_matches_the_oracle():
    from frankenpaxos_b200.epaxos import DependencyGraph
    cap, stride = 1 << 18, _stride()
    assert cap > stride, (cap, stride)
    plan = DgPlan(7, cap, stride)
    assert (plan.absent_hi >= stride).all() and (plan.hi_refs < stride).all()
    dg = DependencyGraph(key_capacity=cap, dep_pool_capacity=1 << 21, max_batch=1 << 15)
    ora, model = O.TarjanDependencyGraph(), DgModel(cap)
    _dg_round0(plan, dg, ora, model)
    assert (model.status == 1).sum() > 140_000
    for rnd in range(4):
        if rnd:
            _dg_later_round(plan, dg, ora, model, blockers)
        comps, blockers = dg.execute_by_component()
        ocomps, oblockers = ora.execute_by_component(cap=cap)
        if rnd == 0:   # the planted pattern is there to be lost: blockers of the second stride, seen from the first
            assert len(np.intersect1d(blockers, plan.absent_hi)) == len(plan.absent_hi)
            assert max(len(c) for c in comps) >= 300
        n_exec = model.check_execution(comps, blockers, ocomps, oblockers)
        assert n_exec > (100_000 if rnd == 0 else 0), (rnd, n_exec)
    dg.close()


@pytest.mark.gpu
def test_depgraph_reverse_chain_across_the_grid_stride():
    """A chain over all of [0, 2^18) committed from the top down: nothing executes until key 0 arrives, then one
    component per key in key order (trim and levels take one grid barrier per link)."""
    from frankenpaxos_b200.epaxos import DependencyGraph
    cap = 1 << 18
    assert cap > _stride()
    dg = DependencyGraph(key_capacity=cap, dep_pool_capacity=cap, max_batch=1 << 15)
    keys = np.arange(cap - 1, 0, -1)
    for b0 in range(0, len(keys), 1 << 15):
        k = keys[b0:b0 + (1 << 15)]
        dg.commit(k, np.zeros(len(k), np.int32), [[x - 1] for x in k.tolist()])
    comps, blockers = dg.execute_by_component()
    assert comps == [] and blockers == [0]
    dg.commit([0], [0], [[]])
    t0 = time.perf_counter()
    comps, blockers = dg.execute_by_component()
    print(f"reverse chain of {cap} keys: execute_by_component {time.perf_counter() - t0:.2f} s")
    assert blockers == [] and len(comps) == cap
    assert all(len(c) == 1 for c in comps) and [c[0] for c in comps] == list(range(cap))
    assert dg.execute_by_component()[0] == []
    dg.close()


def test_oracle_components_are_the_strongly_connected_components():
    """The reference used above, at that scale: the oracle's components are exactly scipy's strongly connected
    components of the committed, eligible subgraph (dependencies on executed keys are not edges), and the keys it
    executes are exactly the eligible ones."""
    import scipy.sparse as sp
    from scipy.sparse.csgraph import connected_components
    cap = 1 << 18
    plan = DgPlan(7, cap, H100_STRIDE)
    ora, model = O.TarjanDependencyGraph(), DgModel(cap)
    _dg_round0(plan, _OracleOnly(), ora, model)
    comps, _ = ora.execute_by_component(cap=cap)
    s, d = model.edges()
    committed = model.status == 1
    # ineligible: a dependency outside the graph or absent, and everything that depends on an ineligible vertex
    out = (d < 0) | (d >= cap)
    dd = np.where(out, 0, d)
    inel = np.zeros(cap, bool)
    inel[s[out | (model.status[dd] == 0)]] = True
    live_edge = ~out & (model.status[dd] == 1)
    es, ed = s[live_edge], dd[live_edge]
    while True:
        nxt = inel.copy()
        nxt[es[inel[ed]]] = True
        if (nxt == inel).all():
            break
        inel = nxt
    elig = committed & ~inel
    keep = elig[es] & elig[ed]
    n_lab, lab = connected_components(sp.csr_matrix((np.ones(int(keep.sum())), (es[keep], ed[keep])), shape=(cap, cap)),
                                      directed=True, connection="strong")
    flat = np.asarray([k for c in comps for k in c], np.int64)
    assert np.array_equal(np.sort(flat), np.nonzero(elig)[0])
    cid = np.repeat(np.arange(len(comps)), [len(c) for c in comps])
    pairs = np.unique(np.stack([cid, lab[flat]], 1), axis=0)
    assert len(pairs) == len(comps) == len(np.unique(lab[flat]))
    assert max(len(c) for c in comps) >= 300 and len(comps) > 100_000


class _OracleOnly:
    """Stands in for the GPU graph where only the oracle runs."""

    def update_executed(self, keys):
        pass

    def commit(self, keys, seqs, deps):
        pass


# =========================================================================== conflict index over many tiles
def _ci_ids(g, lead, n_leaders, next_id, batch):
    """Fresh ids per leader, in descending delivery order for every other leader (alternating by batch): a column's
    maximum then sits in an early tile, and only the carry brings it to the later tiles of the segment."""
    ids = np.zeros(len(lead), np.int32)
    for L in range(n_leaders):
        m = lead == L
        c = int(m.sum())
        ids[m] = next_id[L] + (np.arange(c)[::-1] if (L + batch) % 2 == 0 else np.arange(c))
        next_id[L] += c
    back = g.random(len(lead)) < 0.1                      # some ids out of order
    ids[back] = (ids[back] * g.random(int(back.sum()))).astype(np.int32)
    return ids


def _ci_shape(g, shape, n, pool):
    """key lists of n commands over the key pool"""
    if shape == "hot":                                    # one or two keys over ~128 tiles
        return [[int(k)] for k in g.choice(pool[:2], size=n, p=[0.7, 0.3])]
    if shape.startswith("aligned"):
        # every key 1024 * c (+ 1 or + 1023) accesses, one key per command, commands without keys after
        extra = {"aligned": 0, "aligned+1": 1, "aligned-1": 1023}[shape]
        counts, total = [], 0
        while True:
            c = 1024 * int(g.integers(1, 4)) + extra
            if total + c > n:
                break
            counts.append(c); total += c
        keys = np.repeat(g.choice(pool, size=len(counts), replace=False), counts)
        return [[int(k)] for k in g.permutation(keys)] + [[]] * (n - total)
    if shape == "wide":                                   # 9 of 16 keys per command: over 2^20 accesses, 1152 tiles
        return [[int(x) for x in g.choice(pool[:16], size=9, replace=False)] for _ in range(n)]
    assert shape == "nearfull"                            # 4000 keys in 4096 rows: probes wrap past row_mask
    return [[int(x) for x in g.choice(pool, size=int(g.integers(0, 4)))] for _ in range(n)]


@pytest.mark.gpu
@pytest.mark.parametrize("n_leaders", [1, 8])
@pytest.mark.parametrize("shape", ["hot", "aligned", "aligned+1", "aligned-1", "nearfull", "wide"])
def test_conflict_index_many_tiles_matches_the_oracle(shape, n_leaders):
    """2^17 commands per batch: QUERY_THEN_PUT, then PUT, then QUERY, with snapshots in between; every deps row
    equals KvTopOneConflictIndex.top_one_conflicts bit for bit.  "wide" has more than 1024 tiles of accesses, so
    its tile carries cross from one 1024-tile chunk of the carry kernel to the next."""
    from frankenpaxos_b200.epaxos import ConflictIndex
    n = 1 << 17
    g = np.random.Generator(np.random.PCG64(1000 + 10 * n_leaders + len(shape)))
    ci = ConflictIndex(n_leaders, key_capacity=1 << 12, max_commands=n, max_keys=9 * n)
    ora = O.KvTopOneConflictIndex(n_leaders)
    next_id = [0] * n_leaders
    pool = g.choice(np.arange(-2000, 1 << 24), size=4000, replace=False).astype(np.int32)
    for batch, mode in enumerate((ConflictIndex.QUERY_THEN_PUT, ConflictIndex.PUT, ConflictIndex.QUERY)):
        keys = _ci_shape(g, shape, n, pool)
        assert sum(map(len, keys)) >= (1 << 20 if shape == "wide" else 96 * 1024)
        lead = g.integers(0, n_leaders, size=n).astype(np.int32)
        ids = _ci_ids(g, lead, n_leaders, next_id, batch)
        sets = g.random(n) < 0.4
        got = ci.batch(lead, ids, sets, keys, mode=mode)
        exp = np.zeros((n, n_leaders), np.int32)
        for i in range(n):
            if mode != ConflictIndex.PUT:
                exp[i] = ora.top_one_conflicts(bool(sets[i]), keys[i])
            if mode != ConflictIndex.QUERY:
                ora.put((int(lead[i]), int(ids[i])), bool(sets[i]), keys[i])
        if mode != ConflictIndex.PUT:
            bad = np.nonzero((got != exp).any(axis=1))[0]
            assert len(bad) == 0, (mode, len(bad), int(bad[0]), keys[bad[0]], got[bad[0]].tolist(), exp[bad[0]].tolist())
        L, i = int(g.integers(0, n_leaders)), int(g.integers(0, n))
        ci.put_snapshot(L, i); ora.put_snapshot((L, i))
    ci.close()


@pytest.mark.gpu
@pytest.mark.parametrize("n_leaders", [1, 8])
@pytest.mark.parametrize("bad", ["leader", "id", "key"])
def test_conflict_index_invalid_command_past_the_first_tile(bad, n_leaders):
    """A rejected command in a later tile, on a fresh handle: FPX_ERR_INVALID_ARG at its index (the accesses it
    does not claim stay without a row)."""
    from frankenpaxos_b200.epaxos import ConflictIndex
    n, i = 5000, 3333
    g = np.random.Generator(np.random.PCG64(77))
    ci = ConflictIndex(n_leaders, key_capacity=1 << 12, max_commands=n, max_keys=2 * n)
    lead = g.integers(0, n_leaders, size=n).astype(np.int32)
    ids = np.arange(n, dtype=np.int32)
    keys = [[int(k)] for k in g.integers(0, 300, size=n)]
    if bad == "leader":
        lead[i] = n_leaders
    elif bad == "id":
        ids[i] = -1
    else:
        keys[i] = [I32_MIN]
    assert sum(map(len, keys[:i])) >= 1024
    assert _raises(ci.batch, lead, ids, g.random(n) < 0.5, keys) == (-1, i)
    ci.close()


# =========================================================================== EPaxos handlers across tiles
def _ep_rows(kind, n, rep, num, bord, brep, g):
    m = len(rep)
    w = 6 + (2 * n if kind == "preaccept" else n)
    r = np.zeros((m, w), np.int32)
    r[:, 0], r[:, 1], r[:, 2], r[:, 3] = rep, num, bord, brep
    r[:, 4] = g.integers(0, 1000, size=m)
    r[:, 5] = g.integers(-1, 40, size=m)
    r[:, 6:] = g.integers(0, 50, size=(m, w - 6))
    return r


def _same(a, b, what):
    assert a.shape == b.shape, what
    bad = np.nonzero((a != b).any(axis=1))[0]
    assert len(bad) == 0, f"{what}: {len(bad)} rows differ, first {bad[0]}: engine {a[bad[0]].tolist()} " \
                          f"oracle {b[bad[0]].tolist()}"


def _compare_entries(eng, ora, inst):
    for rep, num in inst:
        e1, l1, b1 = eng.entry(rep, num)
        e2, l2, b2 = ora.entry(rep, num)
        assert e1.tolist() == e2.tolist() and l1 == l2 and b1.tolist() == b2.tolist(), (rep, num, e1, e2)


PER_REPLICA = 40_000


@pytest.mark.gpu
@pytest.mark.parametrize("f", [1, 3])
def test_nack_ballots_carried_across_tiles_and_batches(f):
    """Seed ~20k instances, then PreAccept and Accept batches of ~50k unique instances, ~30 % stale (Nacked).  The
    ballots that proceed stay below the seed's largest except at planted positions (1023, 2048, mid-batch, the
    last record), each followed by Nacks in the same and in the next 1024-record tile; a last batch is Nacks only.
    Replies and cmdLog entries bit for bit with the oracle."""
    from frankenpaxos_b200.epaxos import EpaxosReplica
    n = 2 * f + 1
    g = np.random.Generator(np.random.PCG64(300 + f))
    eng, ora = EpaxosReplica(f, 0, PER_REPLICA, max_batch=1 << 17), O.EPaxos(f, 0)
    total = n * PER_REPLICA
    order = g.permutation(total)
    stored = np.full((total, 2), -9, np.int64)           # cmdLog ballot per instance (-9: none)
    used = 0
    touched = []

    def run(kind, m, hi_ord, nack_share):
        nonlocal used
        known = np.nonzero(stored[:, 0] >= 2)[0]
        is_stale = g.random(m) < nack_share
        bord = g.integers(0, 2, size=m)                  # proceeding: below the seed's ballots
        brep = g.integers(0, n, size=m)
        plant = [p for p in (1023, 2048, m // 2, m - 1) if p < m] if hi_ord is not None else []
        is_stale[[q for p in plant for q in (p + 1, p + 2, p + 700, p + 1030) if q < m]] = True
        is_stale[plant] = False                          # Nacks right after each raise, in its tile and the next
        for t, p in enumerate(plant):
            bord[p], brep[p] = hi_ord + t, t % n
        inst = np.zeros(m, np.int64)
        inst[is_stale] = g.choice(known, size=int(is_stale.sum()), replace=False)
        inst[~is_stale] = order[used:used + int((~is_stale).sum())]
        used += int((~is_stale).sum())
        # stale: strictly below the stored ballot
        s_o, s_r = stored[inst[is_stale], 0], stored[inst[is_stale], 1]
        lower = g.integers(0, s_o)
        bord[is_stale] = lower
        brep[is_stale] = g.integers(0, n, size=int(is_stale.sum()))
        rows = _ep_rows(kind, n, inst % n, inst // n, bord, brep, g)
        a, b = getattr(eng, kind)(rows), getattr(ora, kind)(rows)
        _same(a, b, kind)
        nack = a[:, 0] == 2
        assert nack[is_stale].all() and not nack[~is_stale].any()
        key = bord.astype(np.int64) * 64 + brep
        old = stored[inst, 0] * 64 + stored[inst, 1]
        up = ~is_stale & (key >= old)
        stored[inst[up], 0], stored[inst[up], 1] = bord[up], brep[up]
        touched.extend(inst[g.choice(m, size=min(m, 800), replace=False)].tolist() + inst[plant].tolist())
        for t, p in enumerate(plant):                    # a Nack after a raise carries at least that raise
            q = [x for x in (p + 1, p + 1030) if x < m]
            assert all(a[x, 0] == 2 and a[x, 1] >= hi_ord + t for x in q), (kind, p, [a[x].tolist() for x in q])
        return a

    # seed: fresh instances at ballots (2..7, any replica) -- every later proceeding ballot below them
    m = 20_000
    seed = order[:m]; used = m
    bord, brep = g.integers(2, 8, size=m), g.integers(0, n, size=m)
    rows = _ep_rows("preaccept", n, seed % n, seed // n, bord, brep, g)
    _same(eng.preaccept(rows), ora.preaccept(rows), "seed PreAccept")
    stored[seed, 0], stored[seed, 1] = bord, brep
    run("preaccept", 50_000, 100, 0.3)
    run("accept", 50_000, 200, 0.3)
    run("preaccept", 30_001, 300, 0.3)
    a = run("accept", 5_000, None, 1.0)                  # Nacks only: largestBallot from the earlier batches
    assert (a[:, 1] == 303).all()
    _compare_entries(eng, ora, [(int(x) % n, int(x) // n) for x in sorted(set(touched))])
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("f", [1, 3])
def test_batch_contract_violations_across_ctas(f):
    """E1 and E2 duplicates far apart in one batch: FPX_ERR_BATCH_ORDER at the index of the second delivery."""
    from frankenpaxos_b200.epaxos import EpaxosReplica
    n = 2 * f + 1
    g = np.random.Generator(np.random.PCG64(400 + f))
    inst = g.permutation(n * PER_REPLICA)[:70_100]
    zero = np.zeros(len(inst), np.int64)

    def fresh():
        return EpaxosReplica(f, 0, PER_REPLICA, max_batch=1 << 17)

    # a duplicate pair (5, 70 000), PreAccept and Accept
    for kind in ("preaccept", "accept"):
        dup = inst.copy(); dup[70_000] = dup[5]
        rows = _ep_rows(kind, n, dup % n, dup // n, zero, zero, g)
        eng = fresh()
        assert _raises(getattr(eng, kind), rows) == (-12, 70_000)
        eng.close()
    # the same instance three times
    tri = inst.copy(); tri[40_000] = tri[100]; tri[65_000] = tri[100]
    eng = fresh()
    assert _raises(eng.preaccept, _ep_rows("preaccept", n, tri % n, tri // n, zero, zero, g)) == (-12, 40_000)
    eng.close()
    # PreAcceptOk: one (instance, replica) twice, in different tiles
    mine = np.arange(30_000)
    lead = np.zeros((len(mine), 8 + n), np.int32)
    lead[:, 1] = mine
    eng = fresh()
    eng.lead(lead)
    ok = np.zeros((len(mine) * (n - 1), 6 + n), np.int32)
    ok[:, 1] = np.repeat(mine, n - 1)
    ok[:, 4] = np.tile(np.arange(1, n), len(mine))
    ok = ok[g.permutation(len(ok))][:60_000]
    ok[50_000] = ok[300]
    ok[50_000, 6:] = 1                                  # same replica, other content: still two in one batch
    assert _raises(eng.preacceptok, ok) == (-12, 50_000)
    eng.close()


# =========================================================================== cfg4 round at 2^20 instances
@pytest.mark.gpu
def test_cfg4_round_at_2_20_instances_matches_oracle():
    """BASELINE cfg4 (f = 2) at its full size: lead, PreAccept, PreAcceptOk, AcceptOk of the slow path."""
    from frankenpaxos_b200.epaxos import EpaxosReplica
    f, n, N = 2, 5, 1 << 20
    lead, pa, ok = T.epaxos_cfg4(0, f=f, n_instances=N, me=0)
    eng, ora = EpaxosReplica(f, 0, N // n + 2, max_batch=1 << 19), O.EPaxos(f, 0)
    eng.lead(lead)
    assert ora.lead(lead) == (0, -1)
    for chunk in np.array_split(pa, 3):
        _same(eng.preaccept(chunk), ora.preaccept(chunk), "PreAccept replies")
    evs = []
    for chunk in np.array_split(ok, 4):
        a = eng.preacceptok(chunk)
        _same(a, ora.preacceptok(chunk), "PreAcceptOk events")
        evs.append(a)
    evs = np.concatenate(evs)
    assert {1, 2, 3} <= set(evs[:, 0].tolist()) and not ora.saw_sparse
    slow = ok[evs[:, 0] == 2]
    acc = np.zeros((len(slow) * (n - 1), 6), np.int32)
    acc[:, :4] = np.repeat(slow[:, :4], n - 1, axis=0)
    acc[:, 4] = np.tile(np.arange(1, n), len(slow))
    acc = acc[T.rng(0).permutation(len(acc))]
    for chunk in np.array_split(acc, -(-len(acc) // (1 << 18))):
        _same(eng.acceptok(chunk), ora.acceptok(chunk), "AcceptOk events")
    g = T.rng(1)
    sample = np.concatenate([lead[g.choice(len(lead), 1500, replace=False), :2], pa[g.choice(len(pa), 1500, replace=False), :2]])
    _compare_entries(eng, ora, [(int(r), int(m)) for r, m in sample])
    eng.close()
