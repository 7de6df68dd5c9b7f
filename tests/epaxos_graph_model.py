"""numpy restatement of the dense-prefix execution of EPaxos instances (fpx_epaxos_graph_*, DESIGN §6b), its
reference checks and the traces the tests feed it.

The model computes steps 1-6 directly on whole columns: the column-wise prefix max, the closure tables by pointer
jumping, X per vertex, eligibility, the component order by sorting and the blockers.  `oracle_deps` materialises the
same dependencies as explicit key lists for the oracle's TarjanDependencyGraph; `scc_reference` restates a large
trace's components, eligibility and blockers with scipy over an auxiliary-prefix-node graph."""
import numpy as np

ABSENT, COMMITTED, EXECUTED = 0, 1, 2


class GraphError(Exception):
    def __init__(self, status, index):
        super().__init__(status, index)
        self.status, self.index = status, index


class EgModel:
    def __init__(self, n, cap):
        self.n, self.cap = n, cap
        self.status = np.zeros((n, cap), np.uint8)
        self.seq = np.zeros((n, cap), np.int64)
        self.w = np.zeros((n, cap, n), np.int64)
        self.rounds = 0

    def commit(self, rows):
        rows = np.asarray(rows, np.int64).reshape(-1, 4 + self.n)
        bad = (rows[:, 0] < 0) | (rows[:, 0] >= self.n) | (rows[:, 1] < 0) | (rows[:, 1] >= self.cap)
        if bad.any():
            raise GraphError(-6, int(np.argmax(bad)))          # FPX_ERR_SLOT_RANGE, nothing applied
        _, first = np.unique(rows[:, 0] * self.cap + rows[:, 1], return_index=True)   # the first record wins
        r = rows[first]
        r = r[self.status[r[:, 0], r[:, 1]] == ABSENT]                               # committed / executed: ignored
        self.status[r[:, 0], r[:, 1]] = COMMITTED
        self.seq[r[:, 0], r[:, 1]] = r[:, 3]
        self.w[r[:, 0], r[:, 1]] = np.clip(r[:, 4:], 0, self.cap + 1)

    def update_executed(self, wm):
        for c in range(self.n):
            self.status[c, :max(0, min(int(wm[c]), self.cap))] = EXECUTED

    def _look(self, T, c, k):
        """T_c[k] for an array of k in [0, cap + 1]: beyond cap nothing is live"""
        z = T[c, np.minimum(k, self.cap)].copy()
        z[..., c] = np.maximum(z[..., c], k)
        return z

    def execute(self):
        """(rows [m, 2] {replica, number}, heads [m], blockers [n, cap]); marks the rows executed"""
        n, cap = self.n, self.cap
        live = self.status == COMMITTED
        a = np.where(live[:, :, None], self.w, 0)
        # 1. P_c[k] = max_{j<k} a(c, j)
        P = np.zeros((n, cap + 1, n), np.int64)
        P[:, 1:] = np.maximum.accumulate(a, axis=1)
        # 2. T0_c[k] = max(k e_c, P_c[k]), then T_c[k] = max_c' T_c'[T_c[k][c']] until nothing changes
        T = P.copy()
        ks = np.arange(cap + 1)
        for c in range(n):
            T[c, :, c] = np.maximum(T[c, :, c], ks)
        bound = int(np.ceil(np.log2(n * (cap + 1)))) + 1
        self.rounds = 0
        while True:
            Tn = T.copy()
            for c2 in range(n):
                Tn = np.maximum(Tn, self._look(T, c2, T[:, :, c2]))
            self.rounds += 1
            if np.array_equal(Tn, T):
                break
            assert self.rounds <= bound, "closure did not settle within the bound"
            T = Tn
        # 3. X(v) = max_c T_c[w_c(v)]
        X = np.zeros((n, cap, n), np.int64)
        for c2 in range(n):
            X = np.maximum(X, self._look(T, c2, self.w[:, :, c2]))
        # 4. eligible iff X_c <= A_c, A_c = first absent instance of column c (cap if none)
        A = np.array([int(np.argmax(self.status[c] == ABSENT)) if (self.status[c] == ABSENT).any() else cap
                      for c in range(n)])
        elig = live & (X <= A[None, None, :]).all(axis=2)
        # 5. order: (sum X, !covered, X lexicographically, seq, replica, number)
        rep, num = np.nonzero(elig)
        Xe = X[rep, num]
        covered = num < Xe[np.arange(len(rep)), rep]
        keys = [num, rep, self.seq[rep, num]] + [Xe[:, q] for q in range(n - 1, -1, -1)] + [~covered, Xe.sum(axis=1)]
        order = np.lexsort(keys)
        rep, num, Xe, covered = rep[order], num[order], Xe[order], covered[order]
        heads = np.ones(len(rep), np.uint8)
        if len(rep) > 1:
            same = covered[1:] & covered[:-1] & (Xe[1:] == Xe[:-1]).all(axis=1)
            heads[1:] = ~same
        # 6. blockers: absent (c, j) with j < max over live v of w_c(v), j < cap
        M = np.where(live[:, :, None], self.w, 0).max(axis=(0, 1)) if live.any() else np.zeros(n, np.int64)
        blockers = np.zeros((n, cap), np.uint8)
        for c in range(n):
            m = min(int(M[c]), cap)
            blockers[c, :m] = self.status[c, :m] == ABSENT
        self.status[rep, num] = EXECUTED
        return np.stack([rep, num], axis=1).astype(np.int32), heads, blockers


def components(rows, heads):
    comps = []
    for (c, j), h in zip(rows.tolist(), heads.tolist()):
        if h:
            comps.append([])
        comps[-1].append((c, j))
    return comps


# ---------------------------------------------------------------------------------------------- oracle feed
def oracle_key(c, j, stride):
    return c * stride + j


def oracle_deps(row, n, stride):
    """[0, w_c) of every column, except the instance itself (subtractOne, Replica.scala:582)"""
    c0, j0 = int(row[0]), int(row[1])
    return [oracle_key(c, j, stride) for c in range(n) for j in range(int(max(row[4 + c], 0))) if (c, j) != (c0, j0)]


def respects_dependencies(comps, model_before_status, w, n):
    """every live dependency of a member is executed before, in an earlier component or in the same one"""
    done = model_before_status == EXECUTED
    for comp in comps:
        members = set(comp)
        for c, j in comp:
            for c2 in range(n):
                for j2 in range(min(int(w[c, j, c2]), done.shape[1])):
                    if (c2, j2) != (c, j) and not done[c2, j2] and (c2, j2) not in members:
                        return False
        for c, j in comp:
            done[c, j] = True
    return True


# ---------------------------------------------------------------------------------------------- traces
def random_trace(seed, n, cap, batches=8, lag=6):
    """ops: ('commit', rows) / ('update_executed', wm) / ('execute',).  Instances arrive in a global order that
    interleaves the columns; instance k's watermark of column c is the number of column-c instances before it in
    that order plus a delta in [-lag, lag] (forward references, so cycles; in every other epoch only), its own column's often past itself (the
    self hole), near the end now and then past cap; about 5 % stay absent until a later batch, which commits half of
    those still held."""
    g = np.random.Generator(np.random.PCG64(seed))
    order = []
    nxt = [0] * n
    while min(nxt) < cap:
        c = int(g.integers(0, n))
        if nxt[c] < cap:
            order.append((c, nxt[c]))
            nxt[c] += 1
    before = np.zeros(n, np.int64)
    rows = []
    for k, (c, j) in enumerate(order):
        # forward references only in every other epoch of 40 instances: reach does not percolate to the end
        fwd = (k // 40) % 2 == 0
        w = np.clip(before + g.integers(-lag, (lag if fwd else 0) + 1, size=n), 0, cap)
        if g.random() < 0.3:
            w[c] = min(j + (int(g.integers(1, 4)) if fwd else 1), cap)   # self hole (a recovered instance)
        if k > 0.95 * len(order) and g.random() < 0.05:  # late, so that it does not block everything
            w[int(g.integers(0, n))] = cap + int(g.integers(1, 4))
        rows.append([c, j, 0, int(g.integers(-3, 20))] + w.tolist())
        before[c] += 1
    rows = np.array(rows, np.int64)
    cut = np.sort(g.choice(np.arange(1, len(rows)), size=batches - 1, replace=False))
    ops = []
    held = []
    for b, part in enumerate(np.split(np.arange(len(rows)), cut)):
        keep = part[g.random(len(part)) >= 0.05]          # about 5 % stay absent for now
        held += [int(i) for i in part if i not in set(keep.tolist())]
        batch = rows[keep]
        if b % 3 == 1 and len(batch) > 4:                 # repeated commits in the batch and across batches
            batch = np.concatenate([batch, batch[:3], rows[part[:2]]])
        if len(held):                                      # commit half of what is still held
            g.shuffle(held)
            half, held = held[:len(held) // 2], held[len(held) // 2:]
            batch = np.concatenate([batch, rows[half]]) if len(half) else batch
        ops.append(("commit", batch[g.permutation(len(batch))]))
        if b == batches // 2:
            ops.append(("update_executed", [int(x) for x in g.integers(0, 4, size=n)]))
        ops.append(("execute",))
    if held:
        ops.append(("commit", rows[held]))
        ops.append(("execute",))
    return ops


def tie_break_ops(n=3):
    """a cycle {(0,0), (1,0)} with X = (1, 1, 0...) and an uncovered (2,0) with the same X that only depends on it"""
    def row(c, j, seq, w):
        return [c, j, 0, seq] + w + [0] * (n - len(w))
    rows = [row(2, 0, -5, [1, 1]), row(0, 0, 3, [0, 1]), row(1, 0, 1, [1, 0])]
    return [("commit", np.array(rows)), ("execute",)]


def cfg4_like(seed, n, per_col, p_set=0.2, lag=3):
    """a backlog like BASELINE cfg4's: instances of the n columns interleaved; each instance of a set command sees
    the set instances of every column before it in the global order shifted by a delta in [-lag, lag] (the TopOne
    watermark as that replica saw it); a get depends on the sets only.  Returns commit rows."""
    g = np.random.Generator(np.random.PCG64(seed))
    total = n * per_col
    col = np.repeat(np.arange(n), per_col)
    g.shuffle(col)
    num = np.zeros(total, np.int64)
    cnt = np.zeros(n, np.int64)
    for i, c in enumerate(col):
        num[i] = cnt[c]
        cnt[c] += 1
    is_set = g.random(total) < p_set
    # last set instance (+1) of column c among the first k entries of the global order
    last_set = np.zeros((total + 1, n), np.int64)
    for c in range(n):
        m = (col == c) & is_set
        v = np.where(m, num + 1, 0)
        last_set[1:, c] = np.maximum.accumulate(v)
    k = np.arange(total) + g.integers(-lag, lag + 1, size=total)
    k = np.clip(k, 0, total)
    w = last_set[k]
    rows = np.zeros((total, 4 + n), np.int64)
    rows[:, 0], rows[:, 1], rows[:, 3] = col, num, g.integers(0, 1 << 20, size=total)
    rows[:, 4:] = w
    return rows.astype(np.int32)


# ---------------------------------------------------------------------------------------------- scipy reference
def scc_reference(status, w):
    """components (as a set of frozensets of (replica, number)), eligibility [n, cap] and blockers [n, cap] of the
    live vertices, from scipy's strongly connected components over an auxiliary-prefix-node graph: v -> Pre(c, w_c),
    Pre(c, k) -> (c, k - 1), Pre(c, k - 1); executed and absent vertices have no out-edges; a watermark past cap
    points at one extra node that stands for the instances that can never be committed."""
    from scipy.sparse import csr_matrix
    from scipy.sparse.csgraph import breadth_first_order, connected_components
    n, cap = status.shape
    nv = n * cap
    pre = lambda c, k: nv + c * (cap + 1) + k          # noqa: E731
    never = nv + n * (cap + 1)
    total = never + 1
    live = (status == COMMITTED).reshape(-1)
    src, dst = [], []
    vid = np.arange(nv)
    for c in range(n):
        wc = w[:, :, c].reshape(-1)
        inside = wc <= cap
        src.append(vid[live & inside]); dst.append(pre(c, wc[live & inside]))
        src.append(vid[live & ~inside]); dst.append(np.full(int((live & ~inside).sum()), never))
        k = np.arange(1, cap + 1)
        src.append(pre(c, k)); dst.append(c * cap + k - 1)
        src.append(pre(c, k)); dst.append(pre(c, k - 1))
    src, dst = np.concatenate(src), np.concatenate(dst)
    G = csr_matrix((np.ones(len(src), np.int8), (src, dst)), shape=(total, total))
    _, label = connected_components(G, directed=True, connection="strong")
    # ineligible: reaches an absent instance or `never` (BFS from them over the reversed edges)
    bad = np.concatenate([np.nonzero((status == ABSENT).reshape(-1))[0], [never]])
    R = csr_matrix((np.ones(len(src) + len(bad), np.int8),
                    (np.concatenate([dst, np.full(len(bad), total)]), np.concatenate([src, bad]))),
                   shape=(total + 1, total + 1))
    reach = breadth_first_order(R, total, directed=True, return_predecessors=False)
    inel = np.zeros(total + 1, bool)
    inel[reach] = True
    elig = live & ~inel[:nv]
    comps = {}
    for v in np.nonzero(elig)[0]:
        comps.setdefault(label[v], []).append((int(v // cap), int(v % cap)))
    M = np.where(live.reshape(n, cap)[:, :, None], w, 0).max(axis=(0, 1)) if live.any() else np.zeros(n, np.int64)
    blockers = np.zeros((n, cap), np.uint8)
    for c in range(n):
        m = min(int(M[c]), cap)
        blockers[c, :m] = status[c, :m] == ABSENT
    return {frozenset(x) for x in comps.values()}, elig.reshape(n, cap), blockers


def order_respects_dependencies(rows, heads, status_before, w):
    """every live dependency of an executed vertex is executed before it or in its component, checked with a
    column-wise prefix max of the component positions (no edge is materialised)"""
    n, cap = status_before.shape
    comp_of = np.cumsum(heads.astype(np.int64)) - 1
    pos = np.full((n, cap), -1, np.int64)
    pos[status_before == COMMITTED] = np.iinfo(np.int64).max    # live but not executed now: nothing may wait for it
    pos[rows[:, 0], rows[:, 1]] = comp_of
    pmax = np.full((n, cap + 1), -1, np.int64)
    pmax[:, 1:] = np.maximum.accumulate(pos, axis=1)
    for c in range(n):
        need = pmax[c, np.minimum(w[rows[:, 0], rows[:, 1], c], cap)]
        if (need > comp_of).any():
            return False
    return True
