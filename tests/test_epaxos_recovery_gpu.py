"""EPaxos recovery and the timer-driven transitions on the GPU, bit for bit against the CPU oracle: replies,
events, the cmdLog entry and leader kind of every touched instance, and largestBallot.  Decision table, seeded
mixed traces (small and past one 256-row tile and one 1024-row scan tile), contract violations, the _dev forms,
and a recovery run of n replicas after their command leader falls silent."""
import random

import numpy as np
import pytest

import epaxos_recovery_oracle as R
from epaxos_recovery_traces import CALLS, Trace
from frankenpaxos_b200.engine import FpxError
from frankenpaxos_b200.epaxos import EpaxosReplica
from oracle import fpx_oracle_py as O

pytestmark = pytest.mark.gpu


def L(x):
    return np.asarray(x).tolist()


def entry(b, rep, num):
    row, lk, lb = b.entry(rep, num)
    return L(row), int(lk), L(lb)


def apply(gpu, ora, call, rows):
    """one call on both backends; the outputs must agree exactly"""
    rows = np.asarray(rows, dtype=np.int32)
    a = getattr(ora, call)(rows)
    if call in ("prepare_phase", "prepareok"):
        assert a[0] == 0, (call, a)
        a = a[2]
    elif call == "lead":
        assert a == (0, -1)
    c = getattr(gpu, call)(rows)
    if call not in ("lead", "commit"):
        assert L(c) == L(a), (call, rows.tolist(), L(c), L(a))
    return a


def check_entries(gpu, ora, insts):
    for rep, num in sorted(set(insts)):
        assert entry(gpu, rep, num) == entry(ora, rep, num), (rep, num)


def test_decision_table_every_handler_cmdlog_kind_and_leader_kind():
    for f in (1, 2):
        n, idx = 2 * f + 1, 1
        z = [0] * n
        cmd_setups = ["none", "nocommand", "preaccepted", "accepted", "committed"]
        lead_setups = ["none", "preaccepting", "accepting", "preparing"]
        combos = [(c, l, first) for c in cmd_setups for l in lead_setups for first in ("cmd", "lead")]
        gpu, ora = EpaxosReplica(f, idx, len(combos) * len(CALLS) + 1, 1024), R.EPaxos(f, idx)
        insts = [(2, k) for k in range(len(combos) * len(CALLS))]

        def of(pick):
            return [(2, k * len(CALLS) + h) for k, combo in enumerate(combos) if pick(combo) for h in range(len(CALLS))]

        def setup_cmd(order):
            for kind, call, row in [("nocommand", "prepare", lambda i: [i[0], i[1], 2, 0]),
                                    ("preaccepted", "preaccept", lambda i: [i[0], i[1], 2, 0, 5, 1] + [1] * n + z),
                                    ("accepted", "accept", lambda i: [i[0], i[1], 2, 0, 6, 2] + [2] * n),
                                    ("committed", "commit", lambda i: [i[0], i[1], 7, 3] + [3] * n)]:
                apply(gpu, ora, call, [row(i) for i in of(lambda c: c[0] == kind and c[2] == order)])

        def setup_lead():
            pre = [i for i in of(lambda c: c[1] == "preaccepting") if entry(ora, *i)[0][0] != 4]
            acc = [i for i in of(lambda c: c[1] == "accepting") if entry(ora, *i)[0][0] != 4]
            apply(gpu, ora, "lead", [[i[0], i[1], 3, idx, 9, 0, int(i in acc), 0] + [1] * n for i in pre + acc])
            others = [r for r in range(n) if r != idx][:f]             # own + f = slow quorum: the slow path
            apply(gpu, ora, "preacceptok", [[i[0], i[1], 3, idx, r, 0] + z for i in acc for r in others])
            apply(gpu, ora, "prepare_phase", [[i[0], i[1]] for i in of(lambda c: c[1] == "preparing")])

        setup_cmd("cmd")
        setup_lead()
        setup_cmd("lead")
        check_entries(gpu, ora, insts)
        # one message of each handler per instance
        for h, call in enumerate(CALLS):
            mine = [(2, k * len(CALLS) + h) for k in range(len(combos))]
            if call == "lead":
                rows = [[i[0], i[1], 9, idx, 4, 0, 1, 0] + z for i in mine if entry(ora, *i)[0][0] != 4]
            elif call == "preaccept":
                rows = [[i[0], i[1], 1, 2, 4, 0] + z + z for i in mine]
            elif call == "accept":
                rows = [[i[0], i[1], 4, 2, 4, 0] + z for i in mine]
            elif call == "preacceptok":
                rows = [[i[0], i[1], 3, idx, 0, 1] + [1] * n for i in mine]
            elif call == "acceptok":
                rows = [[i[0], i[1], 3, idx, 0, 0] for i in mine]
            elif call == "commit":
                rows = [[i[0], i[1], 8, 8] + [4] * n for i in mine]
            elif call == "nack":
                rows = [[i[0], i[1], 5, 0] for i in mine]
            elif call == "prepare_phase":
                rows = [[i[0], i[1]] for i in mine]
            elif call == "prepare":
                rows = [[i[0], i[1], 1 + (k % 3) * 2, 0] for k, i in enumerate(mine)]
            elif call == "prepareok":
                rows = [[i[0], i[1], 1, idx, 0, 0, 0, 1, 3] for i in mine]
            else:
                rows = [[i[0], i[1], 3, idx] for i in mine]
            apply(gpu, ora, call, rows)
            check_entries(gpu, ora, mine)
        gpu.close()


def _trace(f, seed, steps, per_replica=4, max_batch=8):
    index = seed % (2 * f + 1)
    gpu, ora = EpaxosReplica(f, index, per_replica, 1 << 16), R.EPaxos(f, index)
    trace = Trace(f, index, per_replica, seed, ora, max_batch=max_batch)
    for _ in range(steps):
        call, rows = trace.step()
        out = apply(gpu, ora, call, rows)
        trace.observe(call, np.asarray(rows), out)
        check_entries(gpu, ora, [(int(r[0]), int(r[1])) for r in rows][:64])
    gpu.close()


@pytest.mark.parametrize("f", [1, 2, 3])
def test_mixed_traces_match_the_oracle(f):
    for seed in range(3):
        _trace(f, 1000 * f + seed, 250)


@pytest.mark.parametrize("f", [1, 2, 3])
def test_mixed_traces_past_one_tile_match_the_oracle(f):
    _trace(f, 7000 + f, 40, per_replica=900, max_batch=1500)


def test_large_batches_running_max_from_earlier_tiles_and_calls():
    f, idx = 2, 4
    n = 2 * f + 1
    z = [0] * n
    P = 3000
    gpu, ora = EpaxosReplica(f, idx, P, 1 << 16), R.EPaxos(f, idx)
    g = random.Random(5)
    # entries at high ballots without raising largestBallot: lead
    apply(gpu, ora, "lead", [[0, k, 50 + k % 7, idx, k, 0, 0, 0] + z for k in range(P)])
    # an earlier call raises largestBallot to (60, 1): the carry into the next call
    apply(gpu, ora, "prepare", [[1, 0, 60, 1]])
    # Prepares: mostly Nacked (ballot below the entry), a rising ballot every 700 rows -> the running max of a Nack
    # comes from an earlier row of its tile, an earlier 256-row tile, an earlier 1024-row scan tile, or the call before
    rows = []
    for k in range(P):
        b = [61 + k // 700, 2] if k % 700 == 0 else [g.randint(0, 45), g.randrange(n)]
        rows.append([0, k, b[0], b[1]])
    out = apply(gpu, ora, "prepare", rows)
    assert (np.asarray(out)[:, 0] == 2).sum() > 2000
    check_entries(gpu, ora, [(0, k) for k in range(0, P, 37)] + [(1, 0)])
    # prepare phase for 2500 instances, then PrepareOk quorums split over three calls, then the restarts' leads
    insts = [(3, k) for k in range(2500)]
    ballots = apply(gpu, ora, "prepare_phase", [[i[0], i[1]] for i in insts])
    for senders in ([0, 1], [2], [3, 4]):
        rows = [[i[0], i[1], int(b[0]), int(b[1]), s, g.choice([-1, 0, 1]), 0, g.randint(0, 2), g.randint(0, 9)]
                for i, b in zip(insts, ballots) for s in senders]
        for r in rows:
            if r[5] == -1:
                r[6], r[7] = -1, 0
        g.shuffle(rows)
        apply(gpu, ora, "prepareok", rows)
    check_entries(gpu, ora, insts[::53])
    apply(gpu, ora, "commit", [[3, k, k, 1] + [1] * n for k in range(0, 2500, 2)])
    apply(gpu, ora, "nack", [[3, k, 70, 0] for k in range(2500)] + [[0, k, 55, 0] for k in range(2000)])
    check_entries(gpu, ora, insts[::53] + [(0, k) for k in range(0, P, 41)])
    gpu.close()


def test_contract_violations_report_the_first_offending_index():
    f, idx = 2, 0
    n = 2 * f + 1
    z = [0] * n

    def fresh():
        return EpaxosReplica(f, idx, 600, 4096)

    def err(fn, rows):
        with pytest.raises(FpxError) as ei:
            fn(np.asarray(rows, dtype=np.int32))
        return ei.value.status, ei.value.index

    for call, mk in [("commit", lambda k: [1, k, 1, 1] + z), ("prepare", lambda k: [1, k, 1, 1]),
                     ("prepare_phase", lambda k: [1, k]), ("slow_path_timer", lambda k: [1, k, 0, 0])]:
        e = fresh()
        rows = [mk(k) for k in range(500)]
        rows[400] = mk(3)                                     # a second message for instance (1, 3)
        rows[450] = mk(7)
        assert err(getattr(e, call), rows) == (-12, 400), call
        e.close()
    e = fresh()
    e.prepare_phase(np.asarray([[0, k] for k in range(300)], dtype=np.int32))
    ok = [[0, k, k + 1, 0, 1, -1, -1, 0, 0] for k in range(300)]
    # two responses of one sender for one instance in one call (E2)
    assert err(e.prepareok, ok[:280] + [[0, 5, 6, 0, 1, -1, -1, 0, 0]] + ok[280:]) == (-12, 280)
    e.close()
    e = fresh()
    e.prepare_phase(np.asarray([[0, k] for k in range(300)], dtype=np.int32))
    # a ballot above the Preparing one fails logger.checkLt (:1792); an older one is ignored
    rows = [[0, k, k + 1, 0, 1, -1, -1, 0, 0] for k in range(300)]
    rows[10][2] = 0
    rows[260][2], rows[290][2] = 900, 901
    assert err(e.prepareok, rows) == (-14, 260)
    e.close()
    e = fresh()
    e.prepare_phase(np.asarray([[0, 0]], dtype=np.int32))
    e.prepareok(np.asarray([[0, 0, 1, 0, 1, 0, 0, 1, 5]], dtype=np.int32))
    # a replacing PrepareOk with new content must be alone for its instance
    assert err(e.prepareok, [[0, 0, 1, 0, 2, -1, -1, 0, 0], [0, 0, 1, 0, 1, 0, 0, 1, 6]]) == (-12, 1)
    e.close()


def test_dev_forms_equal_host_forms():
    torch = pytest.importorskip("torch")
    f, idx = 2, 3
    a, b, ora = EpaxosReplica(f, idx, 6, 4096), EpaxosReplica(f, idx, 6, 4096), R.EPaxos(f, idx)
    trace = Trace(f, idx, 6, 77, ora, max_batch=10)
    widths = {"commit": 0, "nack": 1, "prepare_phase": 2, "prepare": 9 + a.n, "prepareok": 4,
              "slow_path_timer": 2 + a.n}
    for _ in range(300):
        call, rows = trace.step()
        host = apply(a, ora, call, rows)
        rows = np.asarray(rows, dtype=np.int32)
        if call in widths:
            d_in = torch.from_numpy(rows.copy()).cuda()
            w = widths[call]
            d_out = torch.zeros((len(rows), max(w, 1)), dtype=torch.int32, device="cuda")
            torch.cuda.synchronize()
            if w:
                getattr(b, call + "_dev")(d_in.data_ptr(), len(rows), d_out.data_ptr())
            else:
                b.commit_dev(d_in.data_ptr(), len(rows))
            b.sync()
            if w:
                assert L(d_out.cpu()) == L(host), call
        else:
            getattr(b, call)(rows)
        trace.observe(call, rows, host)
        for r in rows:
            assert entry(a, int(r[0]), int(r[1])) == entry(b, int(r[0]), int(r[1]))
    a.close(); b.close()


# ---------------------------------------------------------------------------- a recovery run
def _deps_contain(deps, inst):
    return inst[1] < deps[inst[0]]


@pytest.mark.parametrize("f", [1, 2])
def test_recovery_run_after_the_command_leader_falls_silent(f):
    """Replica 0 leads K instances and its PreAccepts reach random subsets; then it is silent.  Replica 1 recovers
    every instance: prepare phase -> Prepare to the survivors -> PrepareOk -> restart lead (avoid the fast path)
    -> PreAccept -> PreAcceptOk (slow path) -> Accept -> AcceptOk -> Commit to all.  GPU and oracle replicas must
    emit the same messages at every step, every survivor must end with the same Committed triple per instance, and
    two committed commands that conflict must depend on one another (T/epaxos/EPaxos.scala:149-196)."""
    n, K = 2 * f + 1, 40
    g = random.Random(f)
    gpus = [EpaxosReplica(f, r, K, 4096) for r in range(n)]
    oras = [R.EPaxos(f, r) for r in range(n)]
    cis = [O.KvTopOneConflictIndex(n) for _ in range(n)]
    keys = {k: sorted(g.sample(range(8), g.randint(1, 2))) for k in range(K)}
    value_keys = {k: keys[k] for k in range(K)}

    def both(r, call, rows):
        return apply(gpus[r], oras[r], call, rows)

    # replica 0 leads
    lead_rows = []
    for k in range(K):
        deps = cis[0].top_one_conflicts(1, keys[k])
        cis[0].put((0, k), 1, keys[k])
        lead_rows.append([0, k, 0, 0, k, 0, 0, 0] + deps)
    both(0, "lead", lead_rows)
    for r in range(1, n):
        got = [k for k in range(K) if g.random() < 0.5]
        rows = []
        for k in got:
            local = cis[r].top_one_conflicts(1, keys[k])
            cis[r].put((0, k), 1, keys[k])
            rows.append([0, k, 0, 0, k, 0] + local + lead_rows[k][8:])
        if rows:
            both(r, "preaccept", rows)
    # replica 0 is silent from here on; replica 1 recovers everything
    survivors = list(range(1, n))
    rec = 1
    ballots = both(rec, "prepare_phase", [[0, k] for k in range(K)])
    oks = []
    for s in survivors[:f + 1]:
        rep = both(s, "prepare", [[0, k, int(b[0]), int(b[1])] for k, b in zip(range(K), ballots)])
        for k, x in enumerate(rep):
            assert x[0] == 1
            oks.append([0, k, int(x[2]), int(x[3]), s, int(x[4]), int(x[5]), int(x[6]), int(x[7])])
    g.shuffle(oks)
    ev = both(rec, "prepareok", oks)
    restarts = {int(r[1]): (int(e[1]), int(e[2]), int(e[3])) for r, e in zip(oks, ev) if e[0] == 1}
    assert sorted(restarts) == list(range(K))
    # transitionToPreAcceptPhase in the Preparing ballot, avoiding the fast path
    lead = []
    for k, (bo, br, value) in sorted(restarts.items()):
        ks = value_keys.get(value, []) if value != O.NOOP else []
        deps = cis[rec].top_one_conflicts(1, ks)
        cis[rec].put((0, k), 1, ks)
        lead.append([0, k, bo, br, value, 0, 1, 0] + deps)
    both(rec, "lead", lead)
    replies = {}
    for s in survivors:
        if s == rec:
            continue
        rows = []
        for r in lead:
            ks = value_keys.get(r[4], []) if r[4] != O.NOOP else []
            local = cis[s].top_one_conflicts(1, ks)
            cis[s].put((0, r[1]), 1, ks)
            rows.append(r[:6] + local + r[8:])
        replies[s] = both(s, "preaccept", rows)
    acc = None
    for s in survivors:
        if s == rec:
            continue
        rows = [[0, k, int(x[1]), int(x[2]), s, int(x[3])] + L(x[4:]) for k, x in enumerate(replies[s]) if x[0] == 1]
        ev = both(rec, "preacceptok", rows)
        if acc is None and (np.asarray(ev)[:, 0] == 2).any():
            acc = {int(r[1]): e for r, e in zip(rows, ev) if e[0] == 2}
    assert acc is not None and sorted(acc) == list(range(K))
    accepts = [[0, k, lead[k][2], lead[k][3], lead[k][4], int(acc[k][1])] + L(acc[k][2:]) for k in range(K)]
    commits = {}
    for s in survivors:
        if s == rec:
            continue
        rep = both(s, "accept", accepts)
        ev = both(rec, "acceptok", [[0, k, lead[k][2], lead[k][3], s, 0] for k in range(K) if rep[k][0] == 1])
        for e, k in zip(ev, [k for k in range(K) if rep[k][0] == 1]):
            if e[0] == 4:
                commits[k] = [0, k, lead[k][4], int(e[1])] + L(e[2:])
    assert sorted(commits) == list(range(K))
    for s in survivors:
        if s != rec:
            both(s, "commit", [commits[k] for k in range(K)])
    final = {}
    for s in survivors:
        for k in range(K):
            row, lk, lb = entry(gpus[s], 0, k)
            assert (row, lk, lb) == entry(oras[s], 0, k)
            assert row[0] == 4
            final.setdefault(k, row)
            assert row == final[k], (s, k)
    # conflicting committed commands depend on one another
    for a in range(K):
        for b in range(a + 1, K):
            va, vb = final[a][5], final[b][5]
            if va == O.NOOP or vb == O.NOOP or not set(value_keys[va]) & set(value_keys[vb]):
                continue
            assert _deps_contain(final[a][7:], (0, b)) or _deps_contain(final[b][7:], (0, a)), (a, b)
    for x in gpus:
        x.close()
