"""fpx_epaxos_graph_* on the GPU: bit-exact to the numpy model of tests/epaxos_graph_model.py (rows, component
heads and blockers of every execute), and to scipy's strongly connected components on a 2^20-instance backlog."""
import numpy as np
import pytest
import torch

from epaxos_graph_model import (EgModel, cfg4_like, order_respects_dependencies, random_trace, scc_reference,
                                tie_break_ops)
from frankenpaxos_b200 import FpxError
from frankenpaxos_b200.epaxos import EpaxosGraph, EpaxosReplica

pytestmark = pytest.mark.gpu


def run_both(ops, n, cap, graph=None):
    g = graph or EpaxosGraph(n, cap, max_batch=1 << 14)
    model = EgModel(n, cap)
    executed = 0
    for op in ops:
        if op[0] == "commit":
            g.commit(op[1]); model.commit(op[1])
        elif op[0] == "update_executed":
            g.update_executed(op[1]); model.update_executed(op[1])
        else:
            rows, heads, bl = g.execute_raw()
            mrows, mheads, mbl = model.execute()
            assert rows.tolist() == mrows.tolist()
            assert heads.tolist() == mheads.tolist()
            assert np.array_equal(bl, mbl)
            executed += len(rows)
    g.close()
    return executed


@pytest.mark.parametrize("n,cap,seed", [(3, 300, 0), (3, 200, 1), (5, 120, 2), (5, 150, 3), (7, 60, 4), (7, 80, 5)])
def test_random_traces_match_the_model(n, cap, seed):
    assert run_both(random_trace(seed, n, cap), n, cap) > 0


def test_tie_break_and_self_hole():
    g = EpaxosGraph(3, 4)
    g.commit(tie_break_ops(3)[0][1])
    comps, blockers = g.execute_by_component()
    assert comps == [[(1, 0), (0, 0)], [(2, 0)]] and blockers == []
    g.close()
    g = EpaxosGraph(2, 8)
    g.commit([[0, 0, 0, 5, 3, 0], [0, 1, 0, 1, 0, 0], [0, 2, 0, 2, 0, 0]])
    assert g.execute_by_component() == ([[(0, 1)], [(0, 2)], [(0, 0)]], [])
    g.close()


def test_cfg4_backlog_matches_scipy_components():
    """2^20 instances of 5 columns, 20 % sets, each replica's TopOne view shifted by [-3, 3] (cycles, self holes);
    a few late instances held back: the same components, eligibility and blockers as scipy's SCCs over the
    auxiliary-prefix-node graph, in a dependency-respecting order, and bit-exact to the model."""
    n, per = 5, (1 << 20) // 5
    rows = cfg4_like(7, n, per)
    held = np.zeros(len(rows), bool)
    late = np.nonzero((rows[:, 1] > per - per // 20))[0]
    held[np.random.Generator(np.random.PCG64(3)).choice(late, size=8, replace=False)] = True
    g = EpaxosGraph(n, per, max_batch=1 << 20)
    model = EgModel(n, per)
    g.commit(rows[~held]); model.commit(rows[~held])
    status_before = model.status.copy()
    out, heads, bl = g.execute_raw()
    mout, mheads, mbl = model.execute()
    assert out.tolist() == mout.tolist() and heads.tolist() == mheads.tolist() and np.array_equal(bl, mbl)
    comps, elig, sbl = scc_reference(status_before, model.w)
    got = set()
    start = np.nonzero(heads)[0].tolist() + [len(out)]
    for a, b in zip(start[:-1], start[1:]):
        got.add(frozenset(map(tuple, out[a:b].tolist())))
    assert got == comps
    mine = np.zeros_like(elig)
    mine[out[:, 0], out[:, 1]] = True
    assert np.array_equal(mine, elig) and np.array_equal(bl, sbl)
    assert order_respects_dependencies(out, heads, status_before, model.w)
    assert sum(len(c) > 1 for c in comps) > 0 and len(out) > len(rows) // 2
    # the held instances arrive: everything else executes
    g.commit(rows[held]); model.commit(rows[held])
    out2, heads2, bl2 = g.execute_raw()
    mout2, mheads2, mbl2 = model.execute()
    assert out2.tolist() == mout2.tolist() and heads2.tolist() == mheads2.tolist() and not bl2.any()
    assert len(out) + len(out2) == len(rows)
    g.close()


def test_alternating_chain_needs_many_rounds_and_crosses_the_grid_stride():
    """v_i = (i % 2, i // 2) names v_{i+1} (and everything below it in both columns): X grows by one instance per
    step, so the closure needs about log2(2^19) doubling rounds over 2^19 table entries per table (more than one
    grid stride).  With the last instance absent nothing is eligible; once it arrives all is one component."""
    n, cap = 2, 1 << 18
    L = n * cap
    i = np.arange(L)
    rows = np.zeros((L, 4 + n), np.int64)
    rows[:, 0], rows[:, 1], rows[:, 3] = i % 2, i // 2, (i * 7919) % 1000
    rows[i % 2 == 0, 4 + 1] = np.minimum(i[i % 2 == 0] // 2 + 1, cap)      # column 0 names column 1 up to v_{i+1}
    rows[i % 2 == 0, 4 + 0] = i[i % 2 == 0] // 2
    rows[i % 2 == 1, 4 + 0] = np.minimum(i[i % 2 == 1] // 2 + 2, cap)      # column 1 names column 0 up to v_{i+1}
    rows[i % 2 == 1, 4 + 1] = i[i % 2 == 1] // 2
    g = EpaxosGraph(n, cap, max_batch=L)
    model = EgModel(n, cap)
    g.commit(rows[:-1]); model.commit(rows[:-1])
    out, heads, bl = g.execute_raw()
    mout, _, mbl = model.execute()
    assert len(out) == 0 and len(mout) == 0 and np.array_equal(bl, mbl) and bl[1, cap - 1] == 1
    assert model.rounds >= 18
    g.commit(rows[-1:]); model.commit(rows[-1:])
    out, heads, bl = g.execute_raw()
    mout, mheads, _ = model.execute()
    assert out.tolist() == mout.tolist() and heads.tolist() == mheads.tolist()
    assert len(out) == L and heads.sum() == 1
    g.close()


def test_commits_over_several_calls_and_from_the_replicas_commit_buffer():
    """the device buffer fpx_epaxos_commit_dev consumed feeds fpx_epaxos_graph_commit_dev unchanged; the rest
    arrives in host batches; executes in between"""
    f, n, cap = 1, 3, 256
    ops = random_trace(11, n, cap, batches=6)
    commits = [op[1] for op in ops if op[0] == "commit"]
    rep = EpaxosReplica(f, 0, cap, max_batch=1 << 12)
    g = EpaxosGraph(n, cap, max_batch=1 << 12)
    model = EgModel(n, cap)
    dev = torch.device("cuda", 0)
    for k, rows in enumerate(commits):
        rows = np.ascontiguousarray(rows, dtype=np.int32)
        _, first = np.unique(rows[:, 0] * cap + rows[:, 1], return_index=True)
        rows = np.ascontiguousarray(rows[np.sort(first)])     # the replica takes one Commit per instance per call
        if k % 2 == 0:
            d = torch.from_numpy(rows).to(dev)
            torch.cuda.synchronize()
            rep.commit_dev(d.data_ptr(), len(rows)); rep.sync()
            g.commit_dev(d.data_ptr(), len(rows)); g.sync()
        else:
            half = len(rows) // 2
            g.commit(rows[:half]); g.commit(rows[half:])
        model.commit(rows)
        out, heads, bl = g.execute_raw()
        mout, mheads, mbl = model.execute()
        assert out.tolist() == mout.tolist() and heads.tolist() == mheads.tolist() and np.array_equal(bl, mbl)
    assert g.last_kernel_ms() >= 0
    rep.close(); g.close()


def test_duplicates_and_an_out_of_range_instance():
    n, cap = 3, 16
    g = EpaxosGraph(n, cap)
    rows = [[0, 0, 0, 4, 0, 0, 0], [0, 0, 0, 1, 5, 5, 5], [1, 0, 0, 2, 1, 0, 0], [1, 0, 0, 0, 9, 9, 9]]
    g.commit(rows)
    assert g.execute_by_component() == ([[(0, 0)], [(1, 0)]], [])
    with pytest.raises(FpxError) as ei:
        g.commit([[2, 0, 0, 0, 0, 0, 0], [2, 1, 0, 0, 0, 0, 0], [0, 5, 0, 0, 0, 0, 0], [3, 0, 0, 0, 0, 0, 0]])
    assert ei.value.status == -6 and ei.value.index == 3
    with pytest.raises(FpxError) as ei:
        g.commit([[2, 0, 0, 0, 0, 0, 0], [2, cap, 0, 0, 0, 0, 0]])
    assert ei.value.status == -6 and ei.value.index == 1
    assert g.execute_by_component() == ([], [])      # nothing of either batch was applied
    g.commit([[2, 1, 0, 0, 0, 0, 1]])
    assert g.execute_by_component() == ([], [(2, 0)])
    g.close()
