"""The dense-prefix execution of EPaxos instances (DESIGN §6b, restated in numpy by tests/epaxos_graph_model.py)
against the oracle's TarjanDependencyGraph fed the materialised dependency lists: the same components with the same
member order, in a dependency-respecting order, and a superset of the oracle's blockers."""
import numpy as np
import pytest

from epaxos_graph_model import (EgModel, GraphError, components, oracle_deps, oracle_key, random_trace,
                                respects_dependencies, tie_break_ops)
from oracle import fpx_oracle_py as O


def run_against_oracle(ops, n, cap):
    model = EgModel(n, cap)
    stride = cap + 16
    ora = O.TarjanDependencyGraph()
    executes = 0
    for op in ops:
        if op[0] == "commit":
            model.commit(op[1])
            for r in op[1]:
                ora.commit(oracle_key(int(r[0]), int(r[1]), stride), int(r[3]), oracle_deps(r, n, stride))
        elif op[0] == "update_executed":
            model.update_executed(op[1])
            ora.update_executed([oracle_key(c, j, stride) for c in range(n) for j in range(min(op[1][c], cap))])
        else:
            before = model.status.copy()
            rows, heads, blockers = model.execute()
            comps = components(rows, heads)
            ocomps, oblockers = ora.execute_by_component(cap=n * stride)
            ocomps = [[(k // stride, k % stride) for k in comp] for comp in ocomps]
            assert sorted(map(tuple, comps)) == sorted(map(tuple, ocomps))
            assert respects_dependencies(comps, before, model.w, n)
            got = {(c, j) for c, j in zip(*np.nonzero(blockers))}
            # an instance past cap can never be committed: a watermark naming it gives no blocker bit
            assert {(k // stride, k % stride) for k in oblockers if k % stride < cap} <= got
            executes += len(comps)
    return executes


@pytest.mark.parametrize("n,cap,seed", [(3, 300, 0), (3, 200, 1), (5, 120, 2), (5, 150, 3), (7, 60, 4), (7, 80, 5)])
def test_model_matches_the_oracle_on_random_traces(n, cap, seed):
    ops = random_trace(seed, n, cap)
    assert run_against_oracle(ops, n, cap) > 0


def test_tie_break_puts_the_cycle_before_its_dependent():
    model = EgModel(3, 4)
    ops = tie_break_ops(3)
    model.commit(ops[0][1])
    rows, heads, _ = model.execute()
    assert components(rows, heads) == [[(1, 0), (0, 0)], [(2, 0)]]
    assert run_against_oracle(tie_break_ops(3), 3, 4) == 2


def test_self_hole_alone_is_a_singleton():
    """deps[inst_replica] > inst_number names the later instances of the column, not the instance itself"""
    model = EgModel(2, 8)
    model.commit([[0, 0, 0, 5, 3, 0], [0, 1, 0, 1, 0, 0], [0, 2, 0, 2, 0, 0]])
    rows, heads, blockers = model.execute()
    assert components(rows, heads) == [[(0, 1)], [(0, 2)], [(0, 0)]]
    assert not blockers.any()


def test_out_of_range_watermark_is_never_eligible_and_no_blocker():
    model = EgModel(2, 4)
    model.commit([[0, 0, 0, 0, 0, 9], [1, 0, 0, 0, 0, 0]])
    rows, heads, blockers = model.execute()
    assert rows.tolist() == [[1, 0]] and blockers[1, 1:].all() and not blockers[0].any()


def test_out_of_range_instance_applies_nothing():
    model = EgModel(2, 4)
    with pytest.raises(GraphError) as ei:
        model.commit([[0, 0, 0, 0, 0, 0], [1, 4, 0, 0, 0, 0]])
    assert (ei.value.status, ei.value.index) == (-6, 1)
    assert not model.status.any()
