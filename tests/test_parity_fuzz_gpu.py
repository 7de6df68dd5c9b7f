"""Randomised differential fuzzing of the MultiPaxos entry points on the GPU: small
traces drawn with hypothesis, INCLUDING illegal ones (votes for keys that were never
armed, foreign acceptors, stale and future rounds, duplicated arms with other values,
re-votes).  Every observable -- reply streams with order, status + first offending
index, acceptor state, replica log -- must equal the oracle's.  After a fatal status
the engine is reset (the reference process would be dead)."""
import numpy as np
import pytest
from hypothesis import HealthCheck, given, settings, strategies as st

import harness as H
from frankenpaxos_b200 import P2A, P2B, Engine
from oracle import fpx_oracle_py as O

pytestmark = pytest.mark.gpu

SHAPES = {
    "majority3": dict(f=1, num_acceptor_groups=1, acceptors_per_group=3, flexible=False, num_leaders=2, num_replicas=2),
    "grid2x2": dict(f=1, num_acceptor_groups=2, acceptors_per_group=2, flexible=True, num_leaders=2, num_replicas=2),
    "groups2x3": dict(f=1, num_acceptor_groups=2, acceptors_per_group=3, flexible=False, num_leaders=3, num_replicas=2),
    # 7 voters: a 16-word proxy-leader row
    "maj7": H.WIDE_SHAPES["maj7"],
    # a 5 x 6 grid, 30 voters: a full 32-word row
    "grid5x6": H.WIDE_SHAPES["grid5x6"],
}
N_SLOTS = 24
_engines = {}


def engine(shape, exact):
    if shape not in _engines:
        _engines[shape] = Engine(slot_capacity=N_SLOTS, max_batch=4096, overflow_capacity=256, **SHAPES[shape])
    _engines[shape].reset()
    _engines[shape].set_tally_path(exact)
    return _engines[shape]


slot = st.integers(0, N_SLOTS - 1)
rnd = st.integers(0, 3)
arm_rec = st.tuples(slot, rnd, st.integers(0, 5))
# group and acceptor indices are drawn from 0..31 and reduced per shape, so that every voter of the widest
# shape can be drawn
idx = st.integers(0, 31)
step = st.one_of(
    st.tuples(st.just("arm"), st.lists(arm_rec, min_size=1, max_size=12)),
    st.tuples(st.just("p2a"), st.lists(st.tuples(slot, rnd, st.integers(0, 5), idx, idx), min_size=1, max_size=40)),
    st.tuples(st.just("p2b"), st.lists(st.tuples(idx, idx, slot, rnd), min_size=1, max_size=40)),
)


@pytest.mark.parametrize("exact", [False, True], ids=["auto", "exact"])
@pytest.mark.parametrize("shape", list(SHAPES))
@settings(max_examples=120, deadline=None, suppress_health_check=list(HealthCheck))
@given(script=st.lists(step, min_size=1, max_size=8))
def test_fuzz_against_oracle(shape, exact, script):
    """majority3, grid2x2, groups2x3: 8-word rows; maj7: 16-word rows; grid5x6: 32-word rows."""
    cfg = SHAPES[shape]
    G, A = cfg["num_acceptor_groups"], cfg["acceptors_per_group"]
    eng = engine(shape, exact)
    ora = O.MultiPaxos(cfg["f"], G, A, cfg["flexible"], cfg["num_leaders"], cfg["num_replicas"])
    for kind, recs in script:
        if kind == "arm":
            a = np.array([(s, r, s * 100 + r * 10 + v, -1) for s, r, v in recs], dtype=P2A)
            if H.arm(eng, ora, a) != 0:
                return
        elif kind == "p2a":
            rows = []
            for s, r, v, g, acc in recs:
                g, acc = g % G, acc % A
                if not cfg["flexible"]:
                    g = s % G           # precondition of the engine (DESIGN.md section 2)
                rows.append((s, r, s * 100 + r * 10 + v, (g << 16) | acc))
            ob, on = H.phase2a(eng, ora, np.array(rows, dtype=P2A))
            H.compare_acceptors(eng, ora, cfg, 0, N_SLOTS)
        else:
            rows = []
            for g, acc, s, r in recs:
                if not cfg["flexible"]:
                    g, acc = s % G, acc % A   # in-range ids (precondition); unknown (slot, round) stays possible
                else:
                    g, acc = g % (G + 1), acc % (A + 1)   # one row / column past the grid: a foreign voter
                rows.append((g, acc, s, r))
            stt, c = H.phase2b(eng, ora, np.array(rows, dtype=P2B))
            if stt != 0:
                return                  # fatal in both: same status and index were asserted
            H.replica(eng, ora, c)
    H.compare_log(eng, ora, 0, N_SLOTS)
