"""Cross-check of the C++ oracle against an independent line-by-line Python transcription
of the Scala handlers (tests/scala_transcription.py) on random traces, legal and illegal.
The reference cannot be run here; two independent restatements agreeing is the strongest
pin available for the HANDLERS (the helpers are pinned by the reference's own vectors)."""
import numpy as np
from hypothesis import given, settings, strategies as st

import scala_transcription as S
from frankenpaxos_b200.engine import P2A, P2B
from oracle import fpx_oracle_py as O

SHAPES = {
    "majority3": (1, 1, 3, False, 2),
    "majority5": (2, 1, 5, False, 3),
    "grid2x3": (1, 2, 3, True, 2),
    "groups2x3": (1, 2, 3, False, 2),
    # the engine's wider proxy-leader rows: 7 voters (16 words), 15 voters (32 words), a 5 x 6 grid (30 voters)
    "maj7": (3, 1, 7, False, 4),
    "maj15": (7, 1, 15, False, 8),
    "grid5x6": (1, 5, 6, True, 2),
}
slot = st.integers(0, 15)
rnd = st.integers(0, 3)
idx = st.integers(0, 31)     # group / acceptor index, reduced per shape in the test
step = st.one_of(
    st.tuples(st.just("arm"), st.lists(st.tuples(slot, rnd, st.integers(0, 9)), min_size=1, max_size=10)),
    st.tuples(st.just("p2a"), st.lists(st.tuples(slot, rnd, st.integers(0, 9), idx, idx), min_size=1, max_size=30)),
    st.tuples(st.just("p2b"), st.lists(st.tuples(idx, idx, slot, rnd), min_size=1, max_size=30)),
    # one (slot, round) armed, then votes for it only: enough distinct voters to complete a quorum of 8 of 15
    st.tuples(st.just("quorum"), st.tuples(slot, rnd, st.integers(0, 9), st.lists(st.tuples(idx, idx), min_size=1,
                                                                                   max_size=30))),
)


@settings(max_examples=700, deadline=None)
@given(shape=st.sampled_from(sorted(SHAPES)), script=st.lists(step, min_size=1, max_size=8))
def test_cpp_oracle_agrees_with_python_transcription(shape, script):
    """majority3, majority5, grid2x3, groups2x3: up to 6 voters (the engine's 8-word rows); maj7: 7 voters
    (16-word rows); maj15 and grid5x6: 15 and 30 voters (32-word rows)."""
    f, G, A, flexible, L = SHAPES[shape]
    ora = O.MultiPaxos(f, G, A, flexible, L, f + 1)
    ref = S.System(f, G, A, flexible, L)
    for kind, recs in script:
        if kind == "quorum":
            s_, r_, v_, voters = recs
            a = np.array([(s_, r_, v_, -1)], dtype=P2A)
            assert ora.arm(a) == (0, -1)
            ref.arm_batch(a.tolist())
            kind, recs = "p2b", [(g % G, acc % A, s_, r_) for g, acc in voters]     # members only
        if kind == "arm":
            a = np.array([(s, r, v, -1) for s, r, v in recs], dtype=P2A)
            assert ora.arm(a) == (0, -1)
            ref.arm_batch(a.tolist())
        elif kind == "p2a":
            a = np.array([(s, r, v, ((g % G) << 16) | (acc % A)) for s, r, v, g, acc in recs], dtype=P2A)
            st_, _, ob, on = ora.acceptor_phase2a(a)
            rb, rn = ref.acceptor_batch(a.tolist())
            assert st_ == 0 and ob.tolist() == rb and on.tolist() == rn
        else:
            # every member can vote, and so can a group / acceptor id past the last one: non-flexible counts
            # it as a map key (ProxyLeader.scala:237), flexible `require`s (Grid.scala:44-47)
            b = np.array([(g % (G + 1), a % (A + 1 if flexible else A + 3), s, r) for g, a, s, r in recs], dtype=P2B)
            st_, idx, oc = ora.proxyleader_phase2b(b)
            rst, ridx, rc = ref.vote_batch(b.tolist())
            assert (st_, idx) == (rst, ridx) and oc.tolist() == rc
            if st_ != 0:
                return
            ora.replica_chosen(oc)
    assert ora.executed_watermark() == ref.replica.executed_watermark
    for g in range(G):
        for a_ in range(A):
            r, m, vr, vv = ora.snapshot_acceptor(g, a_, 0, 16)
            acc = ref.acceptors[g][a_]
            assert (r, m) == (acc.round, acc.max_voted_slot)
            for s in range(16):
                exp = acc.states.get(s, (-1, -1))
                assert (vr[s], vv[s]) == exp
