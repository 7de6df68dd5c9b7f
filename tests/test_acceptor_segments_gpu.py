"""The acceptor kernel cut into pipelined segments (a batch too large for L2 is processed a segment at a
time; each segment's carry-in is the acceptors' rounds at batch start maxed with everything delivered in
earlier segments).  Batches whose decisions depend on records of an earlier segment, compared bit for bit
with the CPU oracle: Phase2b and Nack streams, round, maxVotedSlot and every vote cell."""
import numpy as np
import pytest

import harness as H
from frankenpaxos_b200 import traces as T

pytestmark = pytest.mark.gpu

CFG = dict(f=1, num_acceptor_groups=1, acceptors_per_group=3, flexible=False, num_leaders=2, num_replicas=2)
M = 4096            # slots per quarter of the batch; 3 * M records = 12288, a multiple of 32
L = 3 * M           # records per quarter: with 4 segments, quarter q is segment q


def quarter(g, cfg, slots, rounds, value_base):
    """Every acceptor's copy of each slot (round per slot), shuffled inside the quarter."""
    q = T.phase2as(g, slots, cfg["f"], cfg["num_acceptor_groups"], cfg["acceptors_per_group"], cfg["flexible"],
                   round_=rounds, values=slots + value_base, thrifty=False)
    return q[g.permutation(len(q))]


def batch(case, seed=11, cfg=CFG):
    """Four quarters of M slots each, every slot sent to all acceptors of its group (cfg's acceptors_per_group
    copies per slot)."""
    g = T.rng(seed)
    s0, s1, s2 = (np.arange(k * M, (k + 1) * M, dtype=np.int32) for k in range(3))
    if case == "nacks":
        # q0 round 5; q1 round 5 on new slots; q2 revisits q0's slots in rounds 3 (stale: Nack, after the
        # round-5 records of the same acceptors two segments earlier) and 6; q3 round 4 (stale behind q2's
        # round 6) and 7
        q = [quarter(g, cfg, s0, 5, 0), quarter(g, cfg, s1, 5, 0),
             quarter(g, cfg, s0, np.where(g.random(M) < 0.5, 3, 6), 50000),
             quarter(g, cfg, s2, np.where(g.random(M) < 0.7, 4, 7), 90000)]
    else:
        # rounds rise from segment to segment: no Nack, dense reply positions
        q = [quarter(g, cfg, s0, 1, 0), quarter(g, cfg, s1, 2, 0), quarter(g, cfg, s0, 2, 50000),
             quarter(g, cfg, s2, 3, 90000)]
    # same round, different value, across the q0 / q1 boundary: q1 opens with a second vote of q0's last
    # (acceptor, slot, round) -- the later delivery must own the vote cell
    last = q[0][-1].copy()
    last["value_id"] += 777
    q[1][0] = last
    out = np.concatenate(q)
    assert len(out) == 4 * M * cfg["acceptors_per_group"]
    return out


@pytest.mark.parametrize("segments", [1, 3, 4, 8])
@pytest.mark.parametrize("case", ["nacks", "dense"])
def test_segmented_acceptor_matches_oracle(case, segments):
    eng, ora = H.make_pair(CFG, 4 * M, max_batch=1 << 16)
    eng.set_acceptor_segments(segments)
    recs = batch(case)
    ob, on = H.phase2a(eng, ora, recs)
    assert (len(on) > 0) == (case == "nacks")
    H.compare_acceptors(eng, ora, CFG, 0, 3 * M)
    # a second batch starts from the rounds the first one left behind
    ob2, on2 = H.phase2a(eng, ora, batch(case, seed=12))
    assert len(on2) > 0
    H.compare_acceptors(eng, ora, CFG, 0, 3 * M)
    eng.close()


# groups2x15: two groups of 15, 30 acceptors, 32-word proxy-leader rows
WIDE = H.WIDE_SHAPES["groups2x15"]


@pytest.mark.parametrize("segments", [1, 3, 8])
@pytest.mark.parametrize("case", ["nacks", "dense"])
def test_segmented_acceptor_with_30_acceptors_matches_oracle(case, segments):
    """groups2x15 (30 acceptors, 15 per slot, 32-word rows): the same batches with every slot sent to the 15
    acceptors of group slot % 2, so all 30 acceptors carry their rounds across the segment boundaries --
    keys 0 to 29 in the acceptor kernel's lane-per-key scan and carry-in."""
    n_slots = 3 * M
    eng, ora = H.make_pair(WIDE, n_slots, max_batch=4 * M * WIDE["acceptors_per_group"])
    eng.set_acceptor_segments(segments)
    ob, on = H.phase2a(eng, ora, batch(case, cfg=WIDE))
    assert (len(on) > 0) == (case == "nacks")
    assert len(np.unique(ob["group"] * 15 + ob["acceptor"])) == 30       # every acceptor voted
    H.compare_acceptors(eng, ora, WIDE, 0, n_slots)
    ob2, on2 = H.phase2a(eng, ora, batch(case, seed=12, cfg=WIDE))
    assert len(on2) > 0
    H.compare_acceptors(eng, ora, WIDE, 0, n_slots)
    eng.close()
