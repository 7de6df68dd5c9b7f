"""The read path's CPU oracle (tests/reads_oracle.cc ReadTally / DeferredReads): known answers derived from the
reference's lines, and agreement with the independent transcription (tests/scala_transcription_reads.py) on seeded
traces.  No GPU."""
import numpy as np
import pytest

import reads_traces as RT
import reads_oracle as RO
import scala_transcription_reads as S


def replies(*rows):
    """(key, id, group, acceptor, slot) tuples -> MAX_SLOT_REPLY records in delivery order"""
    r = np.zeros(len(rows), RO.MAX_SLOT_REPLY)
    for i, (k, id_, grp, acc, s) in enumerate(rows):
        r[i] = (k, id_, grp << 16 | acc, s)
    return r


def requests(*rows):
    r = np.zeros(len(rows), RO.READ_REQUEST)
    for i, (s, h) in enumerate(rows):
        r[i] = (s, h)
    return r


def test_overwrite_with_smaller_slot():
    # Client.scala:877-879 replaces acceptor 0's reply (slot 50) by its second one (slot 4) before the count
    # reaches f+1 = 2 at acceptor 1 (slot 7): max(4, 7) + numAcceptorGroups - 1 = 7 (cfg1: one group)
    t = RO.ReadTally(0, 1, 1, 3)
    t.open([3], [9])
    st, err, out = t.max_slot_replies(replies((3, 9, 0, 0, 50), (3, 9, 0, 0, 4), (3, 9, 0, 1, 7)))
    assert st == 0 and out.tolist() == [(3, 9, 7, 0)]


def test_stale_id_reopen_and_reply_after_completion():
    t = RO.ReadTally(0, 1, 2, 3)      # two groups of 3: slot = max + 1
    t.open([1], [5])
    # id 4 is stale (:864-873), ignored; id 5 counts
    st, _, out = t.max_slot_replies(replies((1, 4, 0, 0, 100), (1, 5, 0, 0, 10), (1, 4, 0, 1, 100)))
    assert st == 0 and len(out) == 0
    # re-open with id 6: MaxSlot(6, {}) replaces the read (:652-660); the id 5 reply is forgotten
    t.open([1], [6])
    st, _, out = t.max_slot_replies(replies((1, 5, 0, 1, 100), (1, 6, 1, 2, 20), (1, 6, 1, 0, 30),
                                            (1, 6, 1, 1, 1000)))
    # completes at the second id 6 reply: max(20, 30) + 2 - 1; the third is a reply after completion (:858-863)
    assert st == 0 and out.tolist() == [(1, 6, 31, 0)]
    st, _, out = t.max_slot_replies(replies((1, 6, 0, 0, 5), (2, 0, 0, 0, 5)))   # done / never opened
    assert st == 0 and len(out) == 0


def test_read_batcher_is_group_blind_on_a_flexible_config():
    # ReadBatcher.scala:584 keys by acceptorIndex only: (row 0, col 1) and (row 1, col 1) are one voter, and
    # f+1 = 2 DISTINCT indices complete the read even though no grid row is covered (:585).  slot = max + rows - 1
    t = RO.ReadTally(1, 1, 2, 3, flexible=True)
    t.open([0], [0])
    st, _, out = t.max_slot_replies(replies((0, 0, 0, 1, 8), (0, 0, 1, 1, 3), (0, 0, 1, 2, 5)))
    # acceptor 1's latest reply is 3: max(3, 5) + 2 - 1 = 6
    assert st == 0 and out.tolist() == [(0, 0, 6, 0)]
    # the Client on the same grid needs a whole row (Client.scala:883-887) and reads at max (:892-898)
    c = RO.ReadTally(0, 1, 2, 3, flexible=True)
    c.open([0], [0])
    st, _, out = c.max_slot_replies(replies((0, 0, 0, 1, 8), (0, 0, 1, 1, 3), (0, 0, 1, 2, 5), (0, 0, 1, 0, 1)))
    assert st == 0 and out.tolist() == [(0, 0, 8, 0)]


def test_flexible_non_member_is_the_require():
    # Grid.isReadQuorum's require (S/quorums/Grid.scala:36-39): acceptor 3 is no column of a 2x3 grid
    c = RO.ReadTally(0, 1, 2, 3, flexible=True)
    c.open([0, 1], [0, 0])
    st, err, _ = c.max_slot_replies(replies((1, 7, 0, 3, 0), (0, 0, 0, 0, 1), (0, 0, 0, 3, 2)))
    assert (st, err) == (-5, 2)   # the first one is ignored (stale id): no require runs for it
    t = S.ReadQuorumTally(0, 1, 2, 3, flexible=True)
    t.read(0, 0)
    t.handle_max_slot_reply(0, 0, 0, 0, 1)
    with pytest.raises(S.IllegalArgument):
        t.handle_max_slot_reply(0, 0, 0, 3, 2)


def test_slot_wraps_like_a_jvm_int():
    t = RO.ReadTally(0, 1, 3, 3)    # + 2
    t.open([0], [0])
    _, _, out = t.max_slot_replies(replies((0, 0, 0, 0, 2 ** 31 - 1), (0, 0, 0, 1, 0)))
    assert out.tolist() == [(0, 0, -(2 ** 31) + 1, 0)]


def test_replica_reply_slots_and_order():
    d = RO.DeferredReads(16)
    # W = 0: an eventual read (slot -1) is immediate, ReadReply.slot = W - 1 = -1 (Replica.scala:521-527);
    # slot 0 is not < W, so it waits (:468)
    st, _, now = d.replica(requests((-1, 10), (0, 11), (3, 12), (1, 13), (3, 14), (1, 15)))
    assert st == 0 and now.tolist() == [(10, -1, -1, 0)]
    # executing slots 0..3: reads leave by slot, by arrival within a slot; a read waiting for slot s runs
    # after entry s, before executedWatermark += 1, so ReadReply.slot = s - 1 (:405-413)
    st, out = d.advance(4)
    assert st == 0 and out.tolist() == [(11, -1, 0, 0), (13, 0, 1, 0), (15, 0, 1, 0), (12, 2, 3, 0), (14, 2, 3, 0)]
    st, _, now = d.replica(requests((3, 16), (4, 17)))
    assert now.tolist() == [(16, 3, 3, 0)] and d.pending == 1
    assert d.advance(3)[0] == -1     # the watermark never goes back


def test_replica_overflow_applies_nothing():
    d = RO.DeferredReads(3)
    d.replica(requests((5, 0), (6, 1)))
    # one free entry: slot 7 takes it; slot 0 is not below W = 0 either, so it is the read that does not fit
    st, err, now = d.replica(requests((-1, 2), (7, 3), (0, 4), (8, 5), (9, 6)))
    assert (st, err) == (-8, 2) and len(now) == 0 and d.pending == 2


@pytest.mark.parametrize("shape", ["cfg1", "maj5", "groups2x3", "grid2x3", "grid5x6"])
@pytest.mark.parametrize("kind", [0, 1])
def test_tally_oracle_matches_transcription(shape, kind):
    cfg = RT.SHAPES[shape]
    G, A, f, flex = cfg["num_acceptor_groups"], cfg["acceptors_per_group"], cfg["f"], cfg["flexible"]
    for seed in range(3):
        trace = RT.tally_trace(100 * seed + kind, cfg, kind, 64, 6, 600, hot_keys=4)
        a = RT.run_tally(RO.ReadTally(kind, f, G, A, flex), trace)
        b = RT.run_tally_transcription(S.ReadQuorumTally(kind, f, G, A, flex), trace)
        RT.same_outputs(a, b, f"{shape} kind {kind} seed {seed}")
        assert sum(len(x) for x in a) > 20


def test_replica_oracle_matches_transcription():
    for seed in range(4):
        trace = RT.replica_trace(seed, 20, 300)
        a = RT.run_replica(RO.DeferredReads(1 << 20), trace)
        b = RT.run_replica_transcription(S.ReplicaReads(), trace)
        RT.same_outputs(a, b, f"seed {seed}")
        assert sum(len(x) for x in a) > 1000
