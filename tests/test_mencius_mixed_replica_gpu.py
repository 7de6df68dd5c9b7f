"""The Compartmentalized Mencius replica's mixed Chosen / ChosenNoopRange call (fpx_mencius_replica_inbound[_dev])
at the edges of what it rests on, against the CPU oracle (wire_mencius_oracle.Replica, bounded by the engine's
live bound base + slot_capacity):

  1. a log ten times slot_capacity through a sliding ring window, with the other writers of the same log
     (replica_chosen, mencius_replica_chosen_range) interleaved;
  2. the renormalisation of the 32-bit log numbers, in the mixed call and in the calls around it;
  3. the split rules at their edges: the range limit of mixed_list_kernel and the tiles of mixed_overlap_kernel;
  4. the device form, which runs every case on a twin engine, and the statuses.

Every split, status, error index, the live log, the watermark and, where a test sets them, the counters equal
the oracle's.  Batches come from mencius_mixed.py; test_mencius_mixed_oracle.py checks that they reach the edges
they claim.  Marked gpu."""
import ctypes as C

import numpy as np
import pytest
import torch

import mencius_mixed as MM
import wire_mencius_oracle as O
from frankenpaxos_b200 import CHOSEN, CHOSEN_RANGE, MENCIUS, MENCIUS_CHOSEN, VALUE_NOOP, Engine
from frankenpaxos_b200 import traces as T

pytestmark = pytest.mark.gpu
SLOT_RANGE, INVALID_ARG = -6, -1
TOP = MM.TOP


def mencius(lg, cap, max_batch=1 << 14, ag=1):
    return Engine(1, ag, 3, num_leaders=2, num_replicas=2, protocol=MENCIUS, num_leader_groups=lg,
                  slot_capacity=cap, max_batch=max_batch, overflow_capacity=1 << 10)


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).copy()).cuda()


def host_call(eng, recs):
    """-> (split, status, err_index) of fpx_mencius_replica_inbound; the split is written with any status but a
    refusal."""
    recs = np.ascontiguousarray(recs, dtype=MENCIUS_CHOSEN)
    split, err = C.c_int32(-7), C.c_int64(-7)
    st = eng._L.fpx_mencius_replica_inbound(eng.h, recs.ctypes.data if len(recs) else None, len(recs),
                                            C.byref(split), C.byref(err))
    return split.value, st, err.value


def dev_call(eng, recs):
    """-> (split, status, err_index) of fpx_mencius_replica_inbound_dev, the status collected by fpx_sync."""
    d_split = torch.full((1,), -7, dtype=torch.int32, device="cuda")
    d_in = dev(recs) if len(recs) else None
    eng.mencius_replica_inbound_dev(d_in.data_ptr() if d_in is not None else None, len(recs), d_split.data_ptr())
    r = eng.sync(check=False)
    return int(d_split.item()), r.status, r.err_index


class Pair:
    """An engine driven through the host form of the mixed call and its twin driven through the device form; every
    other call goes to both."""

    def __init__(self, lg, cap, log_len=None, **kw):
        self.lg, self.cap = lg, cap
        self.a, self.b = mencius(lg, cap, **kw), mencius(lg, cap, **kw)
        self.rep = O.Replica(lg, log_len or cap)
        self.base = 0

    @property
    def lim(self):
        return self.base + self.cap

    def close(self):
        self.a.close(); self.b.close()

    def both(self, name, *args):
        getattr(self.a, name)(*args)
        getattr(self.b, name)(*args)

    def chosen(self, ch):
        self.both("replica_chosen", ch)
        self.rep.apply(MM.records([(int(s), int(s) + 1, int(v)) for s, v in ch]), self.lim)

    def ranges(self, rr):
        self.both("mencius_replica_chosen_range", rr)
        assert self.rep.apply(MM.records([(int(s), int(e), VALUE_NOOP) for s, e in rr]), self.lim) == (0, -1)

    def mixed(self, recs, check_counters=True):
        """Applies the batch from split to split; every call's split, status and error index, the live log and the
        watermark against the oracle.  Returns the splits."""
        splits, start = [], 0
        while True:
            rest = recs[start:]
            want = self.rep.split(rest, self.lim)
            st, err = self.rep.apply(rest[:want], self.lim)
            before = self.a.counters()["rseq_base"]
            got = host_call(self.a, rest)
            assert got == (want, st, err), (start, got, (want, st, err))
            assert dev_call(self.b, rest) == (want, st, err), start
            if check_counters and len(rest):
                n = len(rest)
                after = self.a.counters()["rseq_base"]
                assert after == (1 + n if before > TOP - n - 16 else before + n), (before, after, n)
                assert self.b.counters()["rseq_base"] == after
            splits.append(want)
            start += want
            self.compare()
            if start >= len(recs):
                return splits
            assert want > 0

    def compare(self):
        want = self.rep.log[self.base: self.lim]
        for e in (self.a, self.b):
            assert np.array_equal(e.snapshot_log(self.base, self.cap), want)
            assert e.chosen_watermark() == self.rep.watermark()

    def retire_below(self, slot):
        for e in (self.a, self.b):
            e.chosen_watermark()                         # fpx_retire_below checks the last published watermark
        self.both("retire_below", slot)
        self.rep.retire_below(slot)
        self.base = slot


# --------------------------------------------------------------------------- 1. a sliding ring window
@pytest.mark.parametrize("lg", [1, 3, 5])
def test_mixed_batches_through_a_sliding_window(lg):
    """A log of 40 960 slots through engines of 4096, retired after every window of 2048 slots at points on and
    off the window bounds, so the ring's base index is 2048 or 3584 from the second window on.  Every window
    interleaves replica_chosen and mencius_replica_chosen_range with two mixed batches (mencius_mixed.window_ops):
    ranges across the ring's end, across the retire point, wholly retired and ending at the live bound, Chosens
    at retired slots and at the live bound, Chosens a later range reaches and ones it does not, one record past
    the live bound and one overlapping range.  Every other window the mixed call is the one that closes it."""
    cap, step, total = 4096, 2048, 40960
    g = np.random.default_rng(700 + lg)
    p = Pair(lg, cap, log_len=total + cap)
    n_splits = 0
    for w in range(total // step):
        for kind, recs, _ in MM.window_ops(g, w, lg, p.base, cap, step, total + cap):
            if kind == "chosen":
                p.chosen(recs)
            elif kind == "range":
                p.ranges(recs)
            else:
                n_splits += len(p.mixed(recs)) - 1
            p.compare()
        assert p.rep.watermark() >= (w + 1) * step
        p.retire_below(MM.retire_point(w, step))
    assert n_splits >= total // step
    p.close()


@pytest.mark.parametrize("kind", ["chosens", "ranges"])
def test_watermark_reaches_slots_only_the_mixed_call_put(kind):
    """Past the first lap of the ring (base 6000, ring base index 1904) the mixed call alone fills the live window:
    the watermark scan is bounded by the largest ordinal its kernels report, so a ring index reported in its
    place would stop the watermark short."""
    cap, lg, base = 4096, 3, 6000
    p = Pair(lg, cap, log_len=base + cap)
    fill = np.arange(0, base, dtype=np.int32)
    ch = np.zeros(len(fill), dtype=CHOSEN)
    ch["slot"], ch["value_id"] = fill, fill
    for k in range(0, base, 2000):                      # fill and retire in steps: the bound is base + cap
        p.chosen(ch[k: k + 2000])
        p.retire_below(k + 2000)
    assert p.base == base
    if kind == "chosens":
        recs = MM.records([(s, s + 1, s + 3) for s in range(base, base + cap)])
    else:
        recs = MM.records([(base + r, base + cap, VALUE_NOOP) for r in range(lg)])
    assert p.mixed(recs) == [len(recs)]
    assert p.a.chosen_watermark() == base + cap
    p.close()


# --------------------------------------------------------------------------- 2. the log-number renormalisation
@pytest.mark.parametrize("case", ["below", "at", "above"])
def test_mixed_call_across_the_renormalisation(case):
    """Entries put by replica_chosen just below the top, then a mixed call of n records that starts one below, at
    and one above the bound of renormalize_rlog_if_needed (mencius_mixed.wrap_batch: ranges stopping at the old
    entries and at Chosens of the same call, Chosens losing to old entries and to earlier ranges).  rseq_base is
    old + n afterwards, or 1 + n when the call renormalised.  Then replica_chosen, mencius_replica_chosen_range and
    another mixed call."""
    lg, cap = 3, 1 << 14
    g = np.random.default_rng(31)
    p = Pair(lg, cap)
    recs, _ = MM.wrap_batch(g, lg, cap)
    n = len(recs)
    start = MM.wrap_start(n, case)
    old = MM.old_entries()
    for e in (p.a, p.b):
        e.set_counters(rseq_base=start - len(old))
    p.chosen(old)
    assert p.a.counters()["rseq_base"] == start
    assert p.mixed(recs) == [n]
    assert p.a.counters()["rseq_base"] == (1 + n if case == "above" else start + n)
    late = np.zeros(300, dtype=CHOSEN)
    late["slot"] = g.integers(0, 13000, size=300)
    late["value_id"] = 5
    p.chosen(late)
    p.ranges(np.array([(12000 + r, 16000, ) for r in range(lg)], dtype=CHOSEN_RANGE))
    more = np.zeros(2000, dtype=MENCIUS_CHOSEN)
    more["slot_start"] = g.integers(0, cap - 1, size=2000)
    more["slot_end"] = more["slot_start"] + np.where(g.random(2000) < 0.1, 4 * lg, 1)
    more["value_id"] = np.where(more["slot_end"] - more["slot_start"] > 1, VALUE_NOOP, 9)
    p.mixed(more)
    p.close()


def mencius_votes(g, slots, lg):
    """Arms and f + 1 Phase2as of the slots on an engine of one acceptor group per leader group."""
    arm = T.arms(slots, 0, slots * 4 + 1)
    p2a = T.phase2as(g, slots, 1, lg, 3, False, 0, slots * 4 + 1)
    return arm, p2a


@pytest.mark.parametrize("other", ["fused_step", "range_fill", "dev_queue"])
def test_renormalisation_in_the_call_next_to_the_mixed_call(other):
    """fused_step: step_dev on the Mencius engine (2n log numbers for n votes) renormalises just before a mixed
    call.  range_fill: a mixed call renormalises just before mencius_replica_chosen_range.  dev_queue: the device
    form renormalises while queued behind replica_chosen_dev and another device mixed call on the stream.  The
    next mixed batch's ranges must stop at the entries of the call next to it, and its Chosens lose to them."""
    lg, cap = 2, 1 << 13
    g = np.random.default_rng(41)
    slots = np.arange(0, 3000, 7, dtype=np.int32)
    probe = MM.records([(int(s) - lg * 2, int(s) + lg * 2, VALUE_NOOP) for s in slots[1::3]] +
                       [(int(s), int(s) + 1, 99) for s in slots[2::3]])
    if other == "fused_step":
        p = Pair(lg, cap)
        arm, p2a = mencius_votes(g, slots, lg)
        for e in (p.a, p.b):
            e.proxyleader_arm(arm)
            votes, _ = e.acceptor_phase2a(p2a)
            e.set_counters(rseq_base=TOP - 2 * len(votes) - 15)
            d_v = dev(votes)
            d_c = torch.zeros((len(votes), 2), dtype=torch.int32, device="cuda")
            o_b = torch.zeros((1, 4), dtype=torch.int32, device="cuda")
            o_n = torch.zeros((1, 2), dtype=torch.int32, device="cuda")
            d_wm = torch.zeros(1, dtype=torch.int32, device="cuda")
            e.step_dev(None, 0, None, 0, o_b.data_ptr(), o_n.data_ptr(), d_v.data_ptr(), len(votes), d_c.data_ptr(),
                       d_wm.data_ptr())
            r = e.sync()
            assert e.counters()["rseq_base"] == 1 + 2 * len(votes)
            c = d_c[: r.n_chosen].cpu().numpy().view(CHOSEN).reshape(-1)
            assert sorted(c["slot"].tolist()) == slots.tolist()
        p.rep.apply(MM.records([(int(s), int(s) + 1, int(s) * 4 + 1) for s in c["slot"]]))
        p.compare()
        p.mixed(probe)
    elif other == "range_fill":
        p = Pair(lg, cap)
        first = MM.records([(int(s), int(s) + 1, 3) for s in slots])
        for e in (p.a, p.b):
            e.set_counters(rseq_base=TOP - len(first) - 15)
        p.mixed(first)
        assert p.a.counters()["rseq_base"] == 1 + len(first)
        rr = np.array([(int(s) + 1, int(s) + 1 + 5 * lg) for s in slots[::2]], dtype=CHOSEN_RANGE)
        p.ranges(rr)
        assert p.a.counters()["rseq_base"] == 1 + len(first) + len(rr)
        p.mixed(MM.records([(int(s) - lg, int(s) + 6 * lg, VALUE_NOOP) for s, _ in rr[1::2]] +
                           [(int(s) + lg, int(s) + lg + 1, 98) for s, _ in rr[::2]]))
        p.mixed(probe)
    else:
        e, ref = mencius(lg, cap), mencius(lg, cap)
        rep = O.Replica(lg, cap)
        ch = np.zeros(len(slots), dtype=CHOSEN)
        ch["slot"], ch["value_id"] = slots, slots + 5
        head = MM.records([(int(s) + 1, int(s) + 2, 4) for s in slots])
        n1, n2 = len(head), len(probe)
        start = TOP - len(ch) - n1 - n2 - 15              # the second device mixed call renormalises
        for x in (e, ref):
            x.set_counters(rseq_base=start)
        d_ch, d_head, d_probe = dev(ch), dev(head), dev(probe)
        s1 = torch.full((1,), -1, dtype=torch.int32, device="cuda")
        s2 = torch.full((1,), -1, dtype=torch.int32, device="cuda")
        e.replica_chosen_dev(d_ch.data_ptr(), len(ch))
        e.mencius_replica_inbound_dev(d_head.data_ptr(), n1, s1.data_ptr())
        e.mencius_replica_inbound_dev(d_probe.data_ptr(), n2, s2.data_ptr())
        assert e.counters()["rseq_base"] == 1 + n2
        e.sync()
        ref.replica_chosen(ch)
        rep.apply(MM.records([(int(s), int(s) + 1, int(v)) for s, v in ch]))
        for recs, d in ((head, s1), (probe, s2)):
            want = rep.split(recs)
            assert rep.apply(recs[:want]) == (0, -1)
            assert int(d.item()) == want == ref.mencius_replica_inbound(recs)
        for x in (e, ref):
            assert np.array_equal(x.snapshot_log(0, cap), rep.log)
            assert x.chosen_watermark() == rep.watermark()
        e.close(); ref.close()
        return
    p.close()


# --------------------------------------------------------------------------- 3. the split rules
@pytest.mark.parametrize("k", [MM.MAX_RANGE_BATCH - 1, MM.MAX_RANGE_BATCH, MM.MAX_RANGE_BATCH + 1,
                               MM.MAX_RANGE_BATCH + 2])
def test_range_limit_split(k):
    """k disjoint ranges interleaved with Chosens in one call: up to FPX_MAX_RANGE_BATCH (65 535) ranges the
    whole batch is applied; past it the split is the record index of range number 65 536, and the rest follows."""
    recs, at = MM.spaced_ranges(k, 1)
    p = Pair(1, 1 << 18, max_batch=1 << 18)
    splits = p.mixed(recs)
    assert splits[0] == (len(recs) if k <= MM.MAX_RANGE_BATCH else at[MM.MAX_RANGE_BATCH])
    assert len(splits) == 1 + (k > MM.MAX_RANGE_BATCH)
    p.close()


@pytest.mark.parametrize("where", ["before", "at", "after"])
def test_overlap_and_range_limit_whichever_comes_first(where):
    """An overlapping range (rule a) before, at and after the range-limit cut (rule b): the first one wins."""
    k = MM.MAX_RANGE_BATCH + 40
    recs, at = MM.spaced_ranges(k, 1)
    q = {"before": 1000, "at": MM.MAX_RANGE_BATCH, "after": MM.MAX_RANGE_BATCH + 20}[where]
    MM.overlap_with(recs, at, 1, q, q - 7)
    p = Pair(1, 1 << 18, max_batch=1 << 18)
    splits = p.mixed(recs)
    assert splits[0] == at[min(q, MM.MAX_RANGE_BATCH)]
    p.close()


@pytest.mark.parametrize("lg", [1, 3])
def test_overlap_pairs_at_tile_positions(lg):
    """The later range of an overlapping pair at ranks 255, 256, 257, 511, 512 and 65 534; its earlier partner one
    lane below in the same 256-rank tile, on the last lane of the previous tile, or in tile 0.  The split is
    exactly the later range's index every time."""
    p = Pair(lg, 3 * lg * MM.MAX_RANGE_BATCH + 8 * lg, max_batch=1 << 18)
    cases = 0
    for q in MM.TILE_RANKS:
        for where in MM.PARTNERS:
            pr = MM.partner_rank(q, where)
            if pr is None:
                continue
            recs, at = MM.spaced_ranges(min(MM.MAX_RANGE_BATCH, max(q + 2, 600)), lg)
            i = MM.overlap_with(recs, at, lg, q, pr)
            want = p.rep.split(recs, p.lim)
            assert want == i, (q, where)
            assert host_call(p.a, recs)[0] == dev_call(p.b, recs)[0] == i, (q, where)
            for e in (p.a, p.b):
                e.reset()
            cases += 1
    assert cases == 15
    p.close()


@pytest.mark.parametrize("lg", [3, 5])
def test_near_overlaps_do_not_split(lg):
    """Ranges whose extents intersect but start in different residues, records of one slot whose slot_end >
    slot_start + 1, and zero-slot records, each on top of an earlier range: no split."""
    cap = 1 << 16
    recs, n_ranges = MM.near_overlaps(np.random.default_rng(lg), lg, cap)
    assert n_ranges > 2 * MM.TILE
    p = Pair(lg, cap)
    assert p.mixed(recs) == [len(recs)]
    p.close()


def test_batch_size_limit():
    """n == max_batch is applied; n == max_batch + 1 is refused with FPX_ERR_INVALID_ARG and changes nothing; the
    call after it succeeds."""
    lg, cap, mb = 3, 1 << 14, 3000
    p = Pair(lg, cap, max_batch=mb)
    recs = MM.records([(s, s + 1, s) for s in range(mb + 1)])
    for e, call in ((p.a, host_call), (p.b, dev_call)):
        if call is host_call:
            assert call(e, recs)[1:] == (INVALID_ARG, -1)
        else:
            d = dev(recs)
            s = torch.full((1,), -1, dtype=torch.int32, device="cuda")
            assert e._L.fpx_mencius_replica_inbound_dev(e.h, d.data_ptr(), len(recs), s.data_ptr()) == INVALID_ARG
            e.sync()
        assert (e.snapshot_log(0, cap) == -1).all()
    assert p.mixed(recs[:mb]) == [mb]
    p.close()


# --------------------------------------------------------------------------- 4. statuses
def test_statuses_of_the_device_form():
    """Three records past the live bound in one device call: fpx_sync collects the lowest index, the other records
    are applied.  A bad record at or past the split is not reported by that call; the continuation reports it at
    its own index.  n == 0 writes split 0.  After each of these the next call succeeds."""
    lg, cap = 3, 1 << 12
    p = Pair(lg, cap)
    rows = [(s, s + 1, s) for s in range(0, 600)]
    for i, bad in ((300, (cap, cap + 1, 1)), (120, (cap - 3, cap + 5, VALUE_NOOP)), (450, (-3, 4, VALUE_NOOP))):
        rows[i] = bad
    recs = MM.records(rows)
    assert p.rep.split(recs, p.lim) == len(recs)
    p.mixed(recs)                                         # (split, SLOT_RANGE, 120) from both forms
    rows = [(1000 + 3 * k, 1000 + 3 * k + 2 * lg, VALUE_NOOP) for k in range(0, 40, 2)]
    rows.append((1000 + lg, 1000 + 3 * lg, VALUE_NOOP))   # overlaps the first range: the split
    k = len(rows) - 1
    rows += [(2000 + s, 2001 + s, 1) for s in range(5)] + [(cap, cap + 1, 1)] + [(2100, 2101, 2)]
    recs = MM.records(rows)
    splits = p.mixed(recs)
    assert splits[0] == k
    assert host_call(p.a, recs[:0]) == (0, 0, -1)
    assert dev_call(p.b, recs[:0]) == (0, 0, -1)
    assert p.mixed(MM.records([(3000, 3001, 3)])) == [1]
    p.close()
