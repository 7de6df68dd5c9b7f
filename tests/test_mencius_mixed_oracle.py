"""CPU companion of test_mencius_mixed_replica_gpu.py.  Pins the limit-aware per-message replica of the mixed Chosen /
ChosenNoopRange call (wire_mencius_oracle.Replica) with a second restatement -- every builder batch applied one
message at a time through the MultiPaxos oracle in Mencius mode (replica_chosen for a record of one slot,
replica_chosen_range for the others) -- and checks that every builder of mencius_mixed.py puts its edges where it
claims: ring positions, retire and live bounds, range stops, counter values, ranks and tiles."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import mencius_mixed as MM  # noqa: E402
import wire_mencius_oracle as O  # noqa: E402
from oracle import fpx_oracle_py as F  # noqa: E402

SLOT_RANGE = -6


def mp(lg):
    return F.MultiPaxos(1, 1, 3, False, 2, 2, mencius_leader_groups=lg)


def stops(log, retired, recs, lg, limit):
    """Replica.handleChosen / handleChosenNoopRange over a copy of the log, one record at a time; for each record the
    slot where it stopped (the first of its slots already in the log), or None."""
    log = log.copy()
    out = []
    for r in recs:
        s, e, v = int(r["slot_start"]), int(r["slot_end"]), int(r["value_id"])
        hit = None
        if 0 <= s <= e <= limit:
            for x in range(s, e, lg):
                if x < retired or log[x] != -1:
                    hit = x
                    break
                log[x] = v
        out.append(hit)
    return out, log


def test_limit_bounds_the_oracle_like_the_live_bound():
    """A record past `limit` is FPX_ERR_SLOT_RANGE and is not a range of the split rule, although the oracle's log
    is longer; the other records are applied."""
    rep = O.Replica(3, 1000)
    recs = MM.records([(10, 40, O.VALUE_NOOP), (490, 510, O.VALUE_NOOP), (13, 60, O.VALUE_NOOP), (499, 500, 4),
                       (500, 501, 5)])
    assert rep.split(recs) == 2 and rep.split(recs, 500) == 2
    recs[2] = (600, 700, O.VALUE_NOOP, 0)
    assert rep.split(recs) == 5 and rep.split(recs, 500) == 5
    assert rep.apply(recs, 500) == (SLOT_RANGE, 1)
    assert rep.log[499] == 4 and rep.log[500] == -1 and rep.log[600] == -1 and rep.log[13] == O.VALUE_NOOP
    with pytest.raises(AssertionError):
        rep.split(recs, 1001)


def apply_both(rep, ora, recs, lg, limit):
    """Applies the batch from split to split to the oracle and, one message at a time, to the restatement; the
    statuses agree call by call.  Returns the splits."""
    splits, start = [], 0
    while start < len(recs) or not splits:
        rest = recs[start:]
        want = rep.split(rest, limit)
        assert rep.apply(rest[:want], limit) == MM.per_message(ora, rest[:want], lg, limit)
        splits.append(want)
        start += want
        if want == 0:
            break
    return splits


@pytest.mark.parametrize("lg", [1, 3, 5])
def test_window_batches(lg):
    """Every window of the sliding-window GPU test: the oracle equals the restatement after every call, and the
    batches reach the edges they claim."""
    cap, step, total = 4096, 2048, 40960
    g = np.random.default_rng(700 + lg)
    rep, ora = O.Replica(lg, total + cap), mp(lg)
    base = 0
    ring_crossings = 0
    for w in range(total // step):
        lim = base + cap
        other_slots = set()
        stopped_at_other = reached = not_reached = overwritten = split_calls = 0
        for kind, recs, claims in MM.window_ops(g, w, lg, base, cap, step, total + cap):
            if kind == "chosen":
                rows = MM.records([(int(s), int(s) + 1, int(v)) for s, v in recs])
                assert rep.apply(rows, lim) == MM.per_message(ora, rows, lg, lim) == (0, -1)
                other_slots |= set(recs["slot"].tolist())
            elif kind == "range":
                rows = MM.records([(int(s), int(e), O.VALUE_NOOP) for s, e in recs])
                before = rep.log.copy()
                assert rep.apply(rows, lim) == MM.per_message(ora, rows, lg, lim) == (0, -1)
                other_slots |= set(np.nonzero(before != rep.log)[0].tolist())
            else:
                hit, _ = stops(rep.log, rep.retired, recs, lg, lim)
                s, e = recs["slot_start"].astype(np.int64), recs["slot_end"].astype(np.int64)
                bad = np.nonzero((s < 0) | (e < s) | (e > lim))[0]
                assert bad.tolist() == claims["past_bound"]
                for i in claims.get("ring_end", []):
                    sl = np.arange(s[i], e[i], lg)
                    assert base <= sl[0] and sl[-1] < lim and (np.diff(sl % cap) < 0).any()
                    ring_crossings += 1
                assert ("ring_end" in claims) == (base % cap != 0)
                if base:
                    i, = claims["straddle"]
                    assert s[i] < base < e[i] and hit[i] == s[i]
                    assert claims["retired_range"] and all(e[i] <= base for i in claims["retired_range"])
                    assert all(s[i] < base for i in claims["retired_chosen"])
                assert all(e[i] == lim and MM.covers(s[i], e[i], lg, lim) >= 2 for i in claims.get("range_at_bound", []))
                i, = claims["chosen_at_bound"]
                assert (s[i], e[i]) == (lim - 1, lim)
                for i, j in zip(claims.get("chosen_then_range", []), claims.get("range_after_chosen", [])):
                    assert i < j and s[j] < s[i] < e[j] and (s[i] - s[j]) % lg == 0
                    reached += hit[j] == s[i]
                for i, j in zip(claims.get("chosen_not_reached", []), claims.get("range_stops_at_other", [])):
                    assert i < j and hit[j] is not None and hit[j] < s[i] < e[j]
                    not_reached += 1
                stopped_at_other += sum(h in other_slots for i, h in enumerate(hit) if MM.covers(s[i], e[i], lg, lim) >= 2)
                for j, i in zip(claims.get("range_then_chosen", []), claims.get("chosen_after_range", [])):
                    assert j < i and s[j] < s[i] < e[j]
                    overwritten += hit[j] is None or hit[j] > s[i]      # the range reached the Chosen's slot first
                if "closing" in claims:
                    assert [s[i] for i in claims["closing"]] == list(range(w * step, (w + 1) * step))
                splits = apply_both(rep, ora, recs, lg, lim)
                split_calls += len(splits) - 1
            assert np.array_equal(ora.snapshot_log(0, total + cap), rep.log)
            assert ora.first_hole() == rep.watermark()
        assert reached and not_reached and overwritten and stopped_at_other and split_calls, w
        assert rep.watermark() >= (w + 1) * step
        base = MM.retire_point(w, step)
        rep.retire_below(base)
        assert (w + 1) * step - step // 4 <= base <= (w + 1) * step
    assert ring_crossings >= lg * (total // step - 2)


@pytest.mark.parametrize("case", ["below", "at", "above"])
def test_wrap_batch(case):
    """The renormalisation batch: its counter values sit one below, at and one above the bound; its ranges stop at
    old entries and at Chosens of the same call; its Chosens lose to old entries and to earlier ranges."""
    lg, cap = 3, 1 << 14
    recs, claims = MM.wrap_batch(np.random.default_rng(31), lg, cap)
    n = len(recs)
    start = MM.wrap_start(n, case)
    assert (start > MM.TOP - n - 16) == (case == "above") and start + n <= MM.TOP - 15
    rep, ora = O.Replica(lg, cap), mp(lg)
    old = MM.old_entries()
    rows = MM.records([(int(s), int(s) + 1, int(v)) for s, v in old])
    assert rep.apply(rows) == MM.per_message(ora, rows, lg, cap)
    hit, _ = stops(rep.log, 0, recs, lg, cap)
    s = recs["slot_start"]
    assert all(hit[i] in set(MM.OLD.tolist()) for i in claims["stop_at_old"])
    assert all(hit[i] == s[i - 1] and s[i] < s[i - 1] for i in claims["stop_at_single"])
    assert all(s[i] in set(MM.OLD.tolist()) for i in claims["single_loses"])
    for i in claims["range_wins"]:
        assert hit[i - 1] is None or hit[i - 1] > s[i]
    assert min(len(v) for v in claims.values()) >= 20
    assert apply_both(rep, ora, recs, lg, cap) == [n]
    assert np.array_equal(ora.snapshot_log(0, cap), rep.log)
    assert (rep.log[s[claims["range_wins"]]] == O.VALUE_NOOP).all()
    assert (rep.log[s[claims["single_loses"]]] == s[claims["single_loses"]] + 1).all()


@pytest.mark.parametrize("lg", [1, 3])
def test_spaced_ranges_and_tile_positions(lg):
    """spaced_ranges: disjoint ranges at the ranks claimed, each followed by a Chosen, the restatement agreeing on a
    small one; overlap_with at every tile position overlaps exactly its partner, whose rank and tile are as
    claimed."""
    recs, at = MM.spaced_ranges(700, lg)
    assert MM.range_indices(recs, lg, 1 << 22).tolist() == at.tolist()
    rep, ora = O.Replica(lg, 3 * lg * 700 + 8 * lg), mp(lg)
    assert apply_both(rep, ora, recs, lg, rep.cap) == [len(recs)]
    assert np.array_equal(ora.snapshot_log(0, rep.cap), rep.log)
    seen = 0
    for q in MM.TILE_RANKS:
        for where in MM.PARTNERS:
            p = MM.partner_rank(q, where)
            if p is None:
                continue
            t, tp = q // MM.TILE, p // MM.TILE
            assert {"lane_below": tp == t and p == q - 1, "previous_tile": tp == t - 1 and p % MM.TILE == MM.TILE - 1,
                    "tile0": tp == 0}[where]
            k = max(q + 2, 600)
            recs, at = MM.spaced_ranges(min(k, MM.MAX_RANGE_BATCH), lg)
            i = MM.overlap_with(recs, at, lg, q, p)
            assert MM.range_indices(recs, lg, 1 << 22)[q] == i
            mine = set(range(recs["slot_start"][i], recs["slot_end"][i], lg))
            hits = [r for r in (p - 1, p, p + 1) if r != q and
                    mine & set(range(recs["slot_start"][at[r]], recs["slot_end"][at[r]], lg))]
            assert hits == [p]
            if q < 1000:
                assert O.Replica(lg, 3 * lg * k + 8 * lg).split(recs) == i
            seen += 1
    assert seen == 15


def test_range_limit_batches():
    """The rule-(b) batches: k ranges and k Chosens interleaved, range number 65 536 at the index the GPU test
    expects; one of them through the oracle and the restatement."""
    for k in (MM.MAX_RANGE_BATCH - 1, MM.MAX_RANGE_BATCH, MM.MAX_RANGE_BATCH + 1, MM.MAX_RANGE_BATCH + 2):
        recs, at = MM.spaced_ranges(k, 1)
        assert len(recs) == 2 * k and len(MM.range_indices(recs, 1, 1 << 18)) == k
        assert at[-1] == 2 * (k - 1)
    recs, at = MM.spaced_ranges(MM.MAX_RANGE_BATCH + 1, 1)
    rep, ora = O.Replica(1, 1 << 18), mp(1)
    assert apply_both(rep, ora, recs, 1, 1 << 18) == [at[MM.MAX_RANGE_BATCH], len(recs) - at[MM.MAX_RANGE_BATCH]]
    assert np.array_equal(ora.snapshot_log(0, 1 << 18), rep.log)


@pytest.mark.parametrize("lg", [3, 5])
def test_near_overlaps(lg):
    """Near-overlaps: more than one tile of ranges, every one intersecting an earlier extent in another residue, and
    one-slot and zero-slot records on top of ranges; no split, and the restatement agrees."""
    cap = 1 << 16
    recs, n_ranges = MM.near_overlaps(np.random.default_rng(lg), lg, cap)
    assert n_ranges > 2 * MM.TILE
    s, e = recs["slot_start"].astype(np.int64), recs["slot_end"].astype(np.int64)
    one = ((e - s + lg - 1) // lg == 1) & (e > s + 1)
    assert one.sum() >= n_ranges // 2 and (e == s).sum() >= n_ranges
    rep, ora = O.Replica(lg, cap), mp(lg)
    assert apply_both(rep, ora, recs, lg, cap) == [len(recs)]
    assert np.array_equal(ora.snapshot_log(0, cap), rep.log)
