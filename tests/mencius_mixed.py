"""Batch builders for the Compartmentalized Mencius replica's mixed Chosen / ChosenNoopRange call
(fpx_mencius_replica_inbound) at the edges of the mechanisms it rests on: the ring window of a log that slides,
the renormalisation of the 32-bit log numbers, and its split rules (mixed_list_kernel's range limit and
mixed_overlap_kernel's 256 x 256 tiles of rank pairs).  TEST INFRASTRUCTURE: the GPU tests
(test_mencius_mixed_replica_gpu.py) and their CPU companion (test_mencius_mixed_oracle.py) build the same batches
from here.

A record is (slot_start, slot_end, value_id); a Chosen is (s, s + 1, v), a ChosenNoopRange (s, e, Noop).  Every
builder returns its records in delivery order with the positions of the edges it claims to reach, so that the
companion can check that the edges are really there."""
import numpy as np

from wire_mencius_oracle import MAX_RANGE_BATCH, MENCIUS_CHOSEN, VALUE_NOOP

TILE = 256                       # ranks per tile of mixed_overlap_kernel (kMixThreads)
CHOSEN = np.dtype([("slot", "<i4"), ("value_id", "<i4")])
CHOSEN_RANGE = np.dtype([("slot_start", "<i4"), ("slot_end", "<i4")])
SLOT_RANGE = -6


def records(rows):
    out = np.zeros(len(rows), dtype=MENCIUS_CHOSEN)
    for i, (s, e, v) in enumerate(rows):
        out[i] = (s, e, v, 0)
    return out


def covers(s, e, lg, limit):
    """Slots the record covers; 0 for a record outside 0 <= s <= e <= limit."""
    if s < 0 or e < s or e > limit:
        return 0
    return (e - s + lg - 1) // lg


def range_indices(recs, lg, limit):
    """Record indices of the ranges (records of two or more slots), in delivery order: rank r is entry r."""
    s = recs["slot_start"].astype(np.int64)
    e = recs["slot_end"].astype(np.int64)
    ok = (s >= 0) & (e >= s) & (e <= limit)
    return np.nonzero(ok & ((e - s + lg - 1) // lg >= 2))[0]


def per_message(ora, recs, lg, limit):
    """The records applied one message at a time through the MultiPaxos oracle in Mencius mode: replica_chosen for
    a record of one slot, replica_chosen_range for the others.  A record outside 0 <= s <= e <= limit is skipped
    and its index returned with FPX_ERR_SLOT_RANGE (the first one), as the mixed call reports it."""
    st, err = 0, -1
    run, kind = [], None

    def flush():
        if not run:
            return
        if kind == 1:
            ora.replica_chosen(np.array(run, dtype=CHOSEN))
        else:
            assert ora.replica_chosen_range(np.array(run, dtype=CHOSEN_RANGE), limit) == (0, -1)
        run.clear()

    for i, r in enumerate(recs):
        s, e, v = int(r["slot_start"]), int(r["slot_end"]), int(r["value_id"])
        if s < 0 or e < s or e > limit:
            if st == 0:
                st, err = SLOT_RANGE, i
            continue
        c = covers(s, e, lg, limit)
        if c == 0:
            continue
        k = 1 if c == 1 else 2
        if k != kind:
            flush()
            kind = k
        if k == 1:
            run.append((s, v))
        else:
            assert v == VALUE_NOOP, "a record of two or more slots is a ChosenNoopRange"
            run.append((s, e))
    flush()
    return st, err


class Slots:
    """Which slots the ranges of one batch already cover (ranges of one batch are kept disjoint unless a builder
    wants an overlap), and which slots are taken by the batch's own probes."""

    def __init__(self, total, lg):
        self.lg = lg
        self.used = np.zeros(total + 1, dtype=bool)

    def free(self, s, e):
        return not self.used[s:e:self.lg].any()

    def take(self, s, e):
        self.used[s:e:self.lg] = True


def _range_at(g, sl, lo, hi, lg, min_slots=2, max_slots=24):
    """A fresh range [s, e) inside [lo, hi) of min_slots..max_slots slots whose slots no other range of the batch
    covers, or None."""
    for _ in range(200):
        k = int(g.integers(min_slots, max_slots + 1))
        if hi - lo < lg * k:
            return None
        s = int(g.integers(lo, hi - lg * (k - 1)))
        e = min(hi, s + lg * (k - 1) + int(g.integers(1, lg + 1)))
        if covers(s, e, lg, hi) >= 2 and sl.free(s, e):
            sl.take(s, e)
            return s, e
    return None


# --------------------------------------------------------------------------- 1. a sliding ring window
def retire_point(w, step):
    """Where the log is retired after window w: one half-window below the next window's start after an odd window,
    on it after an even one, so that the ring's base index is not 0 for most of the run."""
    nxt = (w + 1) * step
    return nxt - step // 4 if (w + 1) % 2 == 0 else nxt


def window_ops(g, w, lg, base, cap, step, total):
    """The calls of window w over the live window [base, base + cap), in order: [(kind, records, claims)] with kind
    'chosen' (replica_chosen, CHOSEN), 'range' (mencius_replica_chosen_range, CHOSEN_RANGE), 'mixed' (the mixed
    call, MENCIUS_CHOSEN).  `claims` maps an edge name to the record indices of the mixed batch that reach it."""
    lim = base + cap
    w0, w1 = w * step, (w + 1) * step
    ops = []
    # other writers first: the tally's Chosens and a few noop ranges, entries that mixed ranges must stop at
    other = np.unique(g.integers(w0, lim, size=max(8, (lim - w0) // 32))).astype(np.int32)
    ch = np.zeros(len(other), dtype=CHOSEN)
    ch["slot"], ch["value_id"] = other, other * 8 + 1
    ops.append(("chosen", ch, {}))
    sl = Slots(total, lg)
    rr = [_range_at(g, sl, w0, w1, lg) for _ in range(6)]
    ops.append(("range", np.array([r for r in rr if r], dtype=CHOSEN_RANGE), {}))
    for part in (0, 1):
        sl = Slots(total, lg)
        rows, claims = [], {}

        def claim(name, idx):
            claims.setdefault(name, []).append(idx)

        def add(row, name=None):
            rows.append(row)
            if name:
                claim(name, len(rows) - 1)
            return len(rows) - 1

        fresh = np.setdiff1d(np.arange(w0, w1), other)
        for _ in range(40 + 40 * part):                   # Chosens anywhere in the live window
            s = int(g.integers(w0, lim))
            add((s, s + 1, s * 8 + 2 + part))
        if base % cap:                                  # ranges across the ring's end: ring index cap - 1 -> 0
            k4 = (base // cap + 1) * cap
            for r in range(lg):
                s = k4 - lg * int(g.integers(1, 4)) - ((k4 - r) % lg)
                e = k4 + lg * int(g.integers(1, 6))
                if s >= base and e <= lim and sl.free(s, e):
                    sl.take(s, e)
                    add((s, e, VALUE_NOOP), "ring_end")
        if base > 0:
            s = max(0, base - lg * int(g.integers(1, 4)))  # straddles the retire point
            e = base + lg * int(g.integers(1, 8))
            if sl.free(s, e):
                sl.take(s, e)
                add((s, e, VALUE_NOOP), "straddle")
            lo = max(0, base - 600)
            for _ in range(3):                          # wholly retired ranges, Chosens at retired slots
                r = _range_at(g, sl, lo, base, lg, 2, 6)
                if r:
                    add((r[0], r[1], VALUE_NOOP), "retired_range")
                s = int(g.integers(0, base))
                add((s, s + 1, 5), "retired_chosen")
        # a range and a Chosen that end exactly at the live bound
        s = lim - lg * int(g.integers(2, 6))
        if sl.free(s, lim):
            sl.take(s, lim)
            add((s, lim, VALUE_NOOP), "range_at_bound")
        add((lim - 1, lim, 77), "chosen_at_bound")
        # Chosens a later range of the call reaches (the range stops at them) ...
        for _ in range(4):
            x = int(g.choice(fresh))
            s = x - lg * int(g.integers(1, 5))
            e = x + lg * int(g.integers(1, 5))
            if s >= w0 and sl.free(s, e):
                sl.take(s, e)
                add((x, x + 1, x * 8 + 4), "chosen_then_range")
                add((s, e, VALUE_NOOP), "range_after_chosen")
        # ... and Chosens it does not reach: an entry of the other writers stops it first
        for x in other[:: max(1, len(other) // 4)][:4]:
            x = int(x)
            s, y = x - lg * int(g.integers(1, 4)), x + lg * int(g.integers(1, 4))
            e = y + lg
            if s >= w0 and e <= w1 and sl.free(s, e):
                sl.take(s, e)
                add((y, y + 1, y * 8 + 5), "chosen_not_reached")
                add((s, e, VALUE_NOOP), "range_stops_at_other")
        # Chosens delivered after a range that reaches their slot: the range's earlier number wins
        for _ in range(4):
            r = _range_at(g, sl, w0, w1, lg, 4, 12)
            if r:
                add((r[0], r[1], VALUE_NOOP), "range_then_chosen")
                x = r[0] + lg
                add((x, x + 1, x * 8 + 6), "chosen_after_range")
        for _ in range(20):                             # more ranges of the live window
            r = _range_at(g, sl, w0, lim, lg)
            if r:
                add((r[0], r[1], VALUE_NOOP))
        mine = [i for i, r in enumerate(rows) if covers(r[0], r[1], lg, lim) >= 2 and r[0] >= base]
        i = mine[int(g.integers(0, len(mine)))]     # a range re-proposed: overlaps an earlier one, splits the call
        add((rows[i][0] + lg, min(lim, rows[i][1] + lg), VALUE_NOOP), "overlap")
        order = g.permutation(len(rows))
        # keep the pairs whose order matters in their order: sort each claimed pair's members by position
        rows = _keep_pairs(rows, claims, order)
        rows, claims = rows
        # one record past the live bound, reported at its index while the rest is applied
        bad_at = int(g.integers(0, len(rows)))
        bad = (lim, lim + 1, 9) if (w + part) % 2 else (lim - lg, lim + 1, VALUE_NOOP)
        rows.insert(bad_at, bad)
        claims = {k: [i + (i >= bad_at) for i in v] for k, v in claims.items()}
        claims["past_bound"] = [bad_at]
        if part == 1 and w % 2 == 0:                     # the mixed call closes the window
            first = len(rows)
            rows.extend((s, s + 1, s * 8 + 7) for s in range(w0, w1))
            claims["closing"] = list(range(first, len(rows)))
        ops.append(("mixed", records(rows), claims))
        if part == 0:                                   # the other writers again, between the two mixed calls
            more = np.unique(g.integers(w0, lim, size=16)).astype(np.int32)
            ch = np.zeros(len(more), dtype=CHOSEN)
            ch["slot"], ch["value_id"] = more, more * 8 + 3
            ops.append(("chosen", ch, {}))
            sl2 = Slots(total, lg)
            rr = [_range_at(g, sl2, w0, lim, lg) for _ in range(3)]
            ops.append(("range", np.array([r for r in rr if r], dtype=CHOSEN_RANGE), {}))
    if w % 2 == 1:                                      # the tally's Chosens close the window
        close = np.arange(w0, w1, dtype=np.int32)
        ch = np.zeros(len(close), dtype=CHOSEN)
        ch["slot"], ch["value_id"] = close, close * 8 + 7
        ops.append(("chosen", ch, {}))
    return ops


_PAIRS = (("chosen_then_range", "range_after_chosen"), ("chosen_not_reached", "range_stops_at_other"),
          ("range_then_chosen", "chosen_after_range"))


def _keep_pairs(rows, claims, order):
    """Shuffle the rows by `order` but keep each claimed pair's two members in their original order."""
    pos = np.empty(len(rows), dtype=np.int64)
    pos[order] = np.arange(len(rows))
    for a, b in _PAIRS:
        for i, j in zip(claims.get(a, []), claims.get(b, [])):
            if pos[i] > pos[j]:
                pos[i], pos[j] = pos[j], pos[i]
    inv = np.argsort(pos)
    new_rows = [rows[k] for k in inv]
    where = np.empty(len(rows), dtype=np.int64)
    where[inv] = np.arange(len(rows))
    return new_rows, {k: [int(where[i]) for i in v] for k, v in claims.items()}   # pair members stay aligned


def ring_index(slot, base, cap):
    """Ring index of a live slot of an unsharded engine of `cap` slots: its ordinal modulo the ring."""
    assert base <= slot < base + cap
    return slot % cap


# --------------------------------------------------------------------------- 2. the log-number renormalisation
TOP = 0xFFFFFFFF
OLD = np.arange(0, 6000, 10, dtype=np.int32)     # entries put just below the top before the call


def old_entries():
    ch = np.zeros(len(OLD), dtype=CHOSEN)
    ch["slot"], ch["value_id"] = OLD, OLD + 1
    return ch


def wrap_start(n, case):
    """rseq_base for a call of n records one below ('below'), at ('at') and one above ('above') the bound of
    renormalize_rlog_if_needed: the call renormalises iff rseq_base > 2^32 - 1 - n - 16."""
    return {"below": TOP - n - 17, "at": TOP - n - 16, "above": TOP - n - 15}[case]


def wrap_batch(g, lg, cap):
    """A mixed batch over a log whose slots OLD hold entries put just before it (old_entries).  Claims:
    stop_at_old     ranges whose first covered slot in the log is an old entry;
    stop_at_single  ranges that must stop at a Chosen delivered earlier in the same call;
    single_loses    Chosens for old slots, with another value;
    range_wins      Chosens delivered after a range that reaches their slot."""
    sl = Slots(cap, lg)
    old = set(OLD.tolist())
    rows, claims = [], {}

    def add(row, name=None):
        rows.append(row)
        if name:
            claims.setdefault(name, []).append(len(rows) - 1)

    taken = set()
    for _ in range(60):                                 # ranges stopping at old entries
        s = int(g.integers(1, 5900))
        if s % 10 == 0:
            continue
        stop = next(x for x in range(s, 6000, lg) if x in old)
        e = stop + lg * int(g.integers(1, 4))
        if sl.free(s, e):
            sl.take(s, e)
            add((s, e, VALUE_NOOP), "stop_at_old")
    for _ in range(60):                                 # Chosens for old slots lose
        x = int(g.choice(OLD))
        add((x, x + 1, 900000 + x), "single_loses")
    for _ in range(60):                                 # a Chosen, then a range stopping at it
        x = int(g.integers(6000 + 3 * lg, 12000))
        s, e = x - lg * int(g.integers(1, 4)), x + lg * int(g.integers(1, 4))
        if x not in taken and sl.free(s, e):
            sl.take(s, e)
            taken.add(x)
            add((x, x + 1, 800000 + x))
            add((s, e, VALUE_NOOP), "stop_at_single")
    for _ in range(60):                                 # a range, then a Chosen it overwrote
        r = _range_at(g, sl, 6000, 12000, lg, 3, 10)
        if r and r[0] + lg not in taken:
            add((r[0], r[1], VALUE_NOOP))
            x = r[0] + lg
            taken.add(x)
            add((x, x + 1, 700000 + x), "range_wins")
    for _ in range(800):                                # filler Chosens
        x = int(g.integers(0, cap))
        add((x, x + 1, 600000 + x))
    return records(rows), claims


# --------------------------------------------------------------------------- 3. the split rules
def spaced_ranges(k, lg, with_chosens=True):
    """k disjoint ranges of two slots, range r covering slots 3 * lg * r and 3 * lg * r + lg (residue 0), each
    followed by a Chosen of slot 3 * lg * r + 2 * lg.  Returns (records, record index of each rank)."""
    per = 2 if with_chosens else 1
    recs = np.zeros(per * k, dtype=MENCIUS_CHOSEN)
    b = 3 * lg * np.arange(k, dtype=np.int64)
    recs["slot_start"][0::per] = b
    recs["slot_end"][0::per] = b + lg + 1
    recs["value_id"][0::per] = VALUE_NOOP
    if with_chosens:
        recs["slot_start"][1::2] = b + 2 * lg
        recs["slot_end"][1::2] = b + 2 * lg + 1
        recs["value_id"][1::2] = b + 2 * lg + 3
    return recs, np.arange(0, per * k, per)


def overlap_with(recs, at, lg, q, p):
    """Make range of rank q share exactly one slot with the range of rank p < q: it covers p's second slot and p's
    Chosen's slot (not a range's)."""
    i, j = at[q], at[p]
    s = int(recs["slot_start"][j]) + lg
    recs[i] = (s, s + lg + 1, VALUE_NOOP, 0)
    return i


TILE_RANKS = (255, 256, 257, 511, 512, MAX_RANGE_BATCH - 1)
PARTNERS = ("lane_below", "previous_tile", "tile0")


def partner_rank(q, where):
    """The earlier range of an overlapping pair relative to mixed_overlap_kernel's tiles: one lane below in q's tile,
    the last lane of the previous tile, or in tile 0.  None where q's tile has no such position."""
    t = q // TILE
    if where == "lane_below":
        return q - 1 if q % TILE else None
    if where == "previous_tile":
        return t * TILE - 1 if t >= 1 else None
    return 3 if t >= 1 else (q - 5 if q >= 5 else None)


def near_overlaps(g, lg, cap):
    """Records that look like an overlap but must not split the batch (lg > 1): ranges whose extents intersect
    but start in different residues, records of one slot whose slot_end > slot_start + 1, and zero-slot records,
    each on top of an earlier range.  Returns (records, number of ranges)."""
    rows = []
    s0 = 0
    while s0 + 12 * lg < cap and len(rows) < 4000:
        e = s0 + 6 * lg
        rows.append((s0, e, VALUE_NOOP))                 # a range of residue s0 % lg
        rows.append((s0 + 1, e + 1, VALUE_NOOP))         # same extent shifted: the next residue
        x = s0 + 2 * lg
        rows.append((x, x + lg, VALUE_NOOP))             # one slot although slot_end > slot_start + 1
        rows.append((x + lg, x + lg + 2 if lg > 2 else x + lg + 1, 41))
        rows.append((s0 + lg, s0 + lg, VALUE_NOOP))      # no slot
        rows.append((s0 + 3, s0 + 3, 5))
        s0 += 12 * lg + int(g.integers(0, lg))
    recs = records(rows)
    return recs, len(range_indices(recs, lg, cap))
