"""Seeded traces of the MultiPaxos read path (include/fpx.h fpx_reads_*) and drivers that run them on the GPU
handle, the CPU oracle and the Python transcription, for tests/test_reads_oracle.py and tests/test_reads_gpu.py."""
import numpy as np

from harness import WIDE_SHAPES
import reads_oracle as RO

SHAPES = {
    "cfg1": dict(f=1, num_acceptor_groups=1, acceptors_per_group=3, flexible=False, num_leaders=2, num_replicas=2),
    "maj5": dict(f=2, num_acceptor_groups=1, acceptors_per_group=5, flexible=False, num_leaders=3, num_replicas=3),
    "groups2x3": dict(f=1, num_acceptor_groups=2, acceptors_per_group=3, flexible=False, num_leaders=2,
                      num_replicas=2),
    "grid2x3": dict(f=1, num_acceptor_groups=2, acceptors_per_group=3, flexible=True, num_leaders=2, num_replicas=2),
    "maj15": WIDE_SHAPES["maj15"],
    "grid5x6": WIDE_SHAPES["grid5x6"],
}


def voter(group, acceptor):
    return (np.asarray(group, np.int64) << 16 | np.asarray(acceptor, np.int64)).astype(np.int32)


def read_batcher_voters(cfg, g, n):
    """n random BatchMaxSlotReply voters: an acceptor index of the config; the reply carries no group, so any
    group number may stand in the word (ReadBatcher.scala:584)."""
    return voter(g.integers(0, 1 << 15, n), g.integers(0, cfg["acceptors_per_group"], n))


def tally_trace(seed, cfg, kind, key_capacity, n_batches, batch, hot_keys=0, slot_hi=1 << 20):
    """[("open", keys, ids) | ("replies", MAX_SLOT_REPLY recs)]: opens and re-opens, duplicates and overwrites
    (slots in any order), stale ids, replies after completion, unopened keys and keys outside the handle."""
    g = np.random.default_rng(seed)
    G = cfg["num_acceptor_groups"]
    ids = np.zeros(key_capacity, np.int64)
    trace = []
    for b in range(n_batches):
        n_open = max(1, key_capacity // (2 * n_batches) if b else key_capacity // 2)
        keys = g.integers(0, key_capacity, n_open).astype(np.int32)
        ids[keys] += g.integers(1, 3, n_open)
        trace.append(("open", keys, ids[keys].astype(np.int32)))
        recs = np.zeros(batch, RO.MAX_SLOT_REPLY)
        k = g.integers(0, key_capacity, batch)
        if hot_keys:
            hot = g.random(batch) < 0.5
            k[hot] = g.integers(0, hot_keys, hot.sum())
        recs["key"] = k
        recs["id"] = ids[k]
        stale = g.random(batch) < 0.08
        recs["id"][stale] -= 1
        out = g.random(batch) < 0.01
        recs["key"][out] = key_capacity + g.integers(0, 5, out.sum())
        neg = g.random(batch) < 0.005
        recs["key"][neg] = -1 - g.integers(0, 5, neg.sum())
        if kind == 0:
            # a Client asks one group, or one row of the grid (Client.scala:626-636): here the key's (rarely another)
            grp = (k % G).astype(np.int64)
            other = g.random(batch) < 0.02
            grp[other] = g.integers(0, G, other.sum())
            recs["voter"] = voter(grp, g.integers(0, cfg["acceptors_per_group"], batch))
        else:
            recs["voter"] = read_batcher_voters(cfg, g, batch)
        s = g.integers(-1, slot_hi, batch)
        wrap = g.random(batch) < 0.01
        s[wrap] = (1 << 31) - 1 - g.integers(0, 4, wrap.sum())
        recs["slot"] = s
        trace.append(("replies", recs))
    return trace


def run_tally(h, trace):
    """Engine Reads or oracle ReadTally -> one READ_SLOT array per replies batch."""
    outs = []
    for op in trace:
        if op[0] == "open":
            h.open(op[1], op[2])
        else:
            r = h.max_slot_replies(op[1])
            if isinstance(r, tuple):
                st, err, r = r
                assert st == 0, (st, err)
            outs.append(r)
    return outs


def run_tally_transcription(t, trace):
    outs = []
    for op in trace:
        if op[0] == "open":
            for k, i in zip(op[1], op[2]):
                t.read(int(k), int(i))
            continue
        done = []
        for r in op[1]:
            s = t.handle_max_slot_reply(int(r["key"]), int(r["id"]), int(r["voter"]) >> 16 & 0xffff,
                                        int(r["voter"]) & 0xffff, int(r["slot"]))
            if s is not None:
                done.append((int(r["key"]), int(r["id"]), s, 0))
        outs.append(np.array(done, RO.READ_SLOT))
    return outs


def replica_trace(seed, n_batches, batch, start=0, step=64, spread=96):
    """[("req", READ_REQUEST recs) | ("adv", W)]: slots below, at and above W (ties), eventual reads."""
    g = np.random.default_rng(seed)
    W, handle, trace = start, 0, []
    for _ in range(n_batches):
        recs = np.zeros(batch, RO.READ_REQUEST)
        s = W + g.integers(-spread // 4, spread, batch)
        s[g.random(batch) < 0.05] = -1
        s[g.random(batch) < 0.1] = W
        recs["slot"] = np.maximum(s, -1)
        recs["handle"] = handle + np.arange(batch)
        handle += batch
        trace.append(("req", recs))
        W += int(g.integers(0, step))
        trace.append(("adv", W))
    return trace


def run_replica(h, trace):
    outs = []
    for op in trace:
        if op[0] == "req":
            r = h.replica(op[1])
        else:
            r = h.advance(op[1])
        if isinstance(r, tuple):
            assert r[0] == 0, r
            r = r[-1]
        outs.append(r)
    return outs


def run_replica_transcription(t, trace):
    outs = []
    for op in trace:
        if op[0] == "req":
            now = [t.handle_read(int(r["slot"]), int(r["handle"])) for r in op[1]]
            outs.append(np.array([x + (0,) for x in now if x is not None], RO.READ_REPLY))
        else:
            outs.append(np.array([x + (0,) for x in t.execute_log(op[1])], RO.READ_REPLY))
    return outs


def same_outputs(a, b, what):
    assert len(a) == len(b), what
    for i, (x, y) in enumerate(zip(a, b)):
        x = np.asarray(x).view(np.int32).reshape(-1)
        y = np.asarray(y).view(np.int32).reshape(-1)
        assert x.shape == y.shape, f"{what} step {i}: {x.shape} vs {y.shape}"
        if not np.array_equal(x, y):
            bad = np.nonzero(x != y)[0][0]
            raise AssertionError(f"{what} step {i}: first difference at int {bad}: {x[bad]} vs {y[bad]}")
