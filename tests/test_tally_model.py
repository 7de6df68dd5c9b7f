"""The tally kernel's arithmetic, checked on the CPU against the oracle (no GPU): with every vote numbered in
delivery order and a key keeping, per voter, the SMALLEST number that voter was delivered with, the vote that
sends Chosen has a closed form -- the (f+1)-th smallest stamp of the key (non-flexible, ProxyLeader.scala:238), or
the maximum over grid rows of the row's minimum stamp (flexible, Grid.isWriteQuorum, Grid.scala:49) -- and the
Chosen stream is the keys ordered by that number, restricted to the numbers of the running batch.  This is what
fpx_tally.cuh's row sweep evaluates (DESIGN.md section 2); here the rule itself meets the sequential handlers."""
import numpy as np
import pytest

import harness as H
from frankenpaxos_b200 import traces as T
from frankenpaxos_b200.engine import P2B
from oracle import fpx_oracle_py as O

EMPTY = np.iinfo(np.int64).max


def closed_form_chosen(stamps, value, f, flexible, groups, per_group, lo, hi):
    """stamps[slot, voter] -> [(slot, value)] of the keys whose completing vote number lies in [lo, hi), in order."""
    if not flexible:
        c = np.sort(stamps, axis=1)[:, f]                                        # (f+1)-th smallest first delivery
    else:
        c = stamps.reshape(len(stamps), groups, per_group).min(axis=2).max(axis=1)   # one member of every row
    hit = np.nonzero((c >= lo) & (c < hi))[0]
    order = hit[np.argsort(c[hit], kind="stable")]
    return [(int(s), int(value[s])) for s in order]


@pytest.mark.parametrize("name", ["cfg1", "cfg2", "cfg3", "maj7", "grid2x7", "maj15", "groups2x15", "maj29", "grid5x6"])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_closed_form_completing_vote_matches_the_sequential_handlers(name, seed):
    """cfg1-cfg3: 3, 5 and 6 voters (8-word rows); maj7 and grid2x7: 7 and 14 voters (16-word rows); maj15,
    groups2x15, maj29 and grid5x6: 15, 15, 29 and 30 voters (32-word rows)."""
    cfg = H.WIDE_SHAPES[name] if name in H.WIDE_SHAPES else T.config_by_name(name)[0]
    n_slots = 3000
    f, G, A, flexible = cfg["f"], cfg["num_acceptor_groups"], cfg["acceptors_per_group"], cfg["flexible"]
    g = T.rng(700 + seed)
    a, p, b = T.workload(seed, cfg, n_slots)
    # non-thrifty extras, duplicates and late re-deliveries on top of the thrifty quorum's votes
    extra = b[g.integers(0, len(b), len(b) // 3)]
    votes = np.concatenate([b, extra])
    votes = votes[g.permutation(len(votes))]
    ora = O.MultiPaxos(f, G, A, flexible, cfg["num_leaders"], cfg["num_replicas"])
    assert ora.arm(a) == (0, -1)
    voters = G * A if flexible else A
    stamps = np.full((n_slots, voters), EMPTY, dtype=np.int64)
    value = np.zeros(n_slots, dtype=np.int64)
    value[a["slot"]] = a["value_id"]
    seq = 0
    for chunk in np.array_split(votes, 7):                                       # seven batches: earlier batches' stamps count
        st, _, oc = ora.proxyleader_phase2b(chunk)
        assert st == 0
        v = chunk["group"] * A + chunk["acceptor"] if flexible else chunk["acceptor"]
        np.minimum.at(stamps, (chunk["slot"], v), seq + np.arange(len(chunk)))   # first delivery per voter
        want = closed_form_chosen(stamps, value, f, flexible, G, A, seq, seq + len(chunk))
        assert oc.tolist() == want
        seq += len(chunk)
    assert (np.sort(stamps, axis=1)[:, f] != EMPTY).all() if not flexible else True


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_keyed_prefix_max_rule_of_the_acceptor_kernel_matches_the_sequential_handler(seed):
    """fpx_acceptor.cuh: `round` is one scalar per acceptor (Acceptor.scala:95), so record i to acceptor k is accepted
    iff round_i >= max(round_k at batch start, max over earlier records j to k of round_j) -- rejected records are
    below the running max, so including them changes nothing -- and a Nack carries that running max.  numpy's
    keyed exclusive prefix-max against the oracle's sequential handler, rounds going up and down."""
    cfg, _ = T.config_by_name("cfg2")
    f, G, A = cfg["f"], cfg["num_acceptor_groups"], cfg["acceptors_per_group"]
    g = T.rng(900 + seed)
    ora = O.MultiPaxos(f, G, A, False, cfg["num_leaders"], cfg["num_replicas"])
    start = np.full(A, -1, dtype=np.int64)
    for batch in range(4):
        n = 5000
        recs = np.zeros(n, dtype=T.P2A)
        recs["slot"] = g.integers(0, 4000, n)
        # mostly one round, sprinkled with higher and lower ones (leader changes, stale leaders)
        recs["round"] = batch + g.choice([0, 0, 0, 0, 0, 0, 1, 2, -1], n).clip(-batch, None)
        recs["value_id"] = g.integers(0, 1 << 20, n)
        acc = g.integers(0, A, n)
        recs["dst"] = acc
        st, _, ob, on = ora.acceptor_phase2a(recs)
        assert st == 0
        run = np.empty(n, dtype=np.int64)                     # exclusive prefix max per acceptor, seeded with `start`
        for k in range(A):
            idx = np.nonzero(acc == k)[0]
            r = recs["round"][idx].astype(np.int64)
            incl = np.maximum.accumulate(np.concatenate([[start[k]], r]))
            run[idx] = incl[:-1]
            start[k] = incl[-1]
        accept = recs["round"] >= run
        assert ob["slot"].tolist() == recs["slot"][accept].tolist() and ob["round"].tolist() == recs["round"][accept].tolist()
        assert ob["acceptor"].tolist() == acc[accept].tolist()
        assert on["round"].tolist() == run[~accept].tolist()                     # Nack(round) (:197-198)
        assert on["leader"].tolist() == (recs["round"][~accept] % cfg["num_leaders"]).tolist()
        for k in range(A):
            assert ora.snapshot_acceptor(0, k, 0, 1)[0] == start[k]
