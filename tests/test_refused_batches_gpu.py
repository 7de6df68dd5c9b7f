"""What a caller does with FPX_ERR_BATCH_ORDER -- split the batch at the reported index and resubmit -- on the GPU,
against the CPU oracle fed the undivided stream one message at a time: a refused EPaxos call must leave the replica
exactly as it was (cmdLog entry, leader kind and largestBallot of every instance the batch names), and the split
halves must then produce the reference's replies, events and state.  The vanilla Mencius Phase2a and the Mencius
range fill return the same status for a half-applied call: there the documented way on is fpx_reset."""
import numpy as np
import pytest

import epaxos_recovery_oracle as R
import harness as H
from epaxos_recovery_traces import Trace
from frankenpaxos_b200 import CHOSEN, CHOSEN_RANGE, MENCIUS, P2A, VANILLA_MENCIUS, Engine
from frankenpaxos_b200.engine import FpxError
from frankenpaxos_b200.epaxos import EpaxosReplica
from oracle import fpx_oracle_py as O
from refused_batches import drive, plain, scenario

pytestmark = pytest.mark.gpu


def L(x):
    return None if x is None else np.asarray(x).tolist()


def entry(b, rep, num):
    row, lk, lb = b.entry(rep, num)
    return L(row), int(lk), L(lb)


def refused(fn, rows):
    with pytest.raises(FpxError) as ei:
        fn(np.asarray(rows, dtype=np.int32))
    return ei.value.status, ei.value.index


# ---------------------------------------------------------------------------- a refused call changes nothing
N = 3100
# (earlier, later) rows of the colliding pair: one warp; one 256-row tile, two warps; two tiles; either side of
# the 1024-row scan tile; first and last row
PAIRS = [(5, 20), (10, 200), (100, 700), (900, 1100), (0, N - 1)]
F, IDX = 2, 1
NR = 2 * F + 1
Z = [0] * NR


def _pool(c):
    return [(c % NR, (c // NR) * N + k) for k in range(N)]


def _setup_and_batch(call, e, I):
    """legal calls that bring the instances I of replica e into the state `call` works on (no-ops on a handle that
    has them already would not be legal, so this runs once per handle); returns (row of instance j, the same
    instance's row with different content)"""
    if call == "lead":
        return (lambda j: [*I[j], 1, IDX, j, 0, 0, 0] + [1] * NR), (lambda j: [*I[j], 2, IDX, j + 9, 1, 1, 0] + [2] * NR)
    if call in ("preaccept", "accept", "prepare"):
        e.preaccept([[*i, 2, 0, 7, 0] + Z + Z for i in I])
        if call == "prepare":
            return (lambda j: [*I[j], 3, 3]), (lambda j: [*I[j], 1 if j % 2 else 5, 3])
        tail = (lambda d: [d] * NR + Z) if call == "preaccept" else (lambda d: [d] * NR)
        return (lambda j: [*I[j], 3, 0, j, 1] + tail(1)), (lambda j: [*I[j], 1 if j % 2 else 4, 0, j + 9, 2] + tail(2))
    if call == "commit":
        return (lambda j: [*I[j], j, 1] + [1] * NR), (lambda j: [*I[j], j + 9, 2] + [2] * NR)
    if call == "nack":
        return (lambda j: [*I[j], 50 + j % 9, j % NR]), (lambda j: [NR, 0, 99, 0])
    if call == "prepare_phase":
        return (lambda j: list(I[j])), (lambda j: list(I[j]))
    if call == "prepareok":
        b = e.prepare_phase([list(i) for i in I])
        e.prepareok([[*i, int(x[0]), int(x[1]), s, 0, 0, 1, 5] for i, x in zip(I, b) for s in (0, 3)])
        return (lambda j: [*I[j], int(b[j][0]), int(b[j][1]), 2, 1, 0, 1, 6]), \
               (lambda j: [*I[j], int(b[j][0]), int(b[j][1]), 2 if j % 2 else 0, 1, 1, 1, 8])
    # the leader's rows: PreAccepting with two answers (own + 2 = slow quorum < fast quorum: the timer is armed)
    avoid = int(call == "acceptok")
    e.lead([[*i, 1, IDX, 7, 0, avoid, 0] + [1] * NR for i in I])
    ev = e.preacceptok([[*i, 1, IDX, s, 0] + [1] * NR for i in I for s in (0, 2)])
    assert set(np.asarray(ev)[:, 0].tolist()) == ({0, 2} if avoid else {0, 3})
    if call == "preacceptok":   # sender 3 completes the fast quorum; its copy, or sender 0's new answer, differs
        return (lambda j: [*I[j], 1, IDX, 3, 0] + [1] * NR), (lambda j: [*I[j], 1, IDX, 3 if j % 2 else 0, 1] + [2] * NR)
    if call == "acceptok":      # own + sender 0, then sender 3 completes the slow quorum
        e.acceptok([[*i, 1, IDX, 0, 0] for i in I])
        return (lambda j: [*I[j], 1, IDX, 3, 0]), (lambda j: [*I[j], 1, IDX, 3, 0])
    assert call == "slow_path_timer"
    return (lambda j: [*I[j], 1, IDX]), (lambda j: [*I[j], 1 if j % 2 else 3, IDX])


CALLS = ("lead", "preaccept", "accept", "preacceptok", "acceptok", "commit", "nack", "prepare_phase", "prepare",
         "prepareok", "slow_path_timer")


@pytest.mark.parametrize("call", CALLS)
def test_a_refused_call_leaves_the_replica_as_it_was(call):
    I = _pool(CALLS.index(call))
    a, twin = EpaxosReplica(F, IDX, 3 * N, 1 << 13), EpaxosReplica(F, IDX, 3 * N, 1 << 13)
    row, other = _setup_and_batch(call, a, I)
    _setup_and_batch(call, twin, I)
    before = [entry(twin, *i) for i in I]
    assert [entry(a, *i) for i in I] == before
    for p, q in PAIRS:
        # row q names the instance of row p once more, with other content (the parity of p picks which); for nack,
        # which has no contract, an instance out of range
        rows = [row(j) for j in range(N)]
        rows[q] = other(p)
        assert refused(getattr(a, call), rows) == (-6 if call == "nack" else -12, q), (call, p, q)
        after = [entry(a, *i) for i in I]
        bad = [j for j in range(N) if after[j] != before[j]]
        assert not bad, (call, (p, q), len(bad), bad[:8], after[bad[0]], before[bad[0]])
    # the handle goes on as if the refused calls had never been made: stamps, answers and scratch included
    rows = np.asarray([row(j) for j in range(N)], dtype=np.int32)
    out_a, out_t = getattr(a, call)(rows), getattr(twin, call)(rows)
    assert L(out_a) == L(out_t)
    assert [entry(a, *i) for i in I] == [entry(twin, *i) for i in I]
    a.close(); twin.close()


# ---------------------------------------------------------------------------- split and resubmit
def _compare(want, got):
    assert len(want) == len(got)
    for (wc, wr, wo), (gc, gr, go) in zip(want, got):
        assert wc == gc and np.array_equal(wr, gr), wc
        if wo is not None:
            diff = np.nonzero((np.asarray(wo) != np.asarray(go)).any(axis=1))[0]
            assert len(diff) == 0, (wc, len(diff), diff[:5].tolist(), L(wr[diff[0]]), L(wo[diff[0]]), L(go[diff[0]]))


@pytest.mark.parametrize("f,K", [(1, 9), (2, 9), (3, 9), (1, 700), (2, 3000), (3, 19000)])
def test_split_and_resubmit_equals_the_undivided_stream(f, K):
    """batches from a handful of rows to past 70 000 (f = 3, K = 19000: the PreAcceptOk batch)"""
    index = (f + K) % (2 * f + 1)
    gpu, ora = EpaxosReplica(f, index, 2 * K, 1 << 17), R.EPaxos(f, index)
    refusals = []
    want, insts = scenario(f, index, K, 7 * f + K, lambda call, rows: plain(ora, call, rows))
    got, _ = scenario(f, index, K, 7 * f + K, lambda call, rows: drive(gpu, call, rows, refusals))
    _compare(want, got)
    for inst in insts[::max(1, len(insts) // 6000)]:
        assert entry(gpu, *inst) == entry(ora, *inst), inst
    assert len(refusals) > 10 and any(k > 1 and n - k > 1 for n, k in refusals)
    if K == 19000:
        assert max(len(r) for _, r, _ in want) > 70000
    gpu.close()


class UnawareTrace(Trace):
    """the mixed trace without its care for the contract: instances are drawn with replacement, and a response
    batch may repeat a (instance, sender) with new content"""

    def _instances(self, k, pool=None):
        if pool is None:
            pool = [(r, m) for r in range(self.n) for m in range(self.P)]
        return [self.g.choice(pool) for _ in range(k)]

    def step(self):
        call, rows = super().step()
        if call in ("preacceptok", "prepareok") and self.g.random() < 0.4:
            r = list(self.g.choice(rows))
            r[-1] += 1
            rows.insert(self.g.randrange(len(rows) + 1), r)
        return call, rows


@pytest.mark.parametrize("f", [1, 2, 3])
def test_mixed_trace_that_ignores_the_contract(f):
    index, P = f, 3
    gpu, ora = EpaxosReplica(f, index, P, 4096), R.EPaxos(f, index)
    trace = UnawareTrace(f, index, P, 500 + f, ora, max_batch=8)
    refusals, seen = [], set()
    for _ in range(300):
        call, rows = trace.step()
        want = plain(ora, call, rows)
        got = drive(gpu, call, rows, refusals)
        assert L(got) == L(want), (call, rows)
        trace.observe(call, np.asarray(rows), got if got is not None else [])
        seen.add(call)
        for r in rows:
            assert entry(gpu, int(r[0]), int(r[1])) == entry(ora, int(r[0]), int(r[1])), (call, rows)
    assert len(seen) == 11 and len(refusals) > 30
    gpu.close()


# ---------------------------------------------------------------------------- the _dev forms
def test_dev_calls_queued_behind_a_refused_call_are_refused_with_it():
    torch = pytest.importorskip("torch")
    f, idx = 2, 1
    n = 2 * f + 1
    M = 2000
    gpu, twin, ora = EpaxosReplica(f, idx, M, 1 << 13), EpaxosReplica(f, idx, M, 1 << 13), R.EPaxos(f, idx)
    first = [[0, k, 1, 0, k, 0] + [1] * n + Z for k in range(M)]
    for b in (gpu, twin, ora):
        b.preaccept(np.asarray(first, dtype=np.int32))
    # refused: a second PreAccept of instance (0, 700), in a lower ballot, behind the first
    bad = [[0, k, 3, 0, k + 1, 1] + [2] * n + Z for k in range(M)]
    bad[1500] = [0, 700, 2, 0, 9, 9] + [3] * n + Z
    acc = [[0, k, 4, 0, k + 2, 2] + [3] * n for k in range(0, M, 2)]
    com = [[0, k, k + 3, 3] + [4] * n for k in range(1, M, 3)]
    dev = lambda rows: torch.from_numpy(np.asarray(rows, dtype=np.int32)).cuda()
    d_bad, d_acc, d_com = dev(bad), dev(acc), dev(com)
    r1 = torch.zeros((M, 4 + n), dtype=torch.int32, device="cuda")
    r2 = torch.zeros((len(acc), 4 + n), dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    gpu.preaccept_dev(d_bad.data_ptr(), M, r1.data_ptr())
    gpu.accept_dev(d_acc.data_ptr(), len(acc), r2.data_ptr())
    gpu.commit_dev(d_com.data_ptr(), len(com))
    with pytest.raises(FpxError) as ei:
        gpu.sync()
    assert (ei.value.status, ei.value.index) == (-12, 1500)
    assert [entry(gpu, 0, k) for k in range(M)] == [entry(twin, 0, k) for k in range(M)]
    # all three again, the first one split where it was refused
    for part in (bad[:1500], bad[1500:]):
        out = torch.zeros((len(part), 4 + n), dtype=torch.int32, device="cuda")
        d = dev(part)
        torch.cuda.synchronize()
        gpu.preaccept_dev(d.data_ptr(), len(part), out.data_ptr())
        gpu.sync()
        assert L(out.cpu()) == L(ora.preaccept(np.asarray(part, dtype=np.int32)))
    gpu.accept_dev(d_acc.data_ptr(), len(acc), r2.data_ptr())
    gpu.commit_dev(d_com.data_ptr(), len(com))
    gpu.sync()
    assert L(r2.cpu()) == L(ora.accept(np.asarray(acc, dtype=np.int32)))
    ora.commit(np.asarray(com, dtype=np.int32))
    assert [entry(gpu, 0, k) for k in range(M)] == [entry(ora, 0, k) for k in range(M)]
    gpu.close(); twin.close()


# ---------------------------------------------------------------------------- the 32-bit counters
def test_refused_call_on_the_last_batch_tag_and_under_the_stamp_wrap():
    """The refused call still consumes its batch tag and its range of response stamps: placed on the last tag, the
    claims are forgotten behind it all the same, and the halves resubmitted (numbered past the stamp wrap) count
    the responses of before the wrap."""
    f, idx = 2, 0
    n = 2 * f + 1
    K = 600
    gpu, ora = EpaxosReplica(f, idx, K, 4096), R.EPaxos(f, idx)
    lead = [[idx, k, 1, idx, k, 0, k % 2, 0] + [1] * n for k in range(K)]
    one = [[idx, k, 1, idx, 1, 0] + [1] * n for k in range(K)]
    for b in (gpu, ora):
        b.lead(np.asarray(lead, dtype=np.int32))
    assert L(gpu.preacceptok(one)) == L(ora.preacceptok(one))
    rows = [[idx, k, 1, idx, s, 0] + [1] * n for k in range(K) for s in (2, 3)]
    rows.insert(900, list(rows[40]))                      # sender 2 of instance 20 a second time
    gpu.set_counters(tag=0xfffffffe, seq_base=0xffffffff - len(rows) - 40)
    refusals = []
    got = drive(gpu, "preacceptok", rows, refusals)
    assert refusals == [(len(rows), 900)]
    c = gpu.counters()
    assert c["tag"] == 3 and c["seq_base"] < 4096         # the tag went round, the stamps were renormalized
    assert L(got) == L(ora.preacceptok(rows))
    for k in range(0, K, 7):
        assert entry(gpu, idx, k) == entry(ora, idx, k)
    # the first batches of the new tag cycle: their claims must not meet the old cycle's
    for call, batch in (("slow_path_timer", [[idx, k, 1, idx] for k in range(K)]),
                        ("acceptok", [[idx, k, 1, idx, s, 0] for k in range(K) for s in (1, 4)]),
                        ("commit", [[idx, k, k, 2] + [2] * n for k in range(0, K, 3)])):
        assert L(drive(gpu, call, batch)) == L(plain(ora, call, batch)), call
    for k in range(K):
        assert entry(gpu, idx, k) == entry(ora, idx, k)
    gpu.close()


# ---------------------------------------------------------------------------- the two half-applied refusals
def test_vanilla_mencius_phase2a_refused_then_reset_then_the_stream_cut_at_the_collision():
    f = 1
    n = 2 * f + 1
    S = 3000
    g = np.random.default_rng(3)
    eng = Engine(f, 1, n, num_leaders=f + 1, num_replicas=f + 1, slot_capacity=S, max_batch=1 << 14,
                 protocol=VANILLA_MENCIUS)
    slots = np.arange(S, dtype=np.int32)
    req = np.zeros(S, dtype=P2A)
    req["slot"] = slots; req["value_id"] = slots + 1; req["dst"] = slots % n
    p = np.zeros(S, dtype=P2A)
    p["slot"] = slots; p["round"] = 1; p["value_id"] = slots + 7; p["dst"] = (slots + 1) % n
    p = p[g.permutation(S)]
    # a second Phase2a for one (slot, server), in a lower round: the reference answers Phase2b, then Phase2Nack
    k = 2500
    dup = p[300:301].copy(); dup["round"] = 0
    stream = np.concatenate([p[:k], dup, p[k:]])
    eng.vm_client_request(req)
    with pytest.raises(FpxError) as ei:
        eng.vm_phase2a(stream)
    assert (ei.value.status, ei.value.index) == (-12, k)
    eng.reset()                                            # half applied: fatal like every other status
    ora = O.VanillaMencius(f)
    eng.vm_client_request(req); assert ora.client_request(req) == (0, -1)
    for part in (stream[:k], stream[k:]):
        H.same(eng.vm_phase2a(part), ora.phase2a(part)[2], "vanilla Phase2a replies")
    probe = p.copy(); probe["round"] = 0                   # every entry answers with the round it holds
    rep = eng.vm_phase2a(probe)
    H.same(rep, ora.phase2a(probe)[2], "probe")
    assert (rep["group"] == 1).all() and (rep["round"] == 1).all()
    eng.close()


def test_mencius_range_fill_refused_then_reset_then_the_stream_cut_at_the_collision():
    f, LG, cap = 1, 3, 1 << 16
    eng = Engine(f, 1, 3, num_leaders=2, num_replicas=2, slot_capacity=cap, max_batch=1 << 16, protocol=MENCIUS,
                 num_leader_groups=LG)
    ch = np.array([(3000, 1), (40060, 2)], dtype=CHOSEN)
    r = np.array([(0, 6000), (40000, 40100), (50000, 50010), (40030, 40200), (7, 900)], dtype=CHOSEN_RANGE)
    eng.replica_chosen(ch)
    with pytest.raises(FpxError) as ei:
        eng.mencius_replica_chosen_range(r)
    assert (ei.value.status, ei.value.index) == (-12, 3)
    eng.reset()
    ora = O.MultiPaxos(f, 1, 3, False, 2, 2, mencius_leader_groups=LG)
    eng.replica_chosen(ch); ora.replica_chosen(ch)
    for part in (r[:3], r[3:]):
        eng.mencius_replica_chosen_range(part)
        assert ora.replica_chosen_range(part, cap)[0] == 0
    H.compare_log(eng, ora, 0, cap)
    assert eng.chosen_watermark() == ora.first_hole()
    eng.close()
