"""The contract-unaware driver and its streams, checked without a GPU: `drive` over a replica that enforces the
EPaxos batch contract and refuses atomically must equal the bare oracle fed the undivided stream one message at a
time, and the streams must really break the contract in every way it can be broken."""
import numpy as np
import pytest

import epaxos_recovery_oracle as R
from refused_batches import E1_CALLS, ContractFake, Refused, drive, plain, scenario


def L(x):
    return None if x is None else np.asarray(x).tolist()


def entry(b, rep, num):
    row, lk, lb = b.entry(rep, num)
    return L(row), int(lk), L(lb)


def test_drive_splits_at_the_reported_index_and_keeps_the_order():
    class Pairs:
        """refuses a batch that holds a value twice, at the later index of the first such pair"""
        calls = []

        def echo(self, rows):
            seen, bad = {}, []
            for i, r in enumerate(rows[:, 0].tolist()):
                if r in seen:
                    bad.append(i)
                seen.setdefault(r, i)
            if bad:
                raise Refused(-12, min(bad))
            self.calls.append(rows[:, 0].tolist())
            return rows * 2

    h, refusals = Pairs(), []
    rows = np.array([[1], [2], [1], [3], [3], [1], [4]], dtype=np.int32)
    assert L(drive(h, "echo", rows, refusals)) == L(rows * 2)
    assert h.calls == [[1, 2], [1, 3], [3, 1, 4]] and refusals == [(7, 2), (5, 2)]

    class Fatal:
        def echo(self, rows):
            raise Refused(-13, 0)

    with pytest.raises(Refused):                  # any other status is the caller's to see
        drive(Fatal(), "echo", rows)


@pytest.mark.parametrize("f,K", [(1, 9), (2, 9), (3, 9), (1, 400), (2, 1300), (3, 400)])
def test_driven_fake_equals_the_undivided_stream_on_the_bare_oracle(f, K):
    index = f % (2 * f + 1)
    bare, fake = R.EPaxos(f, index), ContractFake(R.EPaxos(f, index))
    refusals = []
    want, insts = scenario(f, index, K, 40 + f, lambda call, rows: plain(bare, call, rows))
    got, _ = scenario(f, index, K, 40 + f, lambda call, rows: drive(fake, call, rows, refusals))
    assert len(want) == len(got)
    for (wc, wr, wo), (gc, gr, go) in zip(want, got):
        assert wc == gc and L(wr) == L(gr), wc
        assert L(wo) == L(go), wc
    for inst in insts:
        assert entry(bare, *inst) == entry(fake, *inst), inst
    # every kind of violation occurs, for every call that has a contract, and splitting recurses
    for call in E1_CALLS:
        if call != "slow_path_timer" or f >= 2:   # f = 1: slow quorum = fast quorum, the timer is never armed
            assert fake.kinds.get((call, "E1"), 0) > 0, call
    for call in ("preacceptok", "acceptok", "prepareok"):
        assert fake.kinds.get((call, "E2 sender"), 0) > 0, call
    for call in ("preacceptok", "prepareok"):
        assert fake.kinds.get((call, "E2 replace"), 0) > 0, call
    assert any(k > 1 and n - k > 1 for n, k in refusals)
    if f >= 2:
        assert "slow_path_timer" in [c for c, _, _ in want]
    # the stream exercises what it claims: every reply and event kind appears
    kinds = {c: set() for c, _, _ in want}
    for c, _, o in want:
        if o is not None:
            kinds[c] |= set(np.asarray(o)[:, 0].tolist())
    assert {1, 2} <= kinds["preaccept"] and {1, 2} <= kinds["accept"] and {1, 2} <= kinds["prepare"]
    assert {1, 2} <= kinds["preacceptok"] and 4 in kinds["acceptok"] and 1 in kinds["prepareok"]
