"""A caller that does not know the EPaxos batch contract, for tests/test_refused_batches_*.py.  TEST INFRASTRUCTURE.

`drive` is the instruction of include/fpx.h for FPX_ERR_BATCH_ORDER and nothing more: split the batch at the
reported index and resubmit both halves.  `ContractFake` is a replica that enforces E1 / E2 the way the header
states them and refuses a batch without applying any of it; `scenario` is a scripted stream over all eleven
calls whose batches break the contract in every way a delivery order can (`run(call, rows)` executes one batch
on the replica under test and returns its dense output)."""
import random

import numpy as np

from frankenpaxos_b200.engine import FpxError

BATCH_ORDER = -12
E1_CALLS = ("lead", "preaccept", "accept", "commit", "prepare_phase", "prepare", "slow_path_timer")
RESPONSES = {"preacceptok": 1, "acceptok": 2, "prepareok": 3}    # call -> the leader kind it counts for


class Refused(RuntimeError):
    def __init__(self, status, index):
        super().__init__(f"status {status} at record {index}")
        self.status, self.index = status, index


def drive(handle, call, rows, refusals=None):
    """Run `call` on `rows`; a batch refused for its order is split at the reported index k (0 < k < len) and both
    parts are resubmitted, in order.  Returns the dense outputs concatenated (None for calls without output).
    `refusals`, if given, collects (len(batch), k) of every refusal."""
    rows = np.asarray(rows, dtype=np.int32)
    outs, todo = [], [rows]
    while todo:
        part = todo.pop()
        try:
            out = getattr(handle, call)(part)
        except (FpxError, Refused) as e:
            if e.status != BATCH_ORDER:
                raise
            k = int(e.index)
            assert 0 < k < len(part), (call, k, len(part))
            if refusals is not None:
                refusals.append((len(part), k))
            todo += [part[k:], part[:k]]
            continue
        outs.append(out)
    return None if outs[0] is None else np.concatenate(outs)


def plain(ora, call, rows):
    """the same call on a bare epaxos_recovery_oracle.EPaxos: one message after the other, no contract"""
    out = getattr(ora, call)(np.asarray(rows, dtype=np.int32))
    if call == "lead":
        assert out == (0, -1), out
        return None
    if call in ("prepare_phase", "prepareok"):
        assert out[0] == 0, (call, out[:2])
        return out[2]
    return out


class ContractFake:
    """epaxos_recovery_oracle.EPaxos behind the checked batch contract: a batch that breaks E1 or E2 (either
    clause) raises Refused(-12, k), k the later index of the first colliding pair, and nothing of it is applied.
    The oracle does not show a leader row's ballot and stored answers, so they are mirrored here."""

    def __init__(self, ora):
        self.ora, self.n, self.index = ora, ora.n, ora.index
        self.led = {}           # instance -> [leader kind the answers belong to, ballot, {sender: content}]
        self.kinds = {}         # (call, 'E1' | 'E2 sender' | 'E2 replace') -> refusals

    def entry(self, rep, num):
        return self.ora.entry(rep, num)

    def _row_state(self, inst, want):
        """the mirrored row if the oracle's leader state of `inst` is of kind `want`, else None"""
        if self.ora.entry(*inst)[1] != want or inst not in self.led:
            return None
        st = self.led[inst]
        if st[0] != want:       # PreAccepting -> Accepting happened inside the oracle: only the leader's own AcceptOk
            st[0], st[2] = want, {self.index: ()}
        return st

    def _violation(self, call, rows):
        found = []              # (later index of a colliding pair, kind)
        if call in E1_CALLS:
            first = {}
            for i, r in enumerate(rows):
                inst = (int(r[0]), int(r[1]))
                if inst in first:
                    found.append((i, "E1"))
                first.setdefault(inst, i)
        elif call in RESPONSES:
            first, counted, replacing = {}, {}, []
            for i, r in enumerate(rows):
                inst, sender = (int(r[0]), int(r[1])), int(r[4])
                st = self._row_state(inst, RESPONSES[call])
                if st is None or (int(r[2]), int(r[3])) != st[1]:
                    continue
                if (inst, sender) in first:
                    found.append((i, "E2 sender"))
                first.setdefault((inst, sender), i)
                counted.setdefault(inst, []).append(i)
                content = () if call == "acceptok" else tuple(int(x) for x in r[5:])
                if sender in st[2] and st[2][sender] != content:
                    replacing.append((i, inst))
            for i, inst in replacing:
                others = [o for o in counted[inst] if o != i]
                if others:
                    found.append((i if min(others) < i else min(others), "E2 replace"))
        return min(found) if found else None

    def _call(self, call, rows):
        rows = np.asarray(rows, dtype=np.int32)
        v = self._violation(call, rows)
        if v is not None:
            self.kinds[(call, v[1])] = self.kinds.get((call, v[1]), 0) + 1
            raise Refused(BATCH_ORDER, v[0])
        if call in RESPONSES:   # the answers the leader rows will hold, judged against the state before each message
            for r in rows:
                inst = (int(r[0]), int(r[1]))
                st = self._row_state(inst, RESPONSES[call])
                if st is not None and (int(r[2]), int(r[3])) == st[1]:
                    st[2][int(r[4])] = () if call == "acceptok" else tuple(int(x) for x in r[5:])
        out = plain(self.ora, call, rows)
        if call == "lead":
            for r in rows:      # the leader's own PreAcceptOk {seq, deps} (transitionToPreAcceptPhase)
                self.led[(int(r[0]), int(r[1]))] = [1, (int(r[2]), int(r[3])),
                                                    {self.index: tuple(int(x) for x in [r[5]] + list(r[8:]))}]
        if call == "prepare_phase":
            for r, b in zip(rows, out):
                self.led[(int(r[0]), int(r[1]))] = [3, (int(b[0]), int(b[1])), {}]
        return out


for _c in E1_CALLS + tuple(RESPONSES) + ("nack",):
    setattr(ContractFake, _c, (lambda c: lambda self, rows: self._call(c, rows))(_c))


def interleave(g, per_instance):
    """one batch out of per-instance message lists: a random merge that keeps each instance's own order"""
    keyed = []
    for msgs in per_instance:
        for key, m in zip(sorted(g.random() for _ in msgs), msgs):
            keyed.append((key, m))
    keyed.sort(key=lambda x: x[0])
    return [m for _, m in keyed]


def scenario(f, index, K, seed, run):
    """All eleven calls over K instances per step, every batch in an order the contract forbids somewhere.  Returns
    the transcript [(call, rows, out)] and the instances touched.  Adaptive only through the outputs of `run`."""
    n = 2 * f + 1
    g = random.Random(seed)
    others = [r for r in range(n) if r != index]
    col = lambda c: (index + c) % n                       # instance columns: one per family of steps
    every = max(3, K // 40)                               # one instance in `every` gets the out-of-contract extras
    log, touched = [], set()

    def step(call, rows):
        out = run(call, rows)
        log.append((call, np.asarray(rows, dtype=np.int32), None if out is None else np.asarray(out)))
        touched.update((int(r[0]), int(r[1])) for r in rows)
        return out

    def deps(x):
        return [(x + j) % 4 for j in range(n)]

    def odd(k, phase):
        return (k + phase) % every == 0

    # ---- lead: a second transition of the same instance in a higher ballot, later in the batch
    per = []
    for k in range(K):
        m = [[index, k, 1, index, k, k % 3, int(k % 5 == 1), 0] + deps(k)]
        if odd(k, 0):
            m.append([index, k, 2, index, k + 1000, 1, int(k % 2), 0] + deps(k + 1))
        per.append(m)
    step("lead", interleave(g, per))
    lead_b = {k: (2 if odd(k, 0) else 1, index) for k in range(K)}
    lead_dep = {k: deps(k + 1) if odd(k, 0) else deps(k) for k in range(K)}
    lead_seq = {k: 1 if odd(k, 0) else k % 3 for k in range(K)}

    # ---- preaccept / accept: an immediate re-delivery, then a higher and a lower ballot of the same instance
    for call, c in (("preaccept", 1), ("accept", 2)):
        per = []
        for k in range(K):
            tail = (lambda x: deps(x) + deps(x + 2)) if call == "preaccept" else deps
            first = [col(c), k, 1, col(c), k, k % 3 - 1] + tail(k)
            m = [first]
            if odd(k, 1):
                m.append(list(first))
            if odd(k, 2):
                m += [[col(c), k, 3, col(c), k + 7, 2] + tail(k + 1), [col(c), k, 2, col(c), k + 9, 0] + tail(k + 3)]
            per.append(m)
        step(call, interleave(g, per))

    # ---- preacceptok: a sender twice for an instance (same content: the copy sits where the quorum would be
    # completed; new content: the fast-path decision depends on which copy counts), and a response that replaces
    # the content an earlier CALL stored, in the middle of other responses of its instance
    same = lambda k: [lead_seq[k]] + lead_dep[k]          # what makes every answer equal: the fast path
    diff = lambda k: [lead_seq[k] + 1] + [d + 1 for d in lead_dep[k]]
    early = [k for k in range(K) if odd(k, 3) and f > 1]
    if early:
        step("preacceptok", [[index, k, *lead_b[k], others[0]] + same(k) for k in early])
    per = []
    for k in range(K):
        b, s = list(lead_b[k]), others
        if odd(k, 3) and f == 1:    # both quorums are 2: the only answer a live row holds is the leader's own
            m = [[index, k, *b, index] + diff(k), [index, k, *b, s[0]] + same(k)]
        elif odd(k, 3):     # others[0] answered in the call before; its new answer arrives among the others'
            m = [[index, k, *b, s[1]] + same(k), [index, k, *b, s[0]] + diff(k)] + [[index, k, *b, x] + same(k) for x in s[2:]]
        elif odd(k, 4):     # a plain copy ahead of the response that completes the quorum
            m = [[index, k, *b, s[0]] + same(k), [index, k, *b, s[0]] + same(k)] + [[index, k, *b, x] + same(k) for x in s[1:]]
        elif odd(k, 5):     # the second copy differs: slow path over the replaced answer instead of the fast path
            m = [[index, k, *b, s[0]] + same(k), [index, k, *b, s[1]] + same(k), [index, k, *b, s[0]] + diff(k)] \
                + [[index, k, *b, x] + same(k) for x in s[2:]]
        elif odd(k, 6):     # an old ballot among them: ignored, not counted
            m = [[index, k, b[0] - 1, b[1], s[0]] + diff(k)] + [[index, k, *b, x] + same(k) for x in s[:-1]]
        else:
            m = [[index, k, *b, x] + (diff(k) if k % 7 == 3 and x == s[-1] else same(k)) for x in s[:f + k % 2 * (f - 1)]]
        per.append(m)
    rows = interleave(g, per)
    ev = step("preacceptok", rows)
    accepting = {int(r[1]): e for r, e in zip(rows, ev) if e[0] == 2}
    timers = sorted({int(r[1]) for r, e in zip(rows, ev) if e[0] == 3})

    # ---- slow_path_timer: twice, and once in a ballot the row does not lead in
    per = []
    for k in timers:
        m = [[index, k, *lead_b[k]]]
        if odd(k, 1) or odd(k, 5):
            m.append([index, k, *lead_b[k]])
        if odd(k, 2):
            m.insert(0, [index, k, 9, index])
        per.append(m)
    if per:
        rows = interleave(g, per)
        ev = step("slow_path_timer", rows)
        accepting.update({int(r[1]): e for r, e in zip(rows, ev) if e[0] == 2})

    # ---- acceptok: copies of a sender ahead of the response that completes the slow quorum
    per = []
    for k in sorted(accepting):
        b = list(lead_b[k])
        m = [[index, k, *b, x, 0] for x in others[:f]]
        if odd(k, 1) or odd(k, 4) or k % 20 == 1:
            m.insert(1, list(m[0]))
        if odd(k, 2):
            m.insert(0, [index, k, b[0] - 1, b[1], others[-1], 0])
            m.append(list(m[-1]))
        per.append(m)
    if per:
        step("acceptok", interleave(g, per))

    # ---- commit: twice with different triples (the later one stays); nack: no order in it, copies just pass
    per = []
    for k in range(K):
        m = [[col(3), k, k, k % 4] + deps(k)]
        if odd(k, 0):
            m.append([col(3), k, k + 5, 3] + deps(k + 2))
        per.append(m)
    step("commit", interleave(g, per))
    step("nack", interleave(g, [[[index, k, 1 + k % 3, k % n]] * (2 if odd(k, 0) else 1) for k in range(K)]))

    # ---- prepare: on the PreAccepted / Accepted rows above, rising and falling ballots of one instance
    per = []
    for k in range(K):
        c = col(1 + k % 2)
        m = [[c, k, 4, k % n]]
        if odd(k, 1):
            m += [[c, k, 6, k % n], [c, k, 5, k % n]]
        if odd(k, 2):
            m.insert(0, [c, k, 0, 0])
        per.append(m)
    step("prepare", interleave(g, per))

    # ---- prepare_phase: an instance twice (the second transition starts over, in a higher ballot)
    per = [[[col(4 % n), K + k]] * (2 if odd(k, 0) else 1) for k in range(K)]
    rows = interleave(g, per)
    out = step("prepare_phase", rows)
    pb = {}
    for r, b in zip(rows, out):
        pb[int(r[1])] = [int(b[0]), int(b[1])]

    # ---- prepareok: a sender twice with different votes where its second copy decides the restart's value
    everyone = list(range(n))
    per = []
    for k in range(K):
        num, b = K + k, pb[K + k]
        ok = lambda x, vb, st, val: [col(4 % n), num, *b, x, vb, 0 if vb >= 0 else -1, st, val]
        if odd(k, 1):
            m = [ok(everyone[0], 0, 1, 11), ok(everyone[0], 1, 1, 22)] + [ok(x, 0, 1, 33) for x in everyone[1:f + 1]]
        elif odd(k, 2):
            m = [ok(everyone[0], 0, 1, 11)] * 2 + [ok(x, -1, 0, 0) for x in everyone[1:f + 1]]
        elif odd(k, 3):
            m = [ok(everyone[1], 1, 2, 44), ok(everyone[0], 1, 1, 55), ok(everyone[1], 1, 1, 66)] + \
                [ok(x, 0, 1, 77) for x in everyone[2:f + 1]]
        else:
            m = [ok(x, k % 2, 1 + k % 2, 80 + x) for x in everyone[:f + 1 - (k % 3 == 0)]]
        per.append(m)
    rows = interleave(g, per)
    ev = step("prepareok", rows)
    restarts = [[int(r[0]), int(r[1]), int(e[1]), int(e[2]), int(e[3]), 0, 1, 0] + deps(int(r[1]))
                for r, e in zip(rows, ev) if e[0] == 1]
    if restarts:
        step("lead", restarts + restarts[::every])        # some restarts led twice
    return log, sorted(touched)
