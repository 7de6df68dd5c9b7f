"""Seeded traces that mix all eleven fpx_epaxos_* calls on one replica, for tests/test_epaxos_recovery_*.py.

The generator is adaptive: it reads the reference backend (oracle or transcription) through `entry` and the
outputs of the previous call, so every batch keeps the batch contract (E1 / E2), PrepareOks never carry a
ballot above the Preparing one, leads never hit a committed or higher-ballot entry, and every RESTART is
followed by its lead when the reference would not fatal.  Responses are a function of (instance, sender,
ballot), so a re-delivery repeats its content; the rare replacing response with new content comes alone.
"""
import random

CALLS = ("lead", "preaccept", "accept", "preacceptok", "acceptok", "commit", "nack", "prepare_phase", "prepare",
         "prepareok", "slow_path_timer")


class Trace:
    def __init__(self, f, index, per_replica, seed, ref, max_batch=8):
        self.f, self.n, self.index, self.P = f, 2 * f + 1, index, per_replica
        self.g = random.Random(seed)
        self.ref = ref                 # .entry(rep, num) -> (row, leader kind, largest ballot)
        self.max_batch = max_batch
        self.lb = {}                   # instance -> the ballot this replica last led it in
        self.maxord = 1
        self.restarts = []             # (instance, ballot, value) awaiting their lead
        self.salt = {}                 # (instance, sender, ballot, call) -> version of its response content

    # ---- helpers
    def _instances(self, k, pool=None):
        if pool is None:
            pool = [(r, m) for r in range(self.n) for m in range(self.P)]
        return self.g.sample(pool, min(k, len(pool)))

    def _k(self):
        return self.g.randint(1, self.max_batch)

    def _ballot(self):
        return [self.g.randint(0, self.maxord + 1), self.g.randrange(self.n)]

    def _deps(self):
        return [self.g.randint(0, 3) for _ in range(self.n)]

    def _det(self, *key):
        return random.Random(hash((key, self.salt.get(key, 0))))

    def _can_lead(self, inst, b):
        row = self.ref.entry(*inst)[0]
        if row[0] == 4:
            return False
        return (b[0], b[1]) >= (row[1], row[2]) and (row[0] == 1 or (b[0], b[1]) >= (row[3], row[4]))

    # ---- one call
    def step(self):
        g = self.g
        if self.restarts:
            rows = []
            for inst, b, value in self.restarts:
                if self._can_lead(inst, b):
                    rows.append([inst[0], inst[1], b[0], b[1], value, g.randint(0, 3), 1, 0] + self._deps())
                    self.lb[inst] = tuple(b)
            self.restarts = []
            if rows:
                return "lead", rows
        call = g.choice(CALLS)
        if call == "commit" and g.random() < 0.7:      # commits end an instance's story: keep them rare
            call = "nack"
        n, led = self.n, sorted(self.lb)
        if call == "lead":
            rows = []
            for inst in self._instances(self._k()):
                row = self.ref.entry(*inst)[0]
                if row[0] == 4:
                    continue
                b = (max(row[1], row[3], 0) + 1, self.index)
                self.maxord = max(self.maxord, b[0])
                rows.append([inst[0], inst[1], b[0], b[1], g.randint(0, 50), g.randint(0, 3), int(g.random() < 0.2), 0]
                            + self._deps())
                self.lb[inst] = b
            return ("lead", rows) if rows else self.step()
        if call in ("preaccept", "accept"):
            rows = []
            for inst in self._instances(self._k()):
                b = self._ballot()
                if inst in self.lb and g.random() < 0.5:
                    b = list(self.lb[inst])
                r = [inst[0], inst[1], b[0], b[1], g.randint(0, 50), g.randint(-1, 3)] + self._deps()
                rows.append(r + self._deps() if call == "preaccept" else r)
            return call, rows
        if call in ("preacceptok", "acceptok", "prepareok"):
            if not led:
                return self.step()
            replace = g.random() < 0.05             # a replacing response with new content, alone for its instance
            if replace:
                insts, k_from = self._instances(1, led), 1
            else:
                insts, k_from = self._instances(self._k(), led), n
            rows = []
            for inst in insts:
                froms = [x for x in range(n) if call == "prepareok" or x != self.index]
                for fr in g.sample(froms, g.randint(1, min(k_from, len(froms)))):
                    b = list(self.lb[inst])
                    if g.random() < 0.15:
                        b = [b[0] - 1, g.randrange(n)]             # an older ballot: ignored
                    key = (inst, fr, tuple(b), CALLS.index(call))
                    if replace:
                        self.salt[key] = self.salt.get(key, 0) + 1
                    d = self._det(*key)
                    if call == "preacceptok":
                        rows.append([inst[0], inst[1], b[0], b[1], fr, d.randint(0, 1)] + [d.randint(0, 1) for _ in range(n)])
                    elif call == "acceptok":
                        rows.append([inst[0], inst[1], b[0], b[1], fr, 0])
                    else:
                        vb = d.choice([(-1, -1), (0, d.randrange(n)), (1, d.randrange(n)), (max(b[0] - 1, 0), d.randrange(n))])
                        st = 0 if vb == (-1, -1) else d.choice([1, 1, 2])
                        rows.append([inst[0], inst[1], b[0], b[1], fr, vb[0], vb[1], st, d.randint(0, 9)])
            g.shuffle(rows)
            return call, rows
        if call == "commit":
            return call, [[i[0], i[1], g.randint(0, 50), g.randint(0, 5)] + self._deps() for i in self._instances(2)]
        if call == "nack":
            rows = []
            for _ in range(self._k()):
                inst = g.choice(led) if led and g.random() < 0.7 else self._instances(1)[0]
                b = self._ballot()
                if inst in self.lb and g.random() < 0.5:
                    b = [self.lb[inst][0] + g.randint(-1, 1), g.randrange(n)]
                rows.append([inst[0], inst[1], b[0], b[1]])
            return call, rows
        if call == "prepare_phase":
            return call, [[i[0], i[1]] for i in self._instances(g.randint(1, 3))]
        if call == "prepare":
            rows = []
            for inst in self._instances(self._k()):
                b = self._ballot()
                if inst in self.lb and g.random() < 0.5:
                    b = [self.lb[inst][0] + g.randint(-1, 1), self.lb[inst][1]]
                rows.append([inst[0], inst[1], b[0], b[1]])
            return call, rows
        # slow_path_timer
        if not led:
            return self.step()
        rows = []
        for inst in self._instances(self._k(), led):
            b = list(self.lb[inst]) if g.random() < 0.8 else self._ballot()
            rows.append([inst[0], inst[1], b[0], b[1]])
        return call, rows

    def observe(self, call, rows, out):
        if call == "prepare_phase":
            for r, b in zip(rows, out):
                self.lb[(int(r[0]), int(r[1]))] = (int(b[0]), int(b[1]))
                self.maxord = max(self.maxord, int(b[0]))
        if call == "prepareok":
            for r, ev in zip(rows, out):
                if int(ev[0]) == 1:
                    self.restarts.append(((int(r[0]), int(r[1])), (int(ev[1]), int(ev[2])), int(ev[3])))
