"""A vanilla Mencius server's log, transcribed from S/vanillamencius/Server.scala for the revocation tests:
handlePhase2a (:1001-1082), choose (:622-640), advanceWithSkips' fill (:577-620) and handlePhase1a (:831-911).

Entries: None, ("voteless", round), ("pending", round, vote_round, value), ("chosen", value, is_revocation).
One deliberate difference, include/fpx.h fpx_vm_choose: a ChosenEntry learned with and without isRevocation
keeps isRevocation = true."""

NOOP = -(1 << 31)


class Server:
    def __init__(self, index, n, next_slot=None):
        self.index, self.n = index, n
        self.log = {}
        self.next_slot = index if next_slot is None else next_slot

    def phase2a(self, slot, round_, value):
        e = self.log.get(slot)
        if e and e[0] == "chosen":
            return ("chosen", e[1], e[2])
        if e and e[1] > round_:
            return ("nack", e[1])
        self.log[slot] = ("pending", round_, round_, value)
        return ("phase2b", round_)

    def choose(self, slot, value, is_revocation=False):
        e = self.log.get(slot)
        rev = bool(is_revocation) or bool(e and e[0] == "chosen" and e[2])
        self.log[slot] = ("chosen", value, rev)

    def advance_with_skips(self, slot):
        """The log fill; returns the skip range (start, stop) or None."""
        if self.next_slot > slot:
            return None
        new_stop = slot + 1 if slot % self.n == self.index else slot
        start = self.next_slot
        while self.next_slot < new_stop:
            assert self.next_slot not in self.log
            self.log[self.next_slot] = ("chosen", NOOP, False)
            self.next_slot += self.n
        return (start, new_stop)

    def phase1a(self, round_, start, stop):
        """('nack', start, stop, round) or ('phase1b', round, start, stop, infos) and the skip range.  infos:
        (slot, 'pending', vote_round, value) or (slot, 'chosen', value, is_revocation)."""
        skip = None
        if start % self.n == self.index:
            skip = self.advance_with_skips(stop - 1)
        infos = []
        slot = start
        while slot < stop:
            e = self.log.get(slot)
            if e is None:
                self.log[slot] = ("voteless", round_)
            elif e[0] == "voteless":
                if round_ < e[1]:
                    return ("nack", start, stop, e[1]), skip
                self.log[slot] = ("voteless", round_)
            elif e[0] == "pending":
                if round_ < e[1]:
                    return ("nack", start, stop, e[1]), skip
                infos.append((slot, "pending", e[2], e[3]))
                self.log[slot] = ("pending", round_, e[2], e[3])
            else:
                infos.append((slot, "chosen", e[1], e[2]))
            slot += self.n
        return ("phase1b", round_, start, stop, infos), skip

    def entry_row(self, slot):
        """fpx_vm_entries' row {kind, round, vote_round, value, is_revocation}"""
        e = self.log.get(slot)
        if e is None:
            return (0, -1, -1, 0, 0)
        if e[0] == "voteless":
            return (1, e[1], -1, 0, 0)
        if e[0] == "pending":
            return (2, e[1], e[2], e[3], 0)
        return (3, 0, 0, e[1], int(e[2]))
