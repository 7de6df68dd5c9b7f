"""An independent Python restatement of the reference's MultiPaxos read handlers, written as a line-by-line
transcription of the Scala (dicts for mutable.Map, one message per call), sharing no code with
tests/reads_oracle.cc.  tests/test_reads_oracle.py drives both with the same random traces.

S/ = shared/src/main/scala/frankenpaxos/ in mwhittaker/frankenpaxos.
"""
from scala_transcription import Grid, IllegalArgument  # noqa: F401  (Grid.is_read_quorum raises IllegalArgument)


class ReadQuorumTally:
    """Client.handleMaxSlotReply (S/multipaxos/Client.scala:851-931) for kind 0, ReadBatcher.
    handleBatchMaxSlotReply (S/multipaxos/ReadBatcher.scala:568-623) for kind 1; one reply per call."""

    def __init__(self, kind, f, groups, per_group, flexible=False):
        self.kind, self.f, self.flexible = kind, f, flexible
        self.num_groups = groups                       # acceptors.size (Client / ReadBatcher.scala:207-211)
        self.grid = Grid([[(r, c) for c in range(per_group)] for r in range(groups)])
        self.states = {}                                # key -> (id, {voter: slot})

    def read(self, key, id_):                           # Client.scala:652-660, ReadBatcher.scala:472
        self.states[key] = (id_, {})

    def handle_max_slot_reply(self, key, id_, group, acceptor, slot):
        """-> the read's slot when this reply completes it, else None"""
        state = self.states.get(key)
        if state is None or state[0] != id_:            # :858-874 / :572-580
            return None
        replies = state[1]
        if self.kind == 0:
            replies[(group, acceptor)] = slot           # :877-879
            if not self.flexible and len(replies) < self.f + 1:
                return None
            if self.flexible and not self.grid.is_read_quorum(set(replies)):
                return None
        else:
            replies[acceptor] = slot                    # :584
            if len(replies) < self.f + 1:               # :585
                return None
        mx = max(replies.values())
        if self.kind == 0 and self.flexible:
            s = mx
        else:
            s = mx + self.num_groups - 1
        s = (s + 2 ** 31) % 2 ** 32 - 2 ** 31           # JVM Int
        del self.states[key]                            # PendingRead / batchMaxSlotReplies.remove (:601)
        return s


class ReplicaReads:
    """Replica.handleDeferrableRead (S/multipaxos/Replica.scala:463-480), executeRead (:511-529) and the
    deferred-read step of executeLog (:394-413); one read per call."""

    def __init__(self):
        self.executed_watermark = 0
        self.deferred_reads = {}                        # slot -> [handle]

    def handle_read(self, slot, handle):
        """-> (handle, ReadReply.slot, slot executed before) when answered now, else None"""
        if slot >= self.executed_watermark:
            self.deferred_reads.setdefault(slot, []).append(handle)
            return None
        return (handle, self.executed_watermark - 1, self.executed_watermark - 1)

    def execute_log(self, chosen_watermark):
        """the log's entries up to chosen_watermark are executed, one slot at a time"""
        out = []
        while self.executed_watermark < chosen_watermark:
            slot = self.executed_watermark
            for h in self.deferred_reads.pop(slot, []):
                out.append((h, self.executed_watermark - 1, slot))
            self.executed_watermark += 1
        return out
