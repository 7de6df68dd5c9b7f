"""MultiPaxos linearizable reads on the GPU (include/fpx.h fpx_reads_*): the read-quorum tally of a Client or
a ReadBatcher, and a replica's deferred reads, on the device and stream of an Engine.

Record dtypes mirror include/fpx.h; S/ = shared/src/main/scala/frankenpaxos/ in the reference.
"""
import ctypes as C

import numpy as np

from . import _lib
from .engine import READ_REQUEST, _Handle

READS_CLIENT, READS_READ_BATCHER = 0, 1
READ_OPEN = np.dtype([("key", "<i4"), ("id", "<i4")])
# MaxSlotReply / BatchMaxSlotReply with the read's key; voter = group << 16 | acceptor
MAX_SLOT_REPLY = np.dtype([("key", "<i4"), ("id", "<i4"), ("voter", "<i4"), ("slot", "<i4")])
READ_SLOT = np.dtype([("key", "<i4"), ("id", "<i4"), ("slot", "<i4"), ("reserved", "<i4")])
READ_REPLY = np.dtype([("handle", "<i4"), ("reply_slot", "<i4"), ("after_slot", "<i4"), ("reserved", "<i4")])


class Reads(_Handle):
    """One read-quorum tally (kind READS_CLIENT: Client.handleMaxSlotReply, S/multipaxos/Client.scala:851-931;
    READS_READ_BATCHER: ReadBatcher.handleBatchMaxSlotReply, S/multipaxos/ReadBatcher.scala:568-623) and one
    replica's deferred reads (S/multipaxos/Replica.scala:394-529), on `engine`'s GPU."""

    def __init__(self, engine, kind=READS_CLIENT, key_capacity=1 << 16, pending_capacity=1 << 16, max_batch=1 << 16):
        self.engine, self.kind = engine, kind
        self.key_capacity, self.pending_capacity, self.max_batch = key_capacity, pending_capacity, max_batch
        super().__init__("fpx_reads_create", "fpx_reads_destroy", engine.h, kind, key_capacity, pending_capacity,
                         max_batch)

    def open(self, keys, ids):
        """A read request per (key, id): MaxSlot(id, {}) / batchMaxSlotReplies(id) = Map()."""
        recs = np.zeros(len(keys), READ_OPEN)
        recs["key"], recs["id"] = keys, ids
        self._host_call(self._L.fpx_reads_open, recs.ctypes.data, len(recs))

    def max_slot_replies(self, recs):
        """Replies in delivery order -> READ_SLOT records of the reads they complete, by completing reply."""
        recs = np.ascontiguousarray(recs, dtype=MAX_SLOT_REPLY)
        out = np.zeros(max(len(recs), 1), READ_SLOT)
        n = C.c_int32(0)
        self._host_call(self._L.fpx_reads_max_slot_replies, recs.ctypes.data, len(recs), out.ctypes.data, C.byref(n))
        return out[:n.value].copy()

    def replica(self, recs):
        """Read requests in delivery order -> READ_REPLY records of the reads answered now (slot < W)."""
        recs = np.ascontiguousarray(recs, dtype=READ_REQUEST)
        out = np.zeros(max(len(recs), 1), READ_REPLY)
        n = C.c_int32(0)
        self._host_call(self._L.fpx_reads_replica, recs.ctypes.data, len(recs), out.ctypes.data, C.byref(n))
        return out[:n.value].copy()

    def advance(self, watermark):
        """The replica has executed every slot below `watermark`: READ_REPLY records of the released reads."""
        out = np.zeros(self.pending_capacity, READ_REPLY)
        n = C.c_int32(0)
        self._check(self._L.fpx_reads_advance(self.h, int(watermark), out.ctypes.data, C.byref(n)))
        return out[:n.value].copy()

    # device-pointer forms (ints), asynchronous on the engine's stream; counts and status via sync()
    def max_slot_replies_dev(self, d_in, n, d_out):
        self._check(self._L.fpx_reads_max_slot_replies_dev(self.h, d_in, n, d_out))

    def replica_dev(self, d_in, n, d_out):
        self._check(self._L.fpx_reads_replica_dev(self.h, d_in, n, d_out))

    def advance_dev(self, d_watermark, d_out):
        self._check(self._L.fpx_reads_advance_dev(self.h, d_watermark, d_out))

    # -- wire codec (include/fpx.h fpx_reads_wire_*)
    def wire_decode(self, buf, offsets):
        """ClientInbound (READS_CLIENT) or ReadBatcherInbound (READS_READ_BATCHER) bytes -> (kind[n],
        MAX_SLOT_REPLY[n], spans[n, 2]); a record of another member has key -1, which the tally ignores."""
        buf = np.ascontiguousarray(buf, dtype=np.uint8)
        offsets = np.ascontiguousarray(offsets, dtype=np.int32)
        n = len(offsets) - 1
        kind = np.zeros(max(n, 1), dtype=np.int32)
        out = np.zeros(max(n, 1), dtype=MAX_SLOT_REPLY)
        spans = np.zeros((max(n, 1), 2), dtype=np.int32)
        self._host_call(self._L.fpx_reads_wire_decode, buf.ctypes.data if len(buf) else None, offsets.ctypes.data, n,
                        kind.ctypes.data, out.ctypes.data, spans.ctypes.data)
        return kind[:n], out[:n], spans[:n]

    def wire_encode_read_requests(self, recs, arena, value_offsets):
        """READ_SLOT records of completed reads -> (bytes, offsets[n+1]): ReadRequest (Client) or ReadRequestBatch
        (ReadBatcher); arena entry `key` is the message's command field(s), tag and length included."""
        recs = np.ascontiguousarray(recs, dtype=READ_SLOT)
        arena = np.ascontiguousarray(arena, dtype=np.uint8)
        value_offsets = np.ascontiguousarray(value_offsets, dtype=np.int32)
        n = len(recs)
        lens = np.diff(value_offsets)
        ok = (recs["key"] >= 0) & (recs["key"] < len(lens))
        cap = int(17 * n + lens[recs["key"][ok]].sum()) + 16    # tag, length (<= 5) and slot (<= 11) per message
        out = np.zeros(cap, dtype=np.uint8)
        offs = np.zeros(n + 1, dtype=np.int32)
        self._host_call(self._L.fpx_reads_wire_encode_read_requests, recs.ctypes.data, n,
                        arena.ctypes.data if len(arena) else None, value_offsets.ctypes.data, len(value_offsets) - 1,
                        out.ctypes.data, cap, offs.ctypes.data)
        return out[:offs[n]].copy(), offs

    def wire_decode_dev(self, d_bytes, d_offsets, n, d_kind, d_out, d_spans):
        self._check(self._L.fpx_reads_wire_decode_dev(self.h, d_bytes, d_offsets, n, d_kind, d_out, d_spans))

    def wire_encode_read_requests_dev(self, d_in, n, d_arena, d_value_offsets, num_values, d_out, out_capacity,
                                      d_offsets):
        self._check(self._L.fpx_reads_wire_encode_read_requests_dev(self.h, d_in, n, d_arena, d_value_offsets,
                                                                    num_values, d_out, out_capacity, d_offsets))

    def sync(self, check=True):
        r = _lib.ReadsSyncResult()
        st = self._L.fpx_reads_sync(self.h, C.byref(r))
        if check:
            self._check(st, r.err_index)
        return r
