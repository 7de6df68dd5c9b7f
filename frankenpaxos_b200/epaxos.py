"""Python handle over the EPaxos entry points of include/fpx.h (one replica's cmdLog +
leaderStates; shared/src/main/scala/frankenpaxos/epaxos/Replica.scala).  Messages are
int32 matrices, one row per message, dependency sets dense watermark vectors."""
import ctypes as C

import numpy as np

from . import _lib
from ._lib import EpaxosConfig
from .engine import FpxError, _Handle

REPLY_NONE, REPLY_OK, REPLY_NACK, REPLY_COMMIT = 0, 1, 2, 3
EV_NONE, EV_FAST_COMMIT, EV_SLOW_ACCEPT, EV_TIMER, EV_COMMIT = 0, 1, 2, 3, 4
EV_RECOVER_TIMER = 1    # nack(): (re)arm the instance's recoverInstance timer
EV_RESTART = 1          # prepareok(): run lead(avoid_fast_path = 1) in the returned ballot with the returned value
LEADER_NONE, LEADER_PREACCEPTING, LEADER_ACCEPTING, LEADER_PREPARING = 0, 1, 2, 3
STATUS_NOT_SEEN, STATUS_PRE_ACCEPTED, STATUS_ACCEPTED = 0, 1, 2
VALUE_NOOP = -(1 << 31)
# handler calls of the wire codec (include/fpx.h FPX_EP_CALL_*)
CALL_LEAD, CALL_PREACCEPT, CALL_ACCEPT, CALL_PREACCEPTOK, CALL_ACCEPTOK, CALL_COMMIT, CALL_NACK, CALL_PREPARE_PHASE, \
    CALL_PREPARE, CALL_PREPAREOK, CALL_SLOW_PATH_TIMER = range(11)
WIRE_COLS = 12          # a decoded row: 12 + n ints


def wire_pack_width(call, n):
    """ints per row of the handler input that fpx_epaxos_wire_pack writes for `call`"""
    return {CALL_PREACCEPT: 6 + 2 * n, CALL_ACCEPT: 6 + n, CALL_PREACCEPTOK: 6 + n, CALL_ACCEPTOK: 6,
            CALL_COMMIT: 4 + n, CALL_NACK: 4, CALL_PREPARE: 4, CALL_PREPAREOK: 9}.get(call, 1)


class EpaxosReplica(_Handle):
    def __init__(self, f, replica_index, instances_per_replica, max_batch=1 << 16, device=0):
        cfg = EpaxosConfig(C.sizeof(EpaxosConfig), f, replica_index, instances_per_replica, max_batch, device)
        self.f, self.n, self.index = f, 2 * f + 1, replica_index
        super().__init__("fpx_epaxos_create", "fpx_epaxos_destroy", C.byref(cfg))

    def _call(self, fn, rows, width, out_width):
        rows = np.ascontiguousarray(rows, dtype=np.int32).reshape(-1, width)
        out = np.zeros((max(len(rows), 1), max(out_width, 1)), dtype=np.int32)
        self._host_call(fn, rows.ctypes.data, len(rows), *((out.ctypes.data,) if out_width else ()))
        return out[:len(rows)]

    def lead(self, rows):
        """rows: {inst_replica, inst_number, b_ord, b_rep, value_id, seq, avoid_fast_path, 0, deps[n]}"""
        self._call(self._L.fpx_epaxos_lead, rows, 8 + self.n, 0)

    def preaccept(self, rows):
        """rows: {inst_replica, inst_number, b_ord, b_rep, value_id, seq, local_deps[n], msg_deps[n]}
        -> replies {kind, b_ord, b_rep, seq, deps[n]}"""
        return self._call(self._L.fpx_epaxos_preaccept, rows, 6 + 2 * self.n, 4 + self.n)

    def accept(self, rows):
        return self._call(self._L.fpx_epaxos_accept, rows, 6 + self.n, 4 + self.n)

    def preacceptok(self, rows):
        """rows: {inst_replica, inst_number, b_ord, b_rep, from, seq, deps[n]} -> events {kind, seq, deps[n]}"""
        return self._call(self._L.fpx_epaxos_preacceptok, rows, 6 + self.n, 2 + self.n)

    def acceptok(self, rows):
        return self._call(self._L.fpx_epaxos_acceptok, rows, 6, 2 + self.n)

    # -- recovery and the timer-driven transitions (include/fpx.h)
    def commit(self, rows):
        """rows: {inst_replica, inst_number, value_id, seq, deps[n]} (handleCommit); no reply"""
        self._call(self._L.fpx_epaxos_commit, rows, 4 + self.n, 0)

    def nack(self, rows):
        """rows: {inst_replica, inst_number, lb_ord, lb_rep} -> events {kind} (EV_RECOVER_TIMER)"""
        return self._call(self._L.fpx_epaxos_nack, rows, 4, 1)

    def prepare_phase(self, rows):
        """rows: {inst_replica, inst_number} -> {b_ord, b_rep}, the ballot of the Prepare to send"""
        return self._call(self._L.fpx_epaxos_prepare_phase, rows, 2, 2)

    def prepare(self, rows):
        """rows: {inst_replica, inst_number, b_ord, b_rep}
        -> replies {kind, yielded, b_ord, b_rep, vb_ord, vb_rep, status, value_id, seq, deps[n]}"""
        return self._call(self._L.fpx_epaxos_prepare, rows, 4, 9 + self.n)

    def prepareok(self, rows):
        """rows: {inst_replica, inst_number, b_ord, b_rep, from, vb_ord, vb_rep, status, value_id}
        -> events {kind, b_ord, b_rep, value_id} (EV_RESTART)"""
        return self._call(self._L.fpx_epaxos_prepareok, rows, 9, 4)

    def slow_path_timer(self, rows):
        """rows: {inst_replica, inst_number, b_ord, b_rep} -> events {kind, seq, deps[n]} (EV_SLOW_ACCEPT)"""
        return self._call(self._L.fpx_epaxos_slow_path_timer, rows, 4, 2 + self.n)

    def last_kernel_ms(self):
        return float(self._L.fpx_epaxos_last_kernel_ms(self.h))

    # -- device-pointer calls (asynchronous on self.stream; errors collected by sync())
    @property
    def stream(self):
        return self._L.fpx_epaxos_stream(self.h)

    def sync(self):
        self._host_call(self._L.fpx_epaxos_sync)

    def lead_dev(self, d_in, n):
        self._check(self._L.fpx_epaxos_lead_dev(self.h, d_in, n))

    def preaccept_dev(self, d_in, n, d_reply):
        self._check(self._L.fpx_epaxos_preaccept_dev(self.h, d_in, n, d_reply))

    def accept_dev(self, d_in, n, d_reply):
        self._check(self._L.fpx_epaxos_accept_dev(self.h, d_in, n, d_reply))

    def preacceptok_dev(self, d_in, n, d_event):
        self._check(self._L.fpx_epaxos_preacceptok_dev(self.h, d_in, n, d_event))

    def acceptok_dev(self, d_in, n, d_event):
        self._check(self._L.fpx_epaxos_acceptok_dev(self.h, d_in, n, d_event))

    def commit_dev(self, d_in, n):
        self._check(self._L.fpx_epaxos_commit_dev(self.h, d_in, n))

    def nack_dev(self, d_in, n, d_event):
        self._check(self._L.fpx_epaxos_nack_dev(self.h, d_in, n, d_event))

    def prepare_phase_dev(self, d_in, n, d_ballot):
        self._check(self._L.fpx_epaxos_prepare_phase_dev(self.h, d_in, n, d_ballot))

    def prepare_dev(self, d_in, n, d_reply):
        self._check(self._L.fpx_epaxos_prepare_dev(self.h, d_in, n, d_reply))

    def prepareok_dev(self, d_in, n, d_event):
        self._check(self._L.fpx_epaxos_prepareok_dev(self.h, d_in, n, d_event))

    def slow_path_timer_dev(self, d_in, n, d_event):
        self._check(self._L.fpx_epaxos_slow_path_timer_dev(self.h, d_in, n, d_event))

    def preaccept_sets(self, rows, overflow_count):
        """handlePreAccept for possibly sparse sets: FPX_ERR_UNSUPPORTED at the first message that carries
        overflow values (this handle computes with dense watermark vectors)."""
        rows = np.ascontiguousarray(rows, dtype=np.int32).reshape(-1, 6 + 2 * self.n)
        oc = np.ascontiguousarray(overflow_count, dtype=np.int32)
        out = np.zeros((max(len(rows), 1), 4 + self.n), dtype=np.int32)
        self._host_call(self._L.fpx_epaxos_preaccept_sets, rows.ctypes.data, len(rows), oc.ctypes.data, out.ctypes.data)
        return out[:len(rows)]

    # -- wire codec: ReplicaInbound bytes -> handler rows (include/fpx.h, fpx_epaxos_wire_*)
    def wire_decode(self, buf, offsets, value_id_base=0):
        """buf: the messages back to back, offsets[m+1] -> (kind[m], rows[m, 12+n], values[m, 2]): kind = the
        ReplicaInbound member's field number, rows {inst_replica, inst_number, b_ord, b_rep, replica_index, vb_ord,
        vb_rep, status, value_id, seq, flags, overflow, deps[n]}, values = the CommandOrNoop's {off, len} in buf."""
        buf = np.ascontiguousarray(buf, dtype=np.uint8)
        offsets = np.ascontiguousarray(offsets, dtype=np.int32)
        m = len(offsets) - 1
        kind = np.zeros(max(m, 1), dtype=np.int32)
        rows = np.zeros((max(m, 1), WIRE_COLS + self.n), dtype=np.int32)
        values = np.zeros((max(m, 1), 2), dtype=np.int32)
        self._host_call(self._L.fpx_epaxos_wire_decode, buf.ctypes.data if len(buf) else None, offsets.ctypes.data, m,
                        value_id_base, kind.ctypes.data, rows.ctypes.data, values.ctypes.data)
        return kind[:m], rows[:m], values[:m]

    def wire_pack(self, call, kind, rows, first=0, count=None, local_deps=None):
        """Decoded rows [first, first+count) -> the input rows of handler call `call` (CALL_*); local_deps [count, n]
        fills a preaccept row's local columns (zeros if None)."""
        kind = np.ascontiguousarray(kind, dtype=np.int32)
        rows = np.ascontiguousarray(rows, dtype=np.int32).reshape(-1, WIRE_COLS + self.n)
        count = len(rows) - first if count is None else count
        out = np.zeros((max(count, 1), wire_pack_width(call, self.n)), dtype=np.int32)
        ld = None if local_deps is None else np.ascontiguousarray(local_deps, dtype=np.int32).reshape(-1, self.n)
        self._host_call(self._L.fpx_epaxos_wire_pack, call, kind.ctypes.data, rows.ctypes.data, first, count,
                        None if ld is None else ld.ctypes.data, out.ctypes.data)
        return out[:count]

    def wire_encode(self, call, in_rows, out_rows=None, arena=None, value_offsets=None):
        """One canonical ReplicaInbound per record of handler call `call` (its input rows and its replies / events /
        ballots) -> (bytes, offsets[m+1]); a record with nothing to send is a zero-length message.  value_id v is
        arena[value_offsets[v] .. value_offsets[v+1]); the value-less Commit / Accept records read the cmdLog."""
        w_in = {CALL_LEAD: 8 + self.n, CALL_PREACCEPT: 6 + 2 * self.n, CALL_ACCEPT: 6 + self.n,
                CALL_PREACCEPTOK: 6 + self.n, CALL_ACCEPTOK: 6, CALL_PREPARE_PHASE: 2, CALL_PREPARE: 4,
                CALL_SLOW_PATH_TIMER: 4}.get(call, 1)
        in_rows = np.ascontiguousarray(in_rows, dtype=np.int32).reshape(-1, w_in)
        m = len(in_rows)
        out_rows = None if out_rows is None else np.ascontiguousarray(out_rows, dtype=np.int32).reshape(m, -1)
        arena = np.zeros(0, dtype=np.uint8) if arena is None else np.ascontiguousarray(arena, dtype=np.uint8)
        value_offsets = np.zeros(1, dtype=np.int32) if value_offsets is None else \
            np.ascontiguousarray(value_offsets, dtype=np.int32)
        vmax = int(np.diff(value_offsets).max()) if len(value_offsets) > 1 else 2
        cap = m * (128 + 14 * self.n + max(vmax, 2)) + 16
        out = np.zeros(cap, dtype=np.uint8)
        offs = np.zeros(m + 1, dtype=np.int32)
        self._host_call(self._L.fpx_epaxos_wire_encode, call, in_rows.ctypes.data,
                        None if out_rows is None else out_rows.ctypes.data, m, arena.ctypes.data if len(arena) else None,
                        value_offsets.ctypes.data, len(value_offsets) - 1, out.ctypes.data, cap, offs.ctypes.data)
        return out[:offs[m]].copy(), offs

    def wire_encode_dev(self, call, d_in, d_out_rows, m, d_arena, d_value_offsets, num_values, d_out, out_capacity,
                        d_offsets):
        self._check(self._L.fpx_epaxos_wire_encode_dev(self.h, call, d_in, d_out_rows, m, d_arena, d_value_offsets,
                                                       num_values, d_out, out_capacity, d_offsets))

    def wire_decode_dev(self, d_bytes, d_offsets, m, value_id_base, d_kind, d_rows, d_values):
        """device pointers, asynchronous on self.stream: a message that fails refuses like a handler batch (sync())"""
        self._check(self._L.fpx_epaxos_wire_decode_dev(self.h, d_bytes, d_offsets, m, value_id_base, d_kind, d_rows,
                                                       d_values))

    def wire_pack_dev(self, call, d_kind, d_rows, first, count, d_local_deps, d_out):
        self._check(self._L.fpx_epaxos_wire_pack_dev(self.h, call, d_kind, d_rows, first, count, d_local_deps, d_out))

    def entry(self, rep, num):
        out = np.zeros(7 + self.n, dtype=np.int32)
        lk = C.c_int32(0)
        lb = np.zeros(2, dtype=np.int32)
        self._check(self._L.fpx_epaxos_entry(self.h, rep, num, out.ctypes.data, C.byref(lk), lb.ctypes.data))
        return out, lk.value, lb

    # -- test aids (not part of include/fpx.h)
    def set_counters(self, tag=None, seq_base=None):
        """Start the batch tag and the response stamp numbering anywhere in 1 .. 2**32 - 2 (None: unchanged)."""
        cur = self.counters()
        self._check(self._L.fpx_debug_epaxos_set_counters(self.h, cur["tag"] if tag is None else tag,
                                                          cur["seq_base"] if seq_base is None else seq_base))

    def counters(self):
        """{'tag': next batch tag, 'seq_base': next response stamp}"""
        out = np.zeros(2, dtype=np.uint32)
        self._check(self._L.fpx_debug_epaxos_get_counters(self.h, out.ctypes.data))
        return {"tag": int(out[0]), "seq_base": int(out[1])}


def depset_union(watermarks, value_lists, group_off, device=0):
    """Batched IntPrefixSet union on the GPU.  watermarks[j], value_lists[j] (iterable of
    ints > watermark); group q unions sets group_off[q]..group_off[q+1].  Returns a list of
    (watermark, sorted values)."""
    L = _lib.lib()
    wm = np.ascontiguousarray(watermarks, dtype=np.int32)
    off = np.zeros(len(wm) + 1, dtype=np.int32)
    off[1:] = np.cumsum([len(v) for v in value_lists])
    vals = np.ascontiguousarray([x for v in value_lists for x in v], dtype=np.int32) if off[-1] else np.zeros(1, np.int32)
    goff = np.ascontiguousarray(group_off, dtype=np.int32)
    ng = len(goff) - 1
    ow, on = np.zeros(max(ng, 1), np.int32), np.zeros(max(ng, 1), np.int32)
    ov = np.zeros(max(int(off[-1]), 1), np.int32)
    st = L.fpx_depset_union(device, wm.ctypes.data, off.ctypes.data, vals.ctypes.data, len(wm), goff.ctypes.data, ng,
                            ow.ctypes.data, on.ctypes.data, ov.ctypes.data)
    if st != 0:
        raise FpxError(st)
    res = []
    for q in range(ng):
        o = off[goff[q]]
        res.append((int(ow[q]), ov[o:o + on[q]].tolist()))
    return res


def depset_union_dense_dev(d_in, n_groups, sets_per_group, n_replicas, d_out, stream=None, device=0):
    """Dense batched union on device pointers: out[q][k] = max_r in[q][r][k] (asynchronous)."""
    L = _lib.lib()
    st = L.fpx_depset_union_dense_dev(device, d_in, n_groups, sets_per_group, n_replicas, d_out, stream)
    if st != 0:
        raise FpxError(st)


# --------------------------------------------------------------------------- execution side (SURVEY 8(f) rank 4)
class ConflictIndex(_Handle):
    """KeyValueStore's top-1 conflict index on the GPU (include/fpx.h, fpx_conflict_index_*)."""
    QUERY_THEN_PUT, PUT, QUERY = 0, 1, 2

    def __init__(self, num_leaders, key_capacity=1 << 16, max_commands=1 << 16, max_keys=1 << 17, device=0):
        self.n = num_leaders
        super().__init__("fpx_conflict_index_create", "fpx_conflict_index_destroy", num_leaders, key_capacity,
                         max_commands, max_keys, device)

    def put_snapshot(self, leader, id_):
        self._check(self._L.fpx_conflict_index_put_snapshot(self.h, leader, id_))

    def batch(self, leader, id_, is_set, key_lists, mode=0):
        """Commands in delivery order; key_lists[i] = the keys of command i.  Returns deps [n_cmd, num_leaders]
        (None for mode PUT)."""
        n = len(leader)
        leader = np.ascontiguousarray(leader, dtype=np.int32); id_ = np.ascontiguousarray(id_, dtype=np.int32)
        is_set = np.ascontiguousarray(is_set, dtype=np.uint8)
        off = np.zeros(n + 1, dtype=np.int32)
        off[1:] = np.cumsum([len(k) for k in key_lists])
        keys = np.ascontiguousarray(np.concatenate([np.asarray(k, dtype=np.int32) for k in key_lists])
                                    if off[-1] else np.zeros(0, dtype=np.int32), dtype=np.int32)
        out = np.zeros((max(n, 1), self.n), dtype=np.int32)
        self._host_call(self._L.fpx_conflict_index_batch, leader.ctypes.data, id_.ctypes.data, is_set.ctypes.data,
                        off.ctypes.data, keys.ctypes.data if len(keys) else None, n, mode, out.ctypes.data)
        return None if mode == self.PUT else out[:n]


class DependencyGraph(_Handle):
    """TarjanDependencyGraph on the GPU (include/fpx.h, fpx_depgraph_*): int keys in [0, key_capacity)."""

    def __init__(self, key_capacity=1 << 12, dep_pool_capacity=1 << 16, max_batch=1 << 12, device=0):
        self.cap = key_capacity
        super().__init__("fpx_depgraph_create", "fpx_depgraph_destroy", key_capacity, dep_pool_capacity, max_batch,
                         device)

    def commit(self, keys, seqs, dep_lists):
        n = len(keys)
        keys = np.ascontiguousarray(keys, dtype=np.int32); seqs = np.ascontiguousarray(seqs, dtype=np.int32)
        off = np.zeros(n + 1, dtype=np.int32)
        off[1:] = np.cumsum([len(d) for d in dep_lists])
        deps = np.ascontiguousarray(np.concatenate([np.asarray(d, dtype=np.int32) for d in dep_lists])
                                    if off[-1] else np.zeros(0, dtype=np.int32), dtype=np.int32)
        self._host_call(self._L.fpx_depgraph_commit, keys.ctypes.data, seqs.ctypes.data, off.ctypes.data,
                        deps.ctypes.data if len(deps) else None, n)

    def update_executed(self, keys):
        keys = np.ascontiguousarray(keys, dtype=np.int32)
        self._host_call(self._L.fpx_depgraph_update_executed, keys.ctypes.data, len(keys))

    def execute_by_component(self):
        """(components in dependency order, each a list of keys sorted by (seq, key); sorted blockers)."""
        out = np.zeros(self.cap, dtype=np.int32); head = np.zeros(self.cap, dtype=np.uint8)
        bl = np.zeros(self.cap, dtype=np.uint8)
        n = C.c_int32(0)
        self._check(self._L.fpx_depgraph_execute(self.h, out.ctypes.data, head.ctypes.data, C.byref(n), bl.ctypes.data))
        comps = []
        for p in range(n.value):
            if head[p]:
                comps.append([])
            comps[-1].append(int(out[p]))
        return comps, np.nonzero(bl)[0].tolist()


class EpaxosGraph(_Handle):
    """TarjanDependencyGraph over EPaxos instances with dense InstancePrefixSet dependencies on the GPU
    (include/fpx.h, fpx_epaxos_graph_*).  Commit rows are fpx_epaxos_commit's: {inst_replica, inst_number,
    value_id, seq, deps[n]}; deps[inst_replica] > inst_number is the instance's own hole, not a dependency."""

    def __init__(self, n_replicas, instances_per_replica, max_batch=1 << 16, device=0):
        self.n, self.cap = n_replicas, instances_per_replica
        super().__init__("fpx_epaxos_graph_create", "fpx_epaxos_graph_destroy", n_replicas, instances_per_replica,
                         max_batch, device)

    def commit(self, rows):
        rows = np.ascontiguousarray(rows, dtype=np.int32).reshape(-1, 4 + self.n)
        self._host_call(self._L.fpx_epaxos_graph_commit, rows.ctypes.data, len(rows))

    @property
    def stream(self):
        return self._L.fpx_epaxos_graph_stream(self.h)

    def commit_dev(self, d_in, n):
        """the same rows in device memory, asynchronous on self.stream; errors collected by sync()"""
        self._check(self._L.fpx_epaxos_graph_commit_dev(self.h, d_in, n))

    def sync(self):
        self._host_call(self._L.fpx_epaxos_graph_sync)

    def update_executed(self, watermark):
        """updateExecuted of every instance (c, j < watermark[c])"""
        wm = np.ascontiguousarray(watermark, dtype=np.int32)
        self._check(self._L.fpx_epaxos_graph_update_executed(self.h, wm.ctypes.data))

    def execute_raw(self):
        """(rows [m, 2] of {replica, number}, component heads [m], blockers [n, cap] as 0/1)"""
        nv = self.n * self.cap
        out = np.zeros((nv, 2), dtype=np.int32); head = np.zeros(nv, dtype=np.uint8)
        bl = np.zeros((self.n, self.cap), dtype=np.uint8)
        m = C.c_int32(0)
        self._check(self._L.fpx_epaxos_graph_execute(self.h, out.ctypes.data, head.ctypes.data, C.byref(m),
                                                     bl.ctypes.data))
        return out[:m.value], head[:m.value], bl

    def execute_by_component(self):
        """(components in dependency order, each a list of (replica, number) sorted by (seq, replica, number);
        sorted blockers as (replica, number))"""
        out, head, bl = self.execute_raw()
        comps = []
        for p in range(len(out)):
            if head[p]:
                comps.append([])
            comps[-1].append((int(out[p, 0]), int(out[p, 1])))
        return comps, [(int(c), int(j)) for c, j in zip(*np.nonzero(bl))]

    def last_kernel_ms(self):
        return float(self._L.fpx_epaxos_graph_last_kernel_ms(self.h))
