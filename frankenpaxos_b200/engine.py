"""Thin Python handle over the C ABI (include/fpx.h).  Arrays in, arrays out.

Record dtypes mirror the protobuf messages of the reference's hot path
(shared/src/main/scala/frankenpaxos/multipaxos/MultiPaxos.proto:273-290).
"""
import ctypes as C

import numpy as np

from . import _lib

P2A = np.dtype([("slot", "<i4"), ("round", "<i4"), ("value_id", "<i4"), ("dst", "<i4")])
P2B = np.dtype([("group", "<i4"), ("acceptor", "<i4"), ("slot", "<i4"), ("round", "<i4")])
CHOSEN = np.dtype([("slot", "<i4"), ("value_id", "<i4")])
NACK = np.dtype([("leader", "<i4"), ("round", "<i4")])
# S/mencius Phase2aNoopRange / Phase2bNoopRange / ChosenNoopRange, S/vanillamencius Skip (include/fpx.h)
P2A_RANGE = np.dtype([("slot_start", "<i4"), ("slot_end", "<i4"), ("round", "<i4"), ("dst", "<i4")])
P2B_RANGE = np.dtype([("dst", "<i4"), ("slot_start", "<i4"), ("slot_end", "<i4"), ("round", "<i4")])
CHOSEN_RANGE = np.dtype([("slot_start", "<i4"), ("slot_end", "<i4")])
VM_SKIP = np.dtype([("server", "<i4"), ("slot_start", "<i4"), ("slot_stop", "<i4"), ("own", "<i4")])
# fpx_mencius_chosen: one message of the Mencius replica's mixed Chosen / ChosenNoopRange stream
MENCIUS_CHOSEN = np.dtype([("slot_start", "<i4"), ("slot_end", "<i4"), ("value_id", "<i4"), ("reserved", "<i4")])
VALUE_NOOP = -(1 << 31)
WIRE_REC = np.dtype([("a", "<i4"), ("b", "<i4"), ("c", "<i4"), ("d", "<i4")])
# fpx_read_request: ReadRequest / SequentialReadRequest {slot}; EventualReadRequest: slot = -1
READ_REQUEST = np.dtype([("slot", "<i4"), ("handle", "<i4")])
WIRE_PROXYLEADER_INBOUND, WIRE_ACCEPTOR_INBOUND = 0, 1
WIRE_MENCIUS_PROXYLEADER_INBOUND, WIRE_MENCIUS_ACCEPTOR_INBOUND = 2, 3
# ServerInbound members (S/vanillamencius/VanillaMencius.proto:227-241): Engine.wire_decode_vm_server_inbound's kinds
VM_WIRE_CLIENT_REQUEST, VM_WIRE_PHASE2A, VM_WIRE_PHASE2B, VM_WIRE_SKIP, VM_WIRE_CHOSEN, VM_WIRE_PHASE2_NACK = 1, 4, 5, 6, 7, 9

MULTIPAXOS, MENCIUS, VANILLA_MENCIUS = 0, 1, 2
# reply kinds of Engine.vm_phase2a (include/fpx.h FPX_VM_REPLY_*)
VM_REPLY_PHASE2B, VM_REPLY_NACK, VM_REPLY_CHOSEN, VM_REPLY_CHOSEN_RETIRED, VM_REPLY_CHOSEN_REVOCATION = 0, 1, 2, 3, 4
# Engine.vm_entries kinds, and the value id the engine reserves for raised entries (FPX_VALUE_RAISED)
VM_ENTRY_NONE, VM_ENTRY_VOTELESS, VM_ENTRY_PENDING, VM_ENTRY_CHOSEN = 0, 1, 2, 3
VALUE_RAISED = -(1 << 31) + 1

OK = 0
ERR_INVALID_ARG, ERR_CONFIG, ERR_CUDA, ERR_UNKNOWN_SLOT_ROUND, ERR_BAD_ACCEPTOR = -1, -2, -3, -4, -5
ERR_SLOT_RANGE, ERR_ROUND_RANGE, ERR_OVERFLOW_FULL, ERR_CONFLICT, ERR_NO_DEVICE, ERR_UNSUPPORTED = \
    -6, -7, -8, -9, -10, -11


class FpxError(RuntimeError):
    """A negative fpx_status: the reference's logger.fatal / require at `index`."""

    def __init__(self, status, index=-1, detail=""):
        self.status, self.index = status, index
        msg = _lib.lib().fpx_strerror(status).decode()
        super().__init__(f"fpx status {status} ({msg}) at record {index}{(': ' + detail) if detail else ''}")


class _Handle:
    """One handle of the C ABI: `create(&h, *args)` in the constructor (FpxError if it fails), `destroy(h)` on
    close(), at the end of a `with` block, or when the object is collected."""

    def __init__(self, create, destroy, *args):
        self._L = _lib.lib()
        self._destroy = getattr(self._L, destroy)
        self.h = C.c_void_p()
        st = getattr(self._L, create)(C.byref(self.h), *args)
        if st != OK:
            self.h = None
            raise FpxError(st)

    def close(self):
        if getattr(self, "h", None):
            self._destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def _check(self, st, idx=-1):
        if st != OK:
            raise FpxError(st, idx)

    def _host_call(self, fn, *args):
        """fn(h, *args, &err_index), a host-pointer form: FpxError at the record it reports."""
        err = C.c_int64(-1)
        self._check(fn(self.h, *args, C.byref(err)), err.value)


def _varint_fields(body):
    """{field number: int32 value} of the varint fields of a protobuf message body (the last of each wins)."""
    out, p = {}, 0
    def varint():
        nonlocal p
        v, shift = 0, 0
        while p < len(body):
            c = body[p]; p += 1
            v |= (c & 0x7f) << shift; shift += 7
            if not c & 0x80:
                return v
        raise ValueError("truncated varint")
    try:
        while p < len(body):
            tag = varint()
            wt = tag & 7
            if wt == 0:
                v = varint() & 0xffffffff
                out[tag >> 3] = v - (1 << 32) if v >> 31 else v
            elif wt == 2:
                p += varint()
            elif wt in (1, 5):
                p += 8 if wt == 1 else 4
            else:
                break
    except ValueError:
        pass
    return out


def dst(group, acceptor):
    """fpx_p2a.dst encoding."""
    return (np.asarray(group, dtype=np.int32) << 16) | np.asarray(acceptor, dtype=np.int32)


class Engine(_Handle):
    """One GPU-resident {acceptors, proxy leader, replica log} for one config."""

    def __init__(self, f, num_acceptor_groups, acceptors_per_group, flexible=False, num_leaders=None,
                 num_replicas=None, slot_capacity=1 << 20, overflow_capacity=1 << 14, max_batch=1 << 20,
                 device=0, shard_index=0, shard_count=1, protocol=MULTIPAXOS, num_leader_groups=0):
        cfg = _lib.Config()
        cfg.struct_size = C.sizeof(_lib.Config)
        cfg.protocol = protocol
        cfg.f = f
        cfg.num_acceptor_groups = num_acceptor_groups
        cfg.acceptors_per_group = acceptors_per_group
        cfg.flexible = int(bool(flexible))
        cfg.num_leaders = f + 1 if num_leaders is None else num_leaders
        cfg.num_replicas = f + 1 if num_replicas is None else num_replicas
        cfg.slot_capacity = slot_capacity
        cfg.overflow_capacity = overflow_capacity
        cfg.max_batch = max_batch
        cfg.device = device
        cfg.shard_index, cfg.shard_count = shard_index, shard_count
        cfg.num_leader_groups = num_leader_groups
        self.cfg = cfg
        super().__init__("fpx_create", "fpx_destroy", C.byref(cfg))

    # -- life cycle
    def reset(self):
        self._check(self._L.fpx_reset(self.h))

    def retire_below(self, slot):
        """Slide the live window: slots below `slot` (all executed) are recycled for the slots slot_capacity ahead.
        Secondary (slot, round) keys and Mencius noop-range keys of retired slots leave their tables, so
        leader changes and lagging leader groups do not fill them up.  All three protocols; with vanilla
        Mencius a Phase2a for a retired slot is answered with reply kind VM_REPLY_CHOSEN_RETIRED."""
        self._check(self._L.fpx_retire_below(self.h, slot))

    def _check(self, st, idx=-1):
        if st != OK:
            detail = self._L.fpx_last_error(self.h).decode() if st == ERR_CUDA else ""
            raise FpxError(st, idx, detail)

    @property
    def stream(self):
        return self._L.fpx_stream(self.h)

    @property
    def launch_count(self):
        return self._L.fpx_launch_count(self.h)

    # -- the exchange of a sharded log (include/fpx.h, fpx_exchange_*)
    def exchange_export(self):
        """IPC handle (bytes) of this engine's frontier table."""
        buf = C.create_string_buffer(64)
        self._check(self._L.fpx_exchange_export(self.h, buf))
        return buf.raw

    def exchange_attach(self, shard, handle):
        """Open shard `shard`'s table (exported by another process) so that this engine's watermark
        publications are also stored there over NVLink."""
        self._check(self._L.fpx_exchange_attach(self.h, shard, C.c_char_p(bytes(handle))))

    def exchange_attach_local(self, shard, peer):
        self._check(self._L.fpx_exchange_attach_local(self.h, shard, peer.h))

    @property
    def exchange_epoch(self):
        return self._L.fpx_exchange_epoch(self.h)

    def global_watermark(self, epoch=None, timeout_ms=5000):
        """(global executable prefix, every shard's frontier) as of publication `epoch` of every shard
        (default: this engine's own latest publication)."""
        n = self.cfg.shard_count
        fr = np.empty(n, dtype=np.int32)
        out = C.c_int32(0)
        ep = self.exchange_epoch if epoch is None else epoch
        self._check(self._L.fpx_global_watermark(self.h, ep, timeout_ms, C.byref(out), fr.ctypes.data))
        return out.value, fr

    # -- test / profiling aids (not part of include/fpx.h)
    def set_tally_path(self, exact):
        """exact=True: every tally launch evaluates each vote (no row sweep)."""
        self._check(self._L.fpx_debug_set_tally_path(self.h, 2 if exact else 0))

    def set_acceptor_segments(self, segments):
        """Cut every acceptor launch into `segments` pipelined segments (0: automatic, from the L2 size)."""
        self._check(self._L.fpx_debug_set_acceptor_segments(self.h, segments))

    def set_tally_max_sub(self, votes):
        """Cut every tally call into launches of at most `votes` votes (0: the default, 10,485,760)."""
        self._check(self._L.fpx_debug_set_tally_max_sub(self.h, votes))

    COUNTERS = ("seq_base", "rseq_base", "rng_seq_base", "vm_tag")

    def set_counters(self, **values):
        """Start the host's 32-bit counters (COUNTERS; unnamed ones keep their value) anywhere in 1 .. 2**32 - 2,
        e.g. just below their wrap."""
        unknown = set(values) - set(self.COUNTERS)
        if unknown:
            raise ValueError(f"unknown counters {sorted(unknown)}")
        cur = self.counters()
        self._check(self._L.fpx_debug_set_counters(self.h, *(values.get(k, cur[k]) for k in self.COUNTERS)))

    def counters(self):
        """{name: value} of the host's 32-bit counters."""
        out = np.zeros(4, dtype=np.uint32)
        self._check(self._L.fpx_debug_get_counters(self.h, out.ctypes.data))
        return dict(zip(self.COUNTERS, (int(x) for x in out)))

    def _last_paths(self):
        out = np.zeros(2, dtype=np.int32)
        self._check(self._L.fpx_debug_last_paths(self.h, out.ctypes.data))
        return out

    @property
    def last_tally_path(self):
        """'sweep' / 'exact': what the last proxyleader_phase2b launch did."""
        return {1: "sweep", 2: "exact"}.get(int(self._last_paths()[0]), "none")

    @property
    def last_arm_path(self):
        """'cas' / 'fresh': what the last proxyleader_arm launch did (one CAS per record, or a batch certified as
        fresh keys in strict slot order, armed by plain row stores)."""
        return {1: "cas", 2: "fresh"}.get(int(self._last_paths()[1]), "none")

    # -- host-pointer calls (numpy in / numpy out)
    def proxyleader_arm(self, p2a):
        p2a = np.ascontiguousarray(p2a, dtype=P2A)
        self._host_call(self._L.fpx_proxyleader_arm, p2a.ctypes.data, len(p2a))

    def acceptor_phase2a(self, p2a):
        p2a = np.ascontiguousarray(p2a, dtype=P2A)
        n = len(p2a)
        out = np.empty(max(n, 1), dtype=P2B)
        nack = np.empty(max(n, 1), dtype=NACK)
        n1, n2 = C.c_int32(0), C.c_int32(0)
        self._host_call(self._L.fpx_acceptor_phase2a, p2a.ctypes.data, n, out.ctypes.data, C.byref(n1),
                        nack.ctypes.data, C.byref(n2))
        return out[:n1.value], nack[:n2.value]

    def proxyleader_phase2b(self, p2b):
        p2b = np.ascontiguousarray(p2b, dtype=P2B)
        n = len(p2b)
        out = np.empty(max(n, 1), dtype=CHOSEN)
        n1 = C.c_int32(0)
        self._host_call(self._L.fpx_proxyleader_phase2b, p2b.ctypes.data, n, out.ctypes.data, C.byref(n1))
        return out[:n1.value]

    def replica_chosen(self, chosen):
        chosen = np.ascontiguousarray(chosen, dtype=CHOSEN)
        self._host_call(self._L.fpx_replica_chosen, chosen.ctypes.data, len(chosen))

    def chosen_watermark(self):
        out = C.c_int32(0)
        self._check(self._L.fpx_chosen_watermark(self.h, C.byref(out)))
        return out.value

    def quorum_eval(self, which, masks):
        masks = np.ascontiguousarray(masks, dtype=np.uint32)
        out = np.empty(max(len(masks), 1), dtype=np.uint8)
        self._check(self._L.fpx_quorum_eval(self.h, which, masks.ctypes.data, len(masks), out.ctypes.data))
        return out[:len(masks)]

    def snapshot_acceptor(self, group, acceptor, first_slot=0, n_slots=0):
        vr = np.empty(max(n_slots, 1), dtype=np.int32)
        vv = np.empty(max(n_slots, 1), dtype=np.int32)
        r, m = C.c_int32(0), C.c_int32(0)
        self._check(self._L.fpx_snapshot_acceptor(self.h, group, acceptor, C.byref(r), C.byref(m), first_slot,
                                                  n_slots, vr.ctypes.data, vv.ctypes.data))
        return r.value, m.value, vr[:n_slots], vv[:n_slots]

    def snapshot_log(self, first_slot, n_slots):
        v = np.empty(max(n_slots, 1), dtype=np.int32)
        self._check(self._L.fpx_snapshot_log(self.h, first_slot, n_slots, v.ctypes.data))
        return v[:n_slots]

    # -- Phase 1 reads (SURVEY 8(f) rank 2)
    def acceptor_phase1a(self, group, acceptor, round_, chosen_watermark=0):
        """Acceptor.handlePhase1a: returns ('nack', acceptor_round) or ('phase1b', info) with info =
        [(slot, voteRound, voteValue)] from chosen_watermark on, ascending slots."""
        nack = C.c_int32(0)
        self._check(self._L.fpx_acceptor_phase1a(self.h, group, acceptor, round_, C.byref(nack)))
        if nack.value >= 0:
            return "nack", nack.value
        r, m, vr, vv = self.snapshot_acceptor(group, acceptor, chosen_watermark, max(0, self.snapshot_acceptor(group, acceptor)[1] + 1 - chosen_watermark))
        keep = np.nonzero(vr >= 0)[0]
        return "phase1b", [(int(chosen_watermark + i), int(vr[i]), int(vv[i])) for i in keep]

    def leader_safe_values(self, responders, first_slot, n_slots):
        vr = np.empty(max(n_slots, 1), dtype=np.int32)
        vv = np.empty(max(n_slots, 1), dtype=np.int32)
        mx = C.c_int32(-1)
        self._check(self._L.fpx_leader_safe_values(self.h, responders, first_slot, n_slots, vr.ctypes.data,
                                                   vv.ctypes.data, C.byref(mx)))
        return vr[:n_slots], vv[:n_slots], mx.value

    # -- vanilla Mencius (protocol=VANILLA_MENCIUS)
    def vm_client_request(self, p2a):
        p2a = np.ascontiguousarray(p2a, dtype=P2A)
        self._host_call(self._L.fpx_vm_client_request, p2a.ctypes.data, len(p2a))

    def vm_phase2a(self, p2a):
        """dense replies {group = kind (0 Phase2b, 1 Phase2Nack, 2 Chosen, 3 Chosen of a retired slot whose value
        is the shared log's executed entry), acceptor = server, slot, round|value (0 for kind 3)}"""
        p2a = np.ascontiguousarray(p2a, dtype=P2A)
        out = np.empty(max(len(p2a), 1), dtype=P2B)
        self._host_call(self._L.fpx_vm_phase2a, p2a.ctypes.data, len(p2a), out.ctypes.data)
        return out[:len(p2a)]

    def vm_learn_chosen(self, recs):
        recs = np.ascontiguousarray(recs, dtype=P2B)
        self._host_call(self._L.fpx_vm_learn_chosen, recs.ctypes.data, len(recs))

    def vm_choose(self, recs):
        """Server.choose(slot, value, isRevocation) for received Chosen: {group = is_revocation, acceptor = server,
        slot, round = value_id}."""
        recs = np.ascontiguousarray(recs, dtype=P2B)
        self._host_call(self._L.fpx_vm_choose, recs.ctypes.data, len(recs))

    def vm_phase1a_wire(self, data, kind, recs, next_slot, arena=b"", value_offsets=(0,), out_capacity=None):
        """Server.handlePhase1a per decoded ServerInbound record (recs.a = the receiving server).  next_slot (int32
        per server) is updated in place.  Returns (list of reply bytes, one per record, skip records).  The default
        out_capacity is the largest the replies can take: per Phase1a its head and one info per walked slot with the
        arena's longest value."""
        data = bytes(data)
        kind = np.ascontiguousarray(kind, dtype=np.int32)
        recs = np.ascontiguousarray(recs, dtype=WIRE_REC)
        vo = np.ascontiguousarray(value_offsets, dtype=np.int32)
        n = len(kind)
        if out_capacity is None:
            vmax = max([2] + [int(x) for x in np.diff(vo)])
            out_capacity = 64
            for i in np.nonzero(kind == 2)[0]:
                r = recs[i]
                f = _varint_fields(data[max(int(r["c"]), 0): max(int(r["c"]), 0) + max(int(r["d"]), 0)])
                start, stop, servers = f.get(2, 0), f.get(3, 0), self.cfg.acceptors_per_group
                walked = (stop - start + servers - 1) // servers if 0 <= start < stop else 0
                out_capacity += 64 + walked * (48 + vmax)
        out = np.empty(max(out_capacity, 1), dtype=np.uint8)
        offs = np.zeros(n + 1, dtype=np.int32)
        skips = np.zeros(max(n, 1), dtype=VM_SKIP)
        a = np.frombuffer(bytes(arena) + b"\0", dtype=np.uint8)
        b = np.frombuffer(data + b"\0", dtype=np.uint8)
        assert next_slot.dtype == np.int32 and next_slot.flags.c_contiguous
        self._host_call(self._L.fpx_vm_phase1a_wire, b.ctypes.data, len(data), kind.ctypes.data, recs.ctypes.data, n,
                        a.ctypes.data, vo.ctypes.data, len(vo) - 1, next_slot.ctypes.data, out.ctypes.data,
                        out_capacity, offs.ctypes.data, skips.ctypes.data)
        return [out[offs[i]:offs[i + 1]].tobytes() for i in range(n)], skips[:n]

    def vm_phase1a_wire_dev(self, d_bytes, n_bytes, d_kind, d_in, n, d_arena, d_value_offsets, num_values, d_next_slot,
                            d_out, out_capacity, d_offsets, d_skips):
        self._check(self._L.fpx_vm_phase1a_wire_dev(self.h, d_bytes, n_bytes, d_kind, d_in, n, d_arena, d_value_offsets,
                                                    num_values, d_next_slot, d_out, out_capacity, d_offsets, d_skips))

    def vm_choose_dev(self, d_in, n):
        self._check(self._L.fpx_vm_choose_dev(self.h, d_in, n))

    def vm_entries(self, server, first_slot, n_slots):
        """server's entries at [first_slot, first_slot + n_slots): int32 [n_slots, 5] {kind (VM_ENTRY_*), round,
        voteRound, value, isRevocation}."""
        out = np.zeros((max(n_slots, 1), 5), dtype=np.int32)
        self._check(self._L.fpx_vm_entries(self.h, server, first_slot, n_slots, out.ctypes.data))
        return out[:n_slots]

    def vm_skip(self, recs):
        """Server.advanceWithSkips' log fill (own=1) / Server.handleSkip (own=0)."""
        recs = np.ascontiguousarray(recs, dtype=VM_SKIP)
        self._host_call(self._L.fpx_vm_skip, recs.ctypes.data, len(recs))

    # -- S/mencius Phase2aNoopRange path
    def mencius_arm_range(self, recs):
        recs = np.ascontiguousarray(recs, dtype=P2A_RANGE)
        self._host_call(self._L.fpx_mencius_arm_range, recs.ctypes.data, len(recs))

    def mencius_acceptor_noop_range(self, recs):
        recs = np.ascontiguousarray(recs, dtype=P2A_RANGE)
        n = len(recs)
        out = np.zeros(max(n, 1), dtype=P2B_RANGE)
        nack = np.zeros(max(n, 1), dtype=NACK)
        n1, n2 = C.c_int32(0), C.c_int32(0)
        self._host_call(self._L.fpx_mencius_acceptor_noop_range, recs.ctypes.data, n, out.ctypes.data, C.byref(n1),
                        nack.ctypes.data, C.byref(n2))
        return out[:n1.value].copy(), nack[:n2.value].copy()

    def mencius_range_phase2b(self, recs):
        recs = np.ascontiguousarray(recs, dtype=P2B_RANGE)
        n = len(recs)
        out = np.zeros(max(n, 1), dtype=CHOSEN_RANGE)
        n1 = C.c_int32(0)
        self._host_call(self._L.fpx_mencius_range_phase2b, recs.ctypes.data, n, out.ctypes.data, C.byref(n1))
        return out[:n1.value].copy()

    def mencius_replica_chosen_range(self, recs):
        recs = np.ascontiguousarray(recs, dtype=CHOSEN_RANGE)
        self._host_call(self._L.fpx_mencius_replica_chosen_range, recs.ctypes.data, len(recs))

    def mencius_replica_inbound(self, recs):
        """A mixed Chosen / ChosenNoopRange batch (MENCIUS_CHOSEN records) in delivery order: applies the records before
        the returned split, as the reference's replica would one at a time; continue with recs[split:]."""
        recs = np.ascontiguousarray(recs, dtype=MENCIUS_CHOSEN)
        split = C.c_int32(0)
        self._host_call(self._L.fpx_mencius_replica_inbound, recs.ctypes.data, len(recs), C.byref(split))
        return split.value

    def mencius_replica_inbound_dev(self, d_in, n, d_split):
        self._check(self._L.fpx_mencius_replica_inbound_dev(self.h, d_in, n, d_split))

    RANGE_NO_HIT = 0x7f7f7f7f

    def mencius_replica_range_first(self, recs):
        """Per record: this shard's first slot of the range that is already in its log (RANGE_NO_HIT if none)."""
        recs = np.ascontiguousarray(recs, dtype=CHOSEN_RANGE)
        first = np.full(max(len(recs), 1), self.RANGE_NO_HIT, dtype=np.int32)
        self._host_call(self._L.fpx_mencius_replica_range_first, recs.ctypes.data, len(recs), first.ctypes.data)
        return first[:len(recs)]

    def mencius_replica_range_fill(self, recs, first):
        """Noop into this shard's slots of [start, min(end, first[i])): `first` = the minimum over the shards."""
        recs = np.ascontiguousarray(recs, dtype=CHOSEN_RANGE)
        first = np.ascontiguousarray(first, dtype=np.int32)
        assert len(first) == len(recs)
        self._host_call(self._L.fpx_mencius_replica_range_fill, recs.ctypes.data, len(recs), first.ctypes.data)

    # -- wire codec: protobuf bytes of a batch of messages <-> records (include/fpx.h)
    def wire_decode_inbound(self, inbound, buf, offsets):
        """buf: uint8 array with the messages back to back, offsets[n+1].  Returns (kind[n], rec[n])."""
        buf = np.ascontiguousarray(buf, dtype=np.uint8)
        offsets = np.ascontiguousarray(offsets, dtype=np.int32)
        n = len(offsets) - 1
        kind = np.zeros(max(n, 1), dtype=np.int32)
        rec = np.zeros(max(n, 1), dtype=WIRE_REC)
        self._host_call(self._L.fpx_wire_decode_inbound, inbound, buf.ctypes.data if len(buf) else None,
                        offsets.ctypes.data, n, kind.ctypes.data, rec.ctypes.data)
        return kind[:n], rec[:n]

    def _wire_encode(self, fn, recs, dtype, max_per, *extra):
        recs = np.ascontiguousarray(recs, dtype=dtype)
        n = len(recs)
        cap = max(16, n * max_per) if not extra else extra[-1]
        out = np.zeros(cap, dtype=np.uint8)
        offs = np.zeros(n + 1, dtype=np.int32)
        self._host_call(fn, recs.ctypes.data, n, *extra[:-1], out.ctypes.data, cap, offs.ctypes.data)
        return out[:offs[n]].copy(), offs

    def wire_encode_phase2b(self, recs):
        return self._wire_encode(self._L.fpx_wire_encode_phase2b, recs, P2B, 46)

    def wire_encode_nack(self, recs):
        return self._wire_encode(self._L.fpx_wire_encode_nack, recs, NACK, 13)

    def wire_encode_chosen(self, recs, arena, value_offsets):
        arena = np.ascontiguousarray(arena, dtype=np.uint8)
        value_offsets = np.ascontiguousarray(value_offsets, dtype=np.int32)
        recs = np.ascontiguousarray(recs, dtype=CHOSEN)
        lens = np.diff(value_offsets)
        ok = (recs["value_id"] >= 0) & (recs["value_id"] < len(lens))
        cap = int(24 * len(recs) + lens[recs["value_id"][ok]].sum()) + 16
        return self._wire_encode(self._L.fpx_wire_encode_chosen, recs, CHOSEN, 0, arena.ctypes.data if len(arena) else None,
                                 value_offsets.ctypes.data, len(value_offsets) - 1, cap)

    # -- Compartmentalized Mencius noop-range and replica wire codec (protocol=MENCIUS, include/fpx.h)
    def wire_decode_mencius_replica_inbound(self, buf, offsets, value_id_base=0):
        """ReplicaInbound bytes -> (kind[n], recs[n] MENCIUS_CHOSEN, values[n, 2]): row i answers message i; values[i]
        = {off, len} of a Chosen's command_batch_or_noop.  kind 0 (no member) is a row that covers no slot."""
        buf = np.ascontiguousarray(buf, dtype=np.uint8)
        offsets = np.ascontiguousarray(offsets, dtype=np.int32)
        n = len(offsets) - 1
        kind = np.zeros(max(n, 1), dtype=np.int32)
        recs = np.zeros(max(n, 1), dtype=MENCIUS_CHOSEN)
        values = np.zeros((max(n, 1), 2), dtype=np.int32)
        self._host_call(self._L.fpx_wire_decode_mencius_replica_inbound, buf.ctypes.data if len(buf) else None,
                        offsets.ctypes.data, n, value_id_base, kind.ctypes.data, recs.ctypes.data, values.ctypes.data)
        return kind[:n], recs[:n], values[:n]

    def wire_decode_mencius_replica_inbound_dev(self, d_bytes, d_offsets, n, value_id_base, d_kind, d_recs, d_values):
        self._check(self._L.fpx_wire_decode_mencius_replica_inbound_dev(self.h, d_bytes, d_offsets, n, value_id_base,
                                                                        d_kind, d_recs, d_values))

    def wire_encode_mencius_phase2b_range(self, recs):
        """fpx_mencius_acceptor_noop_range's replies -> ProxyLeaderInbound.phase2b_noop_range bytes, offsets[n+1]."""
        return self._wire_encode(self._L.fpx_wire_encode_mencius_phase2b_range, recs, P2B_RANGE, 57)

    def wire_encode_mencius_chosen_range(self, recs):
        """fpx_mencius_range_phase2b's ChosenNoopRanges -> ReplicaInbound.chosen_noop_range bytes, offsets[n+1]."""
        return self._wire_encode(self._L.fpx_wire_encode_mencius_chosen_range, recs, CHOSEN_RANGE, 24)

    def wire_encode_mencius_phase2b_range_dev(self, d_in, n, d_out, out_capacity, d_offsets):
        self._check(self._L.fpx_wire_encode_mencius_phase2b_range_dev(self.h, d_in, n, d_out, out_capacity, d_offsets))

    def wire_encode_mencius_chosen_range_dev(self, d_in, n, d_out, out_capacity, d_offsets):
        self._check(self._L.fpx_wire_encode_mencius_chosen_range_dev(self.h, d_in, n, d_out, out_capacity, d_offsets))

    # -- vanilla Mencius wire codec (protocol=VANILLA_MENCIUS): ServerInbound bytes <-> records (include/fpx.h)
    def wire_decode_vm_server_inbound(self, buf, offsets):
        """Returns (kind[n], rec[n], sender[n]): kind = the ServerInbound member's field number, sender = the
        server field of a Phase2a / Phase2b / Skip, else -1."""
        buf = np.ascontiguousarray(buf, dtype=np.uint8)
        offsets = np.ascontiguousarray(offsets, dtype=np.int32)
        n = len(offsets) - 1
        kind = np.zeros(max(n, 1), dtype=np.int32)
        rec = np.zeros(max(n, 1), dtype=WIRE_REC)
        sender = np.zeros(max(n, 1), dtype=np.int32)
        self._host_call(self._L.fpx_wire_decode_vm_server_inbound, buf.ctypes.data if len(buf) else None,
                        offsets.ctypes.data, n, kind.ctypes.data, rec.ctypes.data, sender.ctypes.data)
        return kind[:n], rec[:n], sender[:n]

    def _wire_encode_valued(self, fn, recs, dtype, value_ids, arena, value_offsets):
        """An encoder whose messages carry a CommandOrNoop: value_id v is arena[value_offsets[v] ..
        value_offsets[v+1]), VALUE_NOOP the Noop."""
        arena = np.zeros(0, dtype=np.uint8) if arena is None else np.ascontiguousarray(arena, dtype=np.uint8)
        value_offsets = np.zeros(1, dtype=np.int32) if value_offsets is None else \
            np.ascontiguousarray(value_offsets, dtype=np.int32)
        lens = np.diff(value_offsets)
        ok = (value_ids >= 0) & (value_ids < len(lens))
        cap = int(48 * len(recs) + lens[value_ids[ok]].sum()) + 16   # 48: the longest head (Phase2a)
        return self._wire_encode(fn, recs, dtype, 0, arena.ctypes.data if len(arena) else None,
                                 value_offsets.ctypes.data, len(value_offsets) - 1, cap)

    def wire_encode_vm_replies(self, replies, arena=None, value_offsets=None):
        """The dense reply stream of vm_phase2a / vm_step_dev -> (bytes, offsets[n+1]); a kind-3 reply
        (VM_REPLY_CHOSEN_RETIRED) is a zero-length message: the caller holds that slot's value."""
        replies = np.ascontiguousarray(replies, dtype=P2B)
        vids = np.where(np.isin(replies["group"], (VM_REPLY_CHOSEN, VM_REPLY_CHOSEN_REVOCATION)), replies["round"], -1)
        return self._wire_encode_valued(self._L.fpx_wire_encode_vm_replies, replies, P2B, vids, arena, value_offsets)

    def wire_encode_vm_chosen(self, recs, arena=None, value_offsets=None):
        recs = np.ascontiguousarray(recs, dtype=CHOSEN)
        return self._wire_encode_valued(self._L.fpx_wire_encode_vm_chosen, recs, CHOSEN, recs["value_id"], arena,
                                        value_offsets)

    def wire_encode_vm_phase2a(self, recs, arena=None, value_offsets=None):
        """Client-request records -> the coordinator's Phase2a (sending_server = slot mod n)."""
        recs = np.ascontiguousarray(recs, dtype=P2A)
        return self._wire_encode_valued(self._L.fpx_wire_encode_vm_phase2a, recs, P2A, recs["value_id"], arena,
                                        value_offsets)

    def wire_encode_vm_skip(self, recs):
        return self._wire_encode(self._L.fpx_wire_encode_vm_skip, recs, VM_SKIP, 46)

    def wire_decode_vm_server_inbound_dev(self, d_bytes, d_offsets, n, d_kind, d_out, d_sender):
        self._check(self._L.fpx_wire_decode_vm_server_inbound_dev(self.h, d_bytes, d_offsets, n, d_kind, d_out, d_sender))

    def wire_encode_vm_replies_dev(self, d_in, n, d_arena, d_value_offsets, num_values, d_out, out_capacity, d_offsets):
        self._check(self._L.fpx_wire_encode_vm_replies_dev(self.h, d_in, n, d_arena, d_value_offsets, num_values, d_out,
                                                           out_capacity, d_offsets))

    def wire_encode_vm_chosen_dev(self, d_in, n, d_arena, d_value_offsets, num_values, d_out, out_capacity, d_offsets):
        self._check(self._L.fpx_wire_encode_vm_chosen_dev(self.h, d_in, n, d_arena, d_value_offsets, num_values, d_out,
                                                          out_capacity, d_offsets))

    def wire_encode_vm_phase2a_dev(self, d_in, n, d_arena, d_value_offsets, num_values, d_out, out_capacity, d_offsets):
        self._check(self._L.fpx_wire_encode_vm_phase2a_dev(self.h, d_in, n, d_arena, d_value_offsets, num_values, d_out,
                                                           out_capacity, d_offsets))

    def wire_encode_vm_skip_dev(self, d_in, n, d_out, out_capacity, d_offsets):
        self._check(self._L.fpx_wire_encode_vm_skip_dev(self.h, d_in, n, d_out, out_capacity, d_offsets))

    def vm_client_request_dev(self, d_in, n):
        self._check(self._L.fpx_vm_client_request_dev(self.h, d_in, n))

    def vm_phase2a_dev(self, d_in, n, d_reply):
        self._check(self._L.fpx_vm_phase2a_dev(self.h, d_in, n, d_reply))

    def wire_decode_inbound_dev(self, inbound, d_bytes, d_offsets, n, d_kind, d_out):
        self._check(self._L.fpx_wire_decode_inbound_dev(self.h, inbound, d_bytes, d_offsets, n, d_kind, d_out))

    def wire_encode_phase2b_dev(self, d_in, n, d_out, out_capacity, d_offsets):
        self._check(self._L.fpx_wire_encode_phase2b_dev(self.h, d_in, n, d_out, out_capacity, d_offsets))

    # -- MultiPaxos replica and acceptor read-path wire codec (include/fpx.h)
    def wire_decode_replica_inbound(self, buf, offsets, value_id_base=0, handle_base=0, reads_capacity=None):
        """ReplicaInbound bytes -> (kind[n], chosen, chosen_values[k, 2], reads, read_commands[k, 2], split): records
        of the messages [0, split) only; continue with offsets[split:].  reads_capacity defaults to a bound no batch
        can exceed: a Command field takes at least 12 bytes (tag, length, command_id with its three required fields,
        command)."""
        buf = np.ascontiguousarray(buf, dtype=np.uint8)
        offsets = np.ascontiguousarray(offsets, dtype=np.int32)
        n = len(offsets) - 1
        cap = int(offsets[-1] - offsets[0]) // 12 + 1 if reads_capacity is None else reads_capacity
        kind = np.zeros(max(n, 1), dtype=np.int32)
        chosen = np.zeros(max(n, 1), dtype=CHOSEN)
        cvals = np.zeros((max(n, 1), 2), dtype=np.int32)
        reads = np.zeros(max(cap, 1), dtype=READ_REQUEST)
        rcmds = np.zeros((max(cap, 1), 2), dtype=np.int32)
        counts = np.zeros(3, dtype=np.int32)
        self._host_call(self._L.fpx_wire_decode_replica_inbound, buf.ctypes.data if len(buf) else None,
                        offsets.ctypes.data, n, value_id_base, handle_base, cap, kind.ctypes.data, chosen.ctypes.data,
                        cvals.ctypes.data, reads.ctypes.data, rcmds.ctypes.data, counts.ctypes.data)
        nc, nr, split = (int(x) for x in counts)
        return kind[:n], chosen[:nc].copy(), cvals[:nc].copy(), reads[:nr].copy(), rcmds[:nr].copy(), split

    def wire_encode_max_slot_replies(self, buf, kind, recs):
        """The acceptor's MaxSlotReply / BatchMaxSlotReply per decoded AcceptorInbound record (a = group << 16 |
        acceptor, b = maxVotedSlot) of the request batch buf -> (bytes, offsets[n+1])."""
        buf = np.ascontiguousarray(buf, dtype=np.uint8)
        kind = np.ascontiguousarray(kind, dtype=np.int32)
        recs = np.ascontiguousarray(recs, dtype=WIRE_REC)
        # a reply is at most 64 bytes of heads plus the request body's client_address
        cap = int(64 * len(recs) + np.where((kind == 3) | (kind == 4), recs["d"], 0).clip(0).sum()) + 16
        n = len(recs)
        out = np.zeros(cap, dtype=np.uint8)
        offs = np.zeros(n + 1, dtype=np.int32)
        self._host_call(self._L.fpx_wire_encode_max_slot_replies, buf.ctypes.data if len(buf) else None, len(buf),
                        kind.ctypes.data, recs.ctypes.data, n, out.ctypes.data, cap, offs.ctypes.data)
        return out[:offs[n]].copy(), offs

    def wire_decode_replica_inbound_dev(self, d_bytes, d_offsets, n, value_id_base, handle_base, reads_capacity, d_kind,
                                        d_chosen, d_chosen_values, d_reads, d_read_commands, d_counts):
        self._check(self._L.fpx_wire_decode_replica_inbound_dev(self.h, d_bytes, d_offsets, n, value_id_base, handle_base,
                                                                reads_capacity, d_kind, d_chosen, d_chosen_values,
                                                                d_reads, d_read_commands, d_counts))

    def wire_encode_max_slot_replies_dev(self, d_bytes, n_bytes, d_kind, d_in, n, d_out, out_capacity, d_offsets):
        self._check(self._L.fpx_wire_encode_max_slot_replies_dev(self.h, d_bytes, n_bytes, d_kind, d_in, n, d_out,
                                                                 out_capacity, d_offsets))

    def leader_phase1b_wire(self, round_, chosen_watermark, buf, offsets, value_id_base=0, out_capacity=None):
        """Leader.handlePhase1b over LeaderInbound bytes in delivery order -> (complete, max_slot, records P2A,
        spans[k, 2]): complete = the index of the message that completed the read quorum (-1: none yet, no records);
        record k re-proposes slot chosen_watermark + k, value_id_base + k with its vote value at spans[k] in buf, or
        VALUE_NOOP.  out_capacity defaults to the engine's slot capacity."""
        buf = np.ascontiguousarray(buf, dtype=np.uint8)
        offsets = np.ascontiguousarray(offsets, dtype=np.int32)
        n = len(offsets) - 1
        cap = self.cfg.slot_capacity if out_capacity is None else out_capacity
        out = np.zeros(max(cap, 1), dtype=P2A)
        spans = np.zeros((max(cap, 1), 2), dtype=np.int32)
        res = np.zeros(3, dtype=np.int32)
        self._host_call(self._L.fpx_leader_phase1b_wire, round_, chosen_watermark, buf.ctypes.data if len(buf) else None,
                        offsets.ctypes.data, n, value_id_base, out.ctypes.data, spans.ctypes.data, cap, res.ctypes.data)
        k = int(res[2])
        return int(res[0]), int(res[1]), out[:k].copy(), spans[:k].copy()

    def leader_phase1b_wire_dev(self, round_, chosen_watermark, d_bytes, n_bytes, d_offsets, n, value_id_base, d_out,
                                d_spans, out_capacity, d_result):
        self._check(self._L.fpx_leader_phase1b_wire_dev(self.h, round_, chosen_watermark, d_bytes, n_bytes, d_offsets, n,
                                                        value_id_base, d_out, d_spans, out_capacity, d_result))

    def acceptor_phase1a_wire(self, buf, kind, recs, arena, value_offsets):
        """Acceptor.handlePhase1a per decoded AcceptorInbound record (a = group << 16 | acceptor) of the request batch
        buf -> (bytes, offsets[n+1]): a Phase1b (votes' values from arena / value_offsets, VALUE_NOOP the Noop) or a
        Nack per Phase1a, a zero-length message for any other kind."""
        buf = np.ascontiguousarray(buf, dtype=np.uint8)
        kind = np.ascontiguousarray(kind, dtype=np.int32)
        recs = np.ascontiguousarray(recs, dtype=WIRE_REC)
        arena = np.ascontiguousarray(arena, dtype=np.uint8)
        value_offsets = np.ascontiguousarray(value_offsets, dtype=np.int32)
        n = len(recs)
        # an info is at most 32 bytes of head plus its value, one per slot up to the acceptor's maxVotedSlot
        longest = max(int(np.diff(value_offsets).max()) if len(value_offsets) > 1 else 0, 2)
        cap = 16 + 16 * n
        for i in np.nonzero(kind == 1)[0]:
            g, a = int(recs["a"][i]) >> 16, int(recs["a"][i]) & 0xffff
            if g < self.cfg.num_acceptor_groups and a < self.cfg.acceptors_per_group:
                cap += 48 + (self.snapshot_acceptor(g, a)[1] + 1) * (32 + longest)
        cap = min(cap, (1 << 31) - 1)
        out = np.zeros(cap, dtype=np.uint8)
        offs = np.zeros(n + 1, dtype=np.int32)
        self._host_call(self._L.fpx_acceptor_phase1a_wire, buf.ctypes.data if len(buf) else None, len(buf),
                        kind.ctypes.data, recs.ctypes.data, n, arena.ctypes.data if len(arena) else None,
                        value_offsets.ctypes.data, len(value_offsets) - 1, out.ctypes.data, cap, offs.ctypes.data)
        return out[:offs[n]].copy(), offs

    def acceptor_phase1a_wire_dev(self, d_bytes, n_bytes, d_kind, d_in, n, d_arena, d_value_offsets, num_values, d_out,
                                  out_capacity, d_offsets):
        self._check(self._L.fpx_acceptor_phase1a_wire_dev(self.h, d_bytes, n_bytes, d_kind, d_in, n, d_arena,
                                                          d_value_offsets, num_values, d_out, out_capacity, d_offsets))

    def wire_encode_phase2a(self, recs, buf, spans, value_id_base=0):
        """P2A records -> ProxyLeaderInbound{phase2a} bytes, offsets[n+1]: value_id v is buf[spans[v - base]], VALUE_NOOP
        the Noop (leader_phase1b_wire's output as it is)."""
        recs = np.ascontiguousarray(recs, dtype=P2A)
        buf = np.ascontiguousarray(buf, dtype=np.uint8)
        spans = np.ascontiguousarray(spans, dtype=np.int32).reshape(-1, 2)
        k = recs["value_id"].astype(np.int64) - value_id_base
        ok = (recs["value_id"] != VALUE_NOOP) & (k >= 0) & (k < len(spans))
        cap = int(32 * len(recs) + spans[k[ok], 1].clip(0).sum()) + 16   # 32: the longest head
        n = len(recs)
        out = np.zeros(cap, dtype=np.uint8)
        offs = np.zeros(n + 1, dtype=np.int32)
        self._host_call(self._L.fpx_wire_encode_phase2a, recs.ctypes.data, n, buf.ctypes.data if len(buf) else None,
                        len(buf), spans.ctypes.data, len(spans), value_id_base, out.ctypes.data, cap, offs.ctypes.data)
        return out[:offs[n]].copy(), offs

    def wire_encode_phase2a_dev(self, d_in, n, d_bytes, n_bytes, d_spans, num_spans, value_id_base, d_out, out_capacity,
                                d_offsets):
        self._check(self._L.fpx_wire_encode_phase2a_dev(self.h, d_in, n, d_bytes, n_bytes, d_spans, num_spans,
                                                        value_id_base, d_out, out_capacity, d_offsets))

    def mencius_acceptor_phase1a_wire(self, buf, kind, recs, arena, value_offsets):
        """Compartmentalized Mencius' Acceptor.handlePhase1a per decoded AcceptorInbound record (a = engine_group << 16
        | acceptor) -> (bytes, offsets[n+1]): a Phase1b (group_index = engine_group % AG, Phase2a and noop-range
        votes alike) or a Nack (member 7) per Phase1a, a zero-length message for any other kind."""
        buf = np.ascontiguousarray(buf, dtype=np.uint8)
        kind = np.ascontiguousarray(kind, dtype=np.int32)
        recs = np.ascontiguousarray(recs, dtype=WIRE_REC)
        arena = np.ascontiguousarray(arena, dtype=np.uint8)
        value_offsets = np.ascontiguousarray(value_offsets, dtype=np.int32)
        n = len(recs)
        # an info is at most 32 bytes of head plus its value, one per slot of the acceptor's residue in the live window
        longest = max(int(np.diff(value_offsets).max()) if len(value_offsets) > 1 else 0, 2)
        held = self.cfg.slot_capacity // (max(self.cfg.num_leader_groups, 1) * self.cfg.num_acceptor_groups) + 1
        cap = min(16 + 16 * n + int((kind == 1).sum()) * (48 + held * (32 + longest)), (1 << 31) - 1)
        out = np.zeros(cap, dtype=np.uint8)
        offs = np.zeros(n + 1, dtype=np.int32)
        self._host_call(self._L.fpx_mencius_acceptor_phase1a_wire, buf.ctypes.data if len(buf) else None, len(buf),
                        kind.ctypes.data, recs.ctypes.data, n, arena.ctypes.data if len(arena) else None,
                        value_offsets.ctypes.data, len(value_offsets) - 1, out.ctypes.data, cap, offs.ctypes.data)
        return out[:offs[n]].copy(), offs

    def mencius_acceptor_phase1a_wire_dev(self, d_bytes, n_bytes, d_kind, d_in, n, d_arena, d_value_offsets, num_values,
                                          d_out, out_capacity, d_offsets):
        self._check(self._L.fpx_mencius_acceptor_phase1a_wire_dev(self.h, d_bytes, n_bytes, d_kind, d_in, n, d_arena,
                                                                  d_value_offsets, num_values, d_out, out_capacity,
                                                                  d_offsets))

    def mencius_leader_phase1b_wire(self, leader_group, round_, chosen_watermark, buf, offsets, recover_slot=-1,
                                    value_id_base=0, out_capacity=None):
        """Compartmentalized Mencius' Leader.handlePhase1b of leader group leader_group over LeaderInbound bytes in
        delivery order -> (complete, max_slot, next_slot, records P2A, spans[k, 2]): record k re-proposes slot
        s0 + k * num_leader_groups (s0 the group's first slot >= chosen_watermark), value_id_base + k with its vote
        value at spans[k] in buf, or VALUE_NOOP; next_slot is the leader's nextSlot afterwards.  complete = -1: no
        quorum yet, no records.  out_capacity defaults to the engine's slot capacity."""
        buf = np.ascontiguousarray(buf, dtype=np.uint8)
        offsets = np.ascontiguousarray(offsets, dtype=np.int32)
        n = len(offsets) - 1
        cap = self.cfg.slot_capacity if out_capacity is None else out_capacity
        out = np.zeros(max(cap, 1), dtype=P2A)
        spans = np.zeros((max(cap, 1), 2), dtype=np.int32)
        res = np.zeros(4, dtype=np.int32)
        self._host_call(self._L.fpx_mencius_leader_phase1b_wire, leader_group, round_, chosen_watermark, recover_slot,
                        buf.ctypes.data if len(buf) else None, offsets.ctypes.data, n, value_id_base, out.ctypes.data,
                        spans.ctypes.data, cap, res.ctypes.data)
        k = int(res[2])
        return int(res[0]), int(res[1]), int(res[3]), out[:k].copy(), spans[:k].copy()

    def mencius_leader_phase1b_wire_dev(self, leader_group, round_, chosen_watermark, recover_slot, d_bytes, n_bytes,
                                        d_offsets, n, value_id_base, d_out, d_spans, out_capacity, d_result):
        self._check(self._L.fpx_mencius_leader_phase1b_wire_dev(self.h, leader_group, round_, chosen_watermark,
                                                                recover_slot, d_bytes, n_bytes, d_offsets, n,
                                                                value_id_base, d_out, d_spans, out_capacity, d_result))

    def wire_encode_mencius_phase2a(self, recs, buf, spans, value_id_base=0):
        """P2A records -> Mencius ProxyLeaderInbound{phase2a = 2} bytes, offsets[n+1], as wire_encode_phase2a
        (mencius_leader_phase1b_wire's output as it is)."""
        recs = np.ascontiguousarray(recs, dtype=P2A)
        buf = np.ascontiguousarray(buf, dtype=np.uint8)
        spans = np.ascontiguousarray(spans, dtype=np.int32).reshape(-1, 2)
        k = recs["value_id"].astype(np.int64) - value_id_base
        ok = (recs["value_id"] != VALUE_NOOP) & (k >= 0) & (k < len(spans))
        cap = int(32 * len(recs) + spans[k[ok], 1].clip(0).sum()) + 16   # 32: the longest head
        n = len(recs)
        out = np.zeros(cap, dtype=np.uint8)
        offs = np.zeros(n + 1, dtype=np.int32)
        self._host_call(self._L.fpx_wire_encode_mencius_phase2a, recs.ctypes.data, n,
                        buf.ctypes.data if len(buf) else None, len(buf), spans.ctypes.data, len(spans), value_id_base,
                        out.ctypes.data, cap, offs.ctypes.data)
        return out[:offs[n]].copy(), offs

    def wire_encode_mencius_phase2a_dev(self, d_in, n, d_bytes, n_bytes, d_spans, num_spans, value_id_base, d_out,
                                        out_capacity, d_offsets):
        self._check(self._L.fpx_wire_encode_mencius_phase2a_dev(self.h, d_in, n, d_bytes, n_bytes, d_spans, num_spans,
                                                                value_id_base, d_out, out_capacity, d_offsets))

    # -- device-pointer calls (raw device addresses, asynchronous on self.stream)
    def proxyleader_arm_dev(self, d_in, n):
        self._check(self._L.fpx_proxyleader_arm_dev(self.h, d_in, n))

    def acceptor_phase2a_dev(self, d_in, n, d_out_p2b, d_out_nack):
        self._check(self._L.fpx_acceptor_phase2a_dev(self.h, d_in, n, d_out_p2b, d_out_nack))

    def proxyleader_phase2b_dev(self, d_in, n, d_out):
        self._check(self._L.fpx_proxyleader_phase2b_dev(self.h, d_in, n, d_out))

    def replica_chosen_dev(self, d_in, n):
        self._check(self._L.fpx_replica_chosen_dev(self.h, d_in, n))

    def replica_chosen_last_dev(self, d_in):
        self._check(self._L.fpx_replica_chosen_last_dev(self.h, d_in))

    def chosen_watermark_dev(self, d_out=None):
        self._check(self._L.fpx_chosen_watermark_dev(self.h, d_out))

    def step_dev(self, d_arm, n_arm, d_p2a, n_p2a, d_out_p2b, d_out_nack, d_p2b, n_p2b, d_out_chosen, d_wm, ring_slot=-1):
        """One step of the co-located roles in one C call: acceptor batch, arm batch (disjoint state: order
        free), then the tally with the replica's handleChosen and the watermark scan fused into it."""
        self._check(self._L.fpx_step_dev(self.h, d_arm, n_arm, d_p2a, n_p2a, d_out_p2b, d_out_nack, d_p2b, n_p2b,
                                         d_out_chosen, d_wm, ring_slot))

    def vm_step_dev(self, d_req, n_req, d_p2a, n_p2a, d_reply, d_p2b, n_p2b, d_out_chosen, d_wm):
        """One step of the co-located vanilla Mencius servers in one C call: client requests, Phase2a batch,
        then the tally with the log put and the watermark fused into it."""
        self._check(self._L.fpx_vm_step_dev(self.h, d_req, n_req, d_p2a, n_p2a, d_reply, d_p2b, n_p2b, d_out_chosen, d_wm))

    def step_submit(self, arm, n_arm, p2a, n_p2a, p2b, n_p2b, out_p2b, out_nack, out_chosen):
        """Asynchronous step from HOST pointers (ints; pinned memory recommended), at most two in flight;
        arm = None arms from the Phase2a batch itself.  Pair with step_wait()."""
        self._check(self._L.fpx_step_submit(self.h, arm, n_arm, p2a, n_p2a, p2b, n_p2b, out_p2b, out_nack, out_chosen))

    def step_wait(self):
        """Completes the oldest submitted step: (n_p2b, n_nack, n_chosen, watermark)."""
        a, b, c, w = C.c_int32(0), C.c_int32(0), C.c_int32(0), C.c_int32(0)
        self._host_call(self._L.fpx_step_wait, C.byref(a), C.byref(b), C.byref(c), C.byref(w))
        return a.value, b.value, c.value, w.value

    def step_kernel_ms(self, ring_slot):
        a, t = C.c_float(0), C.c_float(0)
        self._check(self._L.fpx_step_kernel_ms(self.h, ring_slot, C.byref(a), C.byref(t)))
        return a.value, t.value

    def step_arm_ms(self, ring_slot):
        a = C.c_float(0)
        self._check(self._L.fpx_step_arm_ms(self.h, ring_slot, C.byref(a)))
        return a.value

    def set_coop_ctas_per_sm(self, k):
        """Cap the cooperative kernels at k resident CTAs per SM (0 = full grid) so that
        several engines can run side by side on one GPU."""
        self._check(self._L.fpx_set_coop_ctas_per_sm(self.h, k))

    def sync(self, check=True):
        r = _lib.SyncResult()
        st = self._L.fpx_sync(self.h, C.byref(r))
        if check:
            self._check(st, r.err_index)
        return r
