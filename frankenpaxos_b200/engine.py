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
VALUE_NOOP = -(1 << 31)
WIRE_REC = np.dtype([("a", "<i4"), ("b", "<i4"), ("c", "<i4"), ("d", "<i4")])
WIRE_PROXYLEADER_INBOUND, WIRE_ACCEPTOR_INBOUND = 0, 1
WIRE_MENCIUS_PROXYLEADER_INBOUND, WIRE_MENCIUS_ACCEPTOR_INBOUND = 2, 3

MULTIPAXOS, MENCIUS, VANILLA_MENCIUS = 0, 1, 2

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


def dst(group, acceptor):
    """fpx_p2a.dst encoding."""
    return (np.asarray(group, dtype=np.int32) << 16) | np.asarray(acceptor, dtype=np.int32)


class Engine:
    """One GPU-resident {acceptors, proxy leader, replica log} for one config."""

    def __init__(self, f, num_acceptor_groups, acceptors_per_group, flexible=False, num_leaders=None,
                 num_replicas=None, slot_capacity=1 << 20, overflow_capacity=1 << 14, max_batch=1 << 20,
                 device=0, shard_index=0, shard_count=1, protocol=MULTIPAXOS, num_leader_groups=0):
        L = _lib.lib()
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
        self._L = L
        self.h = C.c_void_p()
        st = L.fpx_create(C.byref(self.h), C.byref(cfg))
        if st != OK:
            self.h = None
            raise FpxError(st)

    # -- life cycle
    def close(self):
        if getattr(self, "h", None):
            self._L.fpx_destroy(self.h)
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

    def reset(self):
        self._check(self._L.fpx_reset(self.h))

    def retire_below(self, slot):
        """Slide the live window: slots below `slot` (all executed) are recycled for the slots slot_capacity ahead."""
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

    @property
    def last_tally_path(self):
        """'sweep' / 'exact': what the last proxyleader_phase2b launch did."""
        return {1: "sweep", 2: "exact"}.get(self._L.fpx_debug_last_tally_path(self.h), "none")

    # -- host-pointer calls (numpy in / numpy out)
    def proxyleader_arm(self, p2a):
        p2a = np.ascontiguousarray(p2a, dtype=P2A)
        err = C.c_int64(-1)
        st = self._L.fpx_proxyleader_arm(self.h, p2a.ctypes.data, len(p2a), C.byref(err))
        self._check(st, err.value)

    def acceptor_phase2a(self, p2a):
        p2a = np.ascontiguousarray(p2a, dtype=P2A)
        n = len(p2a)
        out = np.empty(max(n, 1), dtype=P2B)
        nack = np.empty(max(n, 1), dtype=NACK)
        n1, n2, err = C.c_int32(0), C.c_int32(0), C.c_int64(-1)
        st = self._L.fpx_acceptor_phase2a(self.h, p2a.ctypes.data, n, out.ctypes.data, C.byref(n1),
                                          nack.ctypes.data, C.byref(n2), C.byref(err))
        self._check(st, err.value)
        return out[:n1.value], nack[:n2.value]

    def proxyleader_phase2b(self, p2b):
        p2b = np.ascontiguousarray(p2b, dtype=P2B)
        n = len(p2b)
        out = np.empty(max(n, 1), dtype=CHOSEN)
        n1, err = C.c_int32(0), C.c_int64(-1)
        st = self._L.fpx_proxyleader_phase2b(self.h, p2b.ctypes.data, n, out.ctypes.data, C.byref(n1),
                                             C.byref(err))
        self._check(st, err.value)
        return out[:n1.value]

    def replica_chosen(self, chosen):
        chosen = np.ascontiguousarray(chosen, dtype=CHOSEN)
        err = C.c_int64(-1)
        st = self._L.fpx_replica_chosen(self.h, chosen.ctypes.data, len(chosen), C.byref(err))
        self._check(st, err.value)

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
        err = C.c_int64(-1)
        self._check(self._L.fpx_vm_client_request(self.h, p2a.ctypes.data, len(p2a), C.byref(err)), err.value)

    def vm_phase2a(self, p2a):
        """dense replies {group = kind (0 Phase2b, 1 Phase2Nack, 2 Chosen), acceptor = server, slot, round|value}"""
        p2a = np.ascontiguousarray(p2a, dtype=P2A)
        out = np.empty(max(len(p2a), 1), dtype=P2B)
        err = C.c_int64(-1)
        self._check(self._L.fpx_vm_phase2a(self.h, p2a.ctypes.data, len(p2a), out.ctypes.data, C.byref(err)), err.value)
        return out[:len(p2a)]

    def vm_learn_chosen(self, recs):
        recs = np.ascontiguousarray(recs, dtype=P2B)
        err = C.c_int64(-1)
        self._check(self._L.fpx_vm_learn_chosen(self.h, recs.ctypes.data, len(recs), C.byref(err)), err.value)

    def vm_skip(self, recs):
        """Server.advanceWithSkips' log fill (own=1) / Server.handleSkip (own=0)."""
        recs = np.ascontiguousarray(recs, dtype=VM_SKIP)
        err = C.c_int64(-1)
        self._check(self._L.fpx_vm_skip(self.h, recs.ctypes.data, len(recs), C.byref(err)), err.value)

    # -- S/mencius Phase2aNoopRange path
    def mencius_arm_range(self, recs):
        recs = np.ascontiguousarray(recs, dtype=P2A_RANGE)
        err = C.c_int64(-1)
        self._check(self._L.fpx_mencius_arm_range(self.h, recs.ctypes.data, len(recs), C.byref(err)), err.value)

    def mencius_acceptor_noop_range(self, recs):
        recs = np.ascontiguousarray(recs, dtype=P2A_RANGE)
        n = len(recs)
        out = np.zeros(max(n, 1), dtype=P2B_RANGE)
        nack = np.zeros(max(n, 1), dtype=NACK)
        n1, n2, err = C.c_int32(0), C.c_int32(0), C.c_int64(-1)
        self._check(self._L.fpx_mencius_acceptor_noop_range(self.h, recs.ctypes.data, n, out.ctypes.data, C.byref(n1),
                                                            nack.ctypes.data, C.byref(n2), C.byref(err)), err.value)
        return out[:n1.value].copy(), nack[:n2.value].copy()

    def mencius_range_phase2b(self, recs):
        recs = np.ascontiguousarray(recs, dtype=P2B_RANGE)
        n = len(recs)
        out = np.zeros(max(n, 1), dtype=CHOSEN_RANGE)
        n1, err = C.c_int32(0), C.c_int64(-1)
        self._check(self._L.fpx_mencius_range_phase2b(self.h, recs.ctypes.data, n, out.ctypes.data, C.byref(n1),
                                                      C.byref(err)), err.value)
        return out[:n1.value].copy()

    def mencius_replica_chosen_range(self, recs):
        recs = np.ascontiguousarray(recs, dtype=CHOSEN_RANGE)
        err = C.c_int64(-1)
        self._check(self._L.fpx_mencius_replica_chosen_range(self.h, recs.ctypes.data, len(recs), C.byref(err)),
                    err.value)

    RANGE_NO_HIT = 0x7f7f7f7f

    def mencius_replica_range_first(self, recs):
        """Per record: this shard's first slot of the range that is already in its log (RANGE_NO_HIT if none)."""
        recs = np.ascontiguousarray(recs, dtype=CHOSEN_RANGE)
        first = np.full(max(len(recs), 1), self.RANGE_NO_HIT, dtype=np.int32)
        err = C.c_int64(-1)
        self._check(self._L.fpx_mencius_replica_range_first(self.h, recs.ctypes.data, len(recs), first.ctypes.data,
                                                            C.byref(err)), err.value)
        return first[:len(recs)]

    def mencius_replica_range_fill(self, recs, first):
        """Noop into this shard's slots of [start, min(end, first[i])): `first` = the minimum over the shards."""
        recs = np.ascontiguousarray(recs, dtype=CHOSEN_RANGE)
        first = np.ascontiguousarray(first, dtype=np.int32)
        assert len(first) == len(recs)
        err = C.c_int64(-1)
        self._check(self._L.fpx_mencius_replica_range_fill(self.h, recs.ctypes.data, len(recs), first.ctypes.data,
                                                           C.byref(err)), err.value)

    # -- wire codec: protobuf bytes of a batch of messages <-> records (include/fpx.h)
    def wire_decode_inbound(self, inbound, buf, offsets):
        """buf: uint8 array with the messages back to back, offsets[n+1].  Returns (kind[n], rec[n])."""
        buf = np.ascontiguousarray(buf, dtype=np.uint8)
        offsets = np.ascontiguousarray(offsets, dtype=np.int32)
        n = len(offsets) - 1
        kind = np.zeros(max(n, 1), dtype=np.int32)
        rec = np.zeros(max(n, 1), dtype=WIRE_REC)
        err = C.c_int64(-1)
        self._check(self._L.fpx_wire_decode_inbound(self.h, inbound, buf.ctypes.data if len(buf) else None,
                                                    offsets.ctypes.data, n, kind.ctypes.data, rec.ctypes.data,
                                                    C.byref(err)), err.value)
        return kind[:n], rec[:n]

    def _wire_encode(self, fn, recs, dtype, max_per, *extra):
        recs = np.ascontiguousarray(recs, dtype=dtype)
        n = len(recs)
        cap = max(16, n * max_per) if not extra else extra[-1]
        out = np.zeros(cap, dtype=np.uint8)
        offs = np.zeros(n + 1, dtype=np.int32)
        err = C.c_int64(-1)
        args = [self.h, recs.ctypes.data, n] + list(extra[:-1] if extra else []) + [out.ctypes.data, cap, offs.ctypes.data,
                                                                                     C.byref(err)]
        self._check(fn(*args), err.value)
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

    def vm_client_request_dev(self, d_in, n):
        self._check(self._L.fpx_vm_client_request_dev(self.h, d_in, n))

    def vm_phase2a_dev(self, d_in, n, d_reply):
        self._check(self._L.fpx_vm_phase2a_dev(self.h, d_in, n, d_reply))

    def wire_decode_inbound_dev(self, inbound, d_bytes, d_offsets, n, d_kind, d_out):
        self._check(self._L.fpx_wire_decode_inbound_dev(self.h, inbound, d_bytes, d_offsets, n, d_kind, d_out))

    def wire_encode_phase2b_dev(self, d_in, n, d_out, out_capacity, d_offsets):
        self._check(self._L.fpx_wire_encode_phase2b_dev(self.h, d_in, n, d_out, out_capacity, d_offsets))

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
        a, b, c, w, err = C.c_int32(0), C.c_int32(0), C.c_int32(0), C.c_int32(0), C.c_int64(-1)
        st = self._L.fpx_step_wait(self.h, C.byref(a), C.byref(b), C.byref(c), C.byref(w), C.byref(err))
        self._check(st, err.value)
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
