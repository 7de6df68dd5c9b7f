"""ctypes loader for libfpx.so (the C ABI of include/fpx.h).

There is no CPU fallback: if the shared library is missing it is built with
nvcc; if that fails, or a symbol declared in include/fpx.h is missing, import
of the product raises.
"""
import ctypes as C
import os

from . import build as _build

_lib = None

SYMBOLS = [
    "fpx_abi_version", "fpx_strerror", "fpx_last_error", "fpx_create", "fpx_destroy", "fpx_reset",
    "fpx_proxyleader_arm", "fpx_acceptor_phase2a", "fpx_proxyleader_phase2b", "fpx_replica_chosen",
    "fpx_chosen_watermark", "fpx_quorum_eval", "fpx_snapshot_acceptor", "fpx_snapshot_log",
    "fpx_proxyleader_arm_dev", "fpx_acceptor_phase2a_dev", "fpx_proxyleader_phase2b_dev",
    "fpx_replica_chosen_dev", "fpx_replica_chosen_last_dev", "fpx_chosen_watermark_dev", "fpx_sync",
    "fpx_stream", "fpx_launch_count", "fpx_set_coop_ctas_per_sm", "fpx_step_dev", "fpx_step_kernel_ms", "fpx_step_arm_ms",
    "fpx_acceptor_phase1a", "fpx_leader_safe_values",
    "fpx_vm_client_request", "fpx_vm_phase2a", "fpx_vm_learn_chosen", "fpx_vm_skip", "fpx_vm_client_request_dev", "fpx_vm_phase2a_dev", "fpx_vm_step_dev",
    "fpx_mencius_arm_range", "fpx_mencius_acceptor_noop_range", "fpx_mencius_range_phase2b",
    "fpx_mencius_replica_chosen_range", "fpx_mencius_replica_range_first", "fpx_mencius_replica_range_fill",
    "fpx_wire_decode_inbound", "fpx_wire_decode_inbound_dev", "fpx_wire_encode_phase2b", "fpx_wire_encode_phase2b_dev",
    "fpx_wire_encode_nack", "fpx_wire_encode_chosen",
    "fpx_step_submit", "fpx_step_wait", "fpx_retire_below", "fpx_exchange_export", "fpx_exchange_attach", "fpx_exchange_attach_local", "fpx_exchange_epoch",
    "fpx_global_watermark", "fpx_global_watermark_dev",
    "fpx_conflict_index_create", "fpx_conflict_index_destroy", "fpx_conflict_index_put_snapshot", "fpx_conflict_index_batch",
    "fpx_depgraph_create", "fpx_depgraph_destroy", "fpx_depgraph_commit", "fpx_depgraph_update_executed", "fpx_depgraph_execute",
    "fpx_epaxos_stream", "fpx_epaxos_sync", "fpx_epaxos_lead_dev", "fpx_epaxos_preaccept_dev", "fpx_epaxos_accept_dev",
    "fpx_epaxos_preacceptok_dev", "fpx_epaxos_acceptok_dev", "fpx_epaxos_preaccept_sets",
    "fpx_epaxos_create", "fpx_epaxos_destroy", "fpx_epaxos_lead", "fpx_epaxos_preaccept", "fpx_epaxos_accept",
    "fpx_epaxos_preacceptok", "fpx_epaxos_acceptok", "fpx_epaxos_entry", "fpx_epaxos_last_kernel_ms", "fpx_depset_union", "fpx_depset_union_dense_dev",
]


class Config(C.Structure):
    """struct fpx_config (include/fpx.h)."""
    _fields_ = [(n, C.c_int32) for n in (
        "struct_size", "protocol", "f", "num_acceptor_groups", "acceptors_per_group", "flexible",
        "num_leaders", "num_replicas", "slot_capacity", "overflow_capacity", "max_batch", "device",
        "shard_index", "shard_count", "num_leader_groups")]


class SyncResult(C.Structure):
    """struct fpx_sync_result (include/fpx.h)."""
    _fields_ = [("status", C.c_int32), ("reserved", C.c_int32), ("err_index", C.c_int64),
                ("n_p2b", C.c_int32), ("n_nack", C.c_int32), ("n_chosen", C.c_int32),
                ("watermark", C.c_int32)]


def lib():
    global _lib
    if _lib is not None:
        return _lib
    path = os.environ.get("FPX_LIB_OVERRIDE") or _build.LIB      # override: A/B against another build (profiles/)
    if path == _build.LIB and (not os.path.exists(path) or (_build.stale() and _build.have_nvcc())):
        path = _build.build(force=True)
    L = C.CDLL(path)
    missing = [s for s in SYMBOLS if not hasattr(L, s)]
    if missing:
        raise ImportError(f"libfpx.so lacks symbols declared in include/fpx.h: {missing}")
    vp, i32, i64 = C.c_void_p, C.c_int32, C.c_int64
    p = C.POINTER
    L.fpx_abi_version.restype = i32
    L.fpx_strerror.argtypes = [i32]; L.fpx_strerror.restype = C.c_char_p
    L.fpx_last_error.argtypes = [vp]; L.fpx_last_error.restype = C.c_char_p
    L.fpx_create.argtypes = [p(vp), p(Config)]; L.fpx_create.restype = i32
    L.fpx_destroy.argtypes = [vp]; L.fpx_destroy.restype = None
    L.fpx_reset.argtypes = [vp]; L.fpx_reset.restype = i32
    L.fpx_proxyleader_arm.argtypes = [vp, vp, i32, p(i64)]; L.fpx_proxyleader_arm.restype = i32
    L.fpx_acceptor_phase2a.argtypes = [vp, vp, i32, vp, p(i32), vp, p(i32), p(i64)]
    L.fpx_acceptor_phase2a.restype = i32
    L.fpx_proxyleader_phase2b.argtypes = [vp, vp, i32, vp, p(i32), p(i64)]
    L.fpx_proxyleader_phase2b.restype = i32
    L.fpx_replica_chosen.argtypes = [vp, vp, i32, p(i64)]; L.fpx_replica_chosen.restype = i32
    L.fpx_chosen_watermark.argtypes = [vp, p(i32)]; L.fpx_chosen_watermark.restype = i32
    L.fpx_quorum_eval.argtypes = [vp, i32, vp, i32, vp]; L.fpx_quorum_eval.restype = i32
    L.fpx_snapshot_acceptor.argtypes = [vp, i32, i32, p(i32), p(i32), i32, i32, vp, vp]
    L.fpx_snapshot_acceptor.restype = i32
    L.fpx_snapshot_log.argtypes = [vp, i32, i32, vp]; L.fpx_snapshot_log.restype = i32
    L.fpx_proxyleader_arm_dev.argtypes = [vp, vp, i32]; L.fpx_proxyleader_arm_dev.restype = i32
    L.fpx_acceptor_phase2a_dev.argtypes = [vp, vp, i32, vp, vp]; L.fpx_acceptor_phase2a_dev.restype = i32
    L.fpx_proxyleader_phase2b_dev.argtypes = [vp, vp, i32, vp]; L.fpx_proxyleader_phase2b_dev.restype = i32
    L.fpx_replica_chosen_dev.argtypes = [vp, vp, i32]; L.fpx_replica_chosen_dev.restype = i32
    L.fpx_replica_chosen_last_dev.argtypes = [vp, vp]; L.fpx_replica_chosen_last_dev.restype = i32
    L.fpx_chosen_watermark_dev.argtypes = [vp, vp]; L.fpx_chosen_watermark_dev.restype = i32
    L.fpx_acceptor_phase1a.argtypes = [vp, i32, i32, i32, p(i32)]; L.fpx_acceptor_phase1a.restype = i32
    L.fpx_leader_safe_values.argtypes = [vp, C.c_uint32, i32, i32, vp, vp, p(i32)]; L.fpx_leader_safe_values.restype = i32
    L.fpx_vm_client_request.argtypes = [vp, vp, i32, p(i64)]; L.fpx_vm_client_request.restype = i32
    L.fpx_vm_phase2a.argtypes = [vp, vp, i32, vp, p(i64)]; L.fpx_vm_phase2a.restype = i32
    L.fpx_vm_learn_chosen.argtypes = [vp, vp, i32, p(i64)]; L.fpx_vm_learn_chosen.restype = i32
    L.fpx_vm_skip.argtypes = [vp, vp, i32, p(i64)]; L.fpx_vm_skip.restype = i32
    L.fpx_vm_client_request_dev.argtypes = [vp, vp, i32]; L.fpx_vm_client_request_dev.restype = i32
    L.fpx_vm_phase2a_dev.argtypes = [vp, vp, i32, vp]; L.fpx_vm_phase2a_dev.restype = i32
    L.fpx_mencius_arm_range.argtypes = [vp, vp, i32, p(i64)]; L.fpx_mencius_arm_range.restype = i32
    L.fpx_mencius_acceptor_noop_range.argtypes = [vp, vp, i32, vp, p(i32), vp, p(i32), p(i64)]
    L.fpx_mencius_acceptor_noop_range.restype = i32
    L.fpx_mencius_range_phase2b.argtypes = [vp, vp, i32, vp, p(i32), p(i64)]; L.fpx_mencius_range_phase2b.restype = i32
    L.fpx_mencius_replica_chosen_range.argtypes = [vp, vp, i32, p(i64)]
    L.fpx_mencius_replica_chosen_range.restype = i32
    L.fpx_mencius_replica_range_first.argtypes = [vp, vp, i32, vp, p(i64)]; L.fpx_mencius_replica_range_first.restype = i32
    L.fpx_mencius_replica_range_fill.argtypes = [vp, vp, i32, vp, p(i64)]; L.fpx_mencius_replica_range_fill.restype = i32
    L.fpx_wire_decode_inbound.argtypes = [vp, i32, vp, vp, i32, vp, vp, p(i64)]; L.fpx_wire_decode_inbound.restype = i32
    L.fpx_wire_decode_inbound_dev.argtypes = [vp, i32, vp, vp, i32, vp, vp]; L.fpx_wire_decode_inbound_dev.restype = i32
    L.fpx_wire_encode_phase2b.argtypes = [vp, vp, i32, vp, i32, vp, p(i64)]; L.fpx_wire_encode_phase2b.restype = i32
    L.fpx_wire_encode_phase2b_dev.argtypes = [vp, vp, i32, vp, i32, vp]; L.fpx_wire_encode_phase2b_dev.restype = i32
    L.fpx_wire_encode_nack.argtypes = [vp, vp, i32, vp, i32, vp, p(i64)]; L.fpx_wire_encode_nack.restype = i32
    L.fpx_wire_encode_chosen.argtypes = [vp, vp, i32, vp, vp, i32, vp, i32, vp, p(i64)]
    L.fpx_wire_encode_chosen.restype = i32
    L.fpx_step_dev.argtypes = [vp, vp, i32, vp, i32, vp, vp, vp, i32, vp, vp, i32]; L.fpx_step_dev.restype = i32
    L.fpx_vm_step_dev.argtypes = [vp, vp, i32, vp, i32, vp, vp, i32, vp, vp]; L.fpx_vm_step_dev.restype = i32
    L.fpx_step_kernel_ms.argtypes = [vp, i32, p(C.c_float), p(C.c_float)]; L.fpx_step_kernel_ms.restype = i32
    L.fpx_step_arm_ms.argtypes = [vp, i32, p(C.c_float)]; L.fpx_step_arm_ms.restype = i32
    L.fpx_sync.argtypes = [vp, p(SyncResult)]; L.fpx_sync.restype = i32
    L.fpx_set_coop_ctas_per_sm.argtypes = [vp, i32]; L.fpx_set_coop_ctas_per_sm.restype = i32
    L.fpx_stream.argtypes = [vp]; L.fpx_stream.restype = vp
    L.fpx_launch_count.argtypes = [vp]; L.fpx_launch_count.restype = i64
    L.fpx_retire_below.argtypes = [vp, i32]; L.fpx_retire_below.restype = i32
    L.fpx_step_submit.argtypes = [vp, vp, i32, vp, i32, vp, i32, vp, vp, vp]; L.fpx_step_submit.restype = i32
    L.fpx_step_wait.argtypes = [vp, p(i32), p(i32), p(i32), p(i32), p(i64)]; L.fpx_step_wait.restype = i32
    L.fpx_exchange_export.argtypes = [vp, vp]; L.fpx_exchange_export.restype = i32
    L.fpx_exchange_attach.argtypes = [vp, i32, vp]; L.fpx_exchange_attach.restype = i32
    L.fpx_exchange_attach_local.argtypes = [vp, i32, vp]; L.fpx_exchange_attach_local.restype = i32
    L.fpx_exchange_epoch.argtypes = [vp]; L.fpx_exchange_epoch.restype = C.c_uint32
    L.fpx_global_watermark_dev.argtypes = [vp, C.c_uint32, i32, vp, vp]; L.fpx_global_watermark_dev.restype = i32
    L.fpx_global_watermark.argtypes = [vp, C.c_uint32, i32, p(i32), vp]; L.fpx_global_watermark.restype = i32
    if hasattr(L, "fpx_debug_set_tally_path"):
        L.fpx_debug_set_tally_path.argtypes = [vp, i32]; L.fpx_debug_set_tally_path.restype = i32
        L.fpx_debug_last_tally_path.argtypes = [vp]; L.fpx_debug_last_tally_path.restype = i32
    if hasattr(L, "fpx_debug_set_acceptor_segments"):
        L.fpx_debug_set_acceptor_segments.argtypes = [vp, i32]; L.fpx_debug_set_acceptor_segments.restype = i32
    if L.fpx_abi_version() != 1:
        raise ImportError("libfpx.so ABI version mismatch")
    _lib = L
    return L
