"""frankenpaxos_b200 -- H100-native engine for FrankenPaxos's quorum-vote hot path.

The product is libfpx.so (CUDA, sm_90a) behind the C ABI of include/fpx.h; this
package is the Python handle over it plus mirrors of the reference's classes on
the path (quorums.Grid / SimpleMajority, multipaxos.Config / ProxyLeader /
Acceptor).  Importing the package does not need a GPU; constructing an Engine
does -- there is no CPU fallback.
"""
from .engine import (CHOSEN, NACK, P2A, P2B, Engine, FpxError, dst,  # noqa: F401
                     MULTIPAXOS, MENCIUS, VANILLA_MENCIUS, VM_REPLY_PHASE2B, VM_REPLY_NACK, VM_REPLY_CHOSEN,
                     VM_REPLY_CHOSEN_RETIRED, P2A_RANGE, P2B_RANGE, CHOSEN_RANGE, MENCIUS_CHOSEN, VM_SKIP, VALUE_NOOP,
                     WIRE_REC, WIRE_PROXYLEADER_INBOUND, WIRE_ACCEPTOR_INBOUND,
                     WIRE_MENCIUS_PROXYLEADER_INBOUND, WIRE_MENCIUS_ACCEPTOR_INBOUND, VM_WIRE_CLIENT_REQUEST,
                     VM_WIRE_PHASE2A, VM_WIRE_PHASE2B, VM_WIRE_SKIP, VM_WIRE_CHOSEN, VM_WIRE_PHASE2_NACK)

from .reads import (Reads, READS_CLIENT, READS_READ_BATCHER, READ_OPEN, MAX_SLOT_REPLY, READ_SLOT,  # noqa: F401
                    READ_REQUEST, READ_REPLY)

__all__ = ["Engine", "FpxError", "P2A", "P2B", "CHOSEN", "NACK", "dst", "Reads"]
