"""frankenpaxos_b200 -- H100-native engine for FrankenPaxos's quorum-vote hot path.

The product is libfpx.so (CUDA, sm_90a) behind the C ABI of include/fpx.h; this
package is the Python handle over it plus mirrors of the reference's classes on
the path (quorums.Grid / SimpleMajority, multipaxos.Config / ProxyLeader /
Acceptor).  Importing the package does not need a GPU; constructing an Engine
does -- there is no CPU fallback.
"""
from .engine import (CHOSEN, NACK, P2A, P2B, Engine, FpxError, dst,  # noqa: F401
                     MULTIPAXOS, MENCIUS, VANILLA_MENCIUS, P2A_RANGE, P2B_RANGE, CHOSEN_RANGE, VM_SKIP, VALUE_NOOP,
                     WIRE_REC, WIRE_PROXYLEADER_INBOUND, WIRE_ACCEPTOR_INBOUND,
                     WIRE_MENCIUS_PROXYLEADER_INBOUND, WIRE_MENCIUS_ACCEPTOR_INBOUND)

__all__ = ["Engine", "FpxError", "P2A", "P2B", "CHOSEN", "NACK", "dst"]
