"""CPU model of the proxy leader arm's fresh-key certificate and of the fresh frontier (fpx_arm.cuh arm_certify /
arm_kernel<true>, DevStatus::fresh_rows in fpx_common.cuh).  TEST INFRASTRUCTURE, plain numpy.

A batch is armed with plain whole-row stores ("fresh") only if pass 1 of the certifying kernel finds every record
in this shard's live window with a round in 0 .. FPX_MAX_ROUND, every ordinal at or above the frontier, and the
slots strictly increasing over every adjacent pair; anything else takes the per-record CAS ("cas").  The frontier
is raised by every launch of the certifying kernel and by every tally launch, left alone by fpx_retire_below and
put back to 0 by fpx_reset.

Pass 1's geometry, whose seams are where a certificate can go wrong: CTAs of 1024 threads (kArmThreads); each
warp takes 4 consecutive 32-record chunks per stride (kArmCertUnroll), so warp w of CTA b starts at record
(b * 32 + w) * 128 and CTA b's first stride covers records [b * 4096, (b + 1) * 4096); lane 31 of a chunk compares
against the next chunk's first slot, loaded by itself.  The grid is sized for the per-record loop,
ceil(n / 8192) CTAs (kArmThreads * kArmUnroll) capped at the SM count, so pass 1 covers half of it per stride and
every batch above 4096 records runs a second stride.  The fallback of the certifying kernel keeps 6 chunks per
warp in flight (kArmUnrollCertified)."""
from dataclasses import dataclass

import numpy as np

THREADS = 1024                  # kArmThreads: threads per arm CTA
CHUNK = 32                      # records per warp chunk
CERT_UNROLL = 4                 # kArmCertUnroll: chunks per warp per stride in pass 1 (and pass 2)
UNROLL = 8                      # kArmUnroll: chunks per warp in flight in the plain CAS kernel
FALLBACK_UNROLL = 6             # kArmUnrollCertified: the same in the certifying kernel's CAS fallback
WARP_GROUP = CHUNK * CERT_UNROLL                    # 128 records: one warp's pass-1 unroll group
CERT_CTA = THREADS * CERT_UNROLL                    # 4096 records: one CTA's share of a pass-1 stride
GRID_CTA = THREADS * UNROLL                         # 8192 records per CTA when the grid is sized
MAX_ROUND = 0x7ffffff0                              # FPX_MAX_ROUND
RETIRED = -2                                        # kLocalRetired

MULTIPAXOS, MENCIUS, VANILLA = "multipaxos", "mencius", "vanilla"


def arm_blocks(n, num_sms):
    """CTAs of one arm launch (arm_launch in fpx_engine.cu)"""
    return min(-(-n // GRID_CTA), num_sms)


def cert_stride(n, num_sms):
    """records pass 1 covers per grid stride"""
    return arm_blocks(n, num_sms) * CERT_CTA


@dataclass
class Geometry:
    """The live window of one shard: ordinals base_local .. base_local + local_slots - 1 (fpx_create,
    fpx_retire_below)."""
    capacity: int                       # the engine's slot_capacity
    shard_index: int = 0
    shard_count: int = 1
    base_local: int = 0

    @property
    def local_slots(self):
        return max(1, (self.capacity - self.shard_index + self.shard_count - 1) // self.shard_count)

    @property
    def slot_capacity(self):
        """one past the last slot of the live window"""
        return min(self.capacity + self.base_local * self.shard_count, 0x7fffffff)

    def retire_below(self, slot):
        """the first ordinal whose slot is >= `slot` becomes the base (fpx_retire_below)"""
        self.base_local = max(self.base_local, (slot - self.shard_index + self.shard_count - 1) // self.shard_count)


def local_ordinal(slot, g):
    """Ordinal (slot / shard_count) of each slot in this shard's live window; -1 for a slot outside the window, of
    another shard or at or above slot_capacity; RETIRED below the window (local_slot in fpx_common.cuh, in
    ordinals instead of ring indices)."""
    s = np.asarray(slot, dtype=np.int64)
    out = np.full(s.shape, -1, dtype=np.int64)
    ok = (s >= 0) & (s < g.slot_capacity) & (s % g.shard_count == g.shard_index)
    u = s // g.shard_count
    rel = u - g.base_local
    out[ok & (rel < 0)] = RETIRED
    live = ok & (rel >= 0) & (rel < g.local_slots)
    out[live] = u[live]
    return out


def certified(batch, g, frontier):
    """Would pass 1 certify the batch (P2A records) for plain row stores?"""
    n = len(batch)
    if n == 0:
        return False
    slot = np.asarray(batch["slot"], dtype=np.int64)
    rnd = np.asarray(batch["round"], dtype=np.int64)
    ords = local_ordinal(slot, g)
    if (ords < 0).any():
        return False
    if ((rnd < 0) | (rnd > MAX_ROUND)).any():
        return False
    if (ords < frontier).any():
        return False
    return bool((slot[:-1] < slot[1:]).all())


def live_top(slots, g):
    """largest ordinal of the slots in the live window, or -1"""
    ords = local_ordinal(slots, g)
    live = ords[ords >= 0]
    return int(live.max()) if len(live) else -1


class Frontier:
    """The fresh frontier of one engine and the engine state that decides an arm's path.  kind: MULTIPAXOS,
    MENCIUS (compartmentalized) or VANILLA."""

    def __init__(self, kind, g):
        self.kind, self.g = kind, g
        self.value = 0
        self.unit_ranges = False       # a one-slot noop range was armed since the last reset (fpx_engine_ranges.inc)
        self.last_path = "none"

    def certifying(self):
        """does an arm launch run the certifying kernel?"""
        return self.kind != VANILLA and not self.unit_ranges

    def expected_path(self, batch):
        """"fresh" / "cas" for a non-empty batch; an empty one launches nothing: the last path stands"""
        if len(batch) == 0:
            return self.last_path
        if not self.certifying():
            return "cas"
        return "fresh" if certified(batch, self.g, self.value) else "cas"

    def arm(self, batch):
        """One arm call: -> the path it takes (expected_path), with the frontier moved as the kernel moves it."""
        path = self.expected_path(batch)
        if len(batch) and self.certifying():
            self.value = max(self.value, live_top(batch["slot"], self.g) + 1)
        self.last_path = path
        return path

    def tally(self, votes):
        """One tally call (P2B records, any number of launches)."""
        if len(votes):
            self.value = max(self.value, live_top(votes["slot"], self.g) + 1)

    def arm_range(self, ranges):
        """A Mencius Phase2aNoopRange call (P2A_RANGE records)."""
        if len(ranges) and ((np.asarray(ranges["slot_end"]) - np.asarray(ranges["slot_start"])) == 1).any():
            self.unit_ranges = True

    def retire_below(self, slot):
        self.g.retire_below(slot)

    def reset(self):
        self.value = 0
        self.unit_ranges = False
        self.last_path = "none"
        self.g.base_local = 0
