"""Batch builders of the wire codec's edge tests (tests/test_wire_edges_*.py).  TEST INFRASTRUCTURE.

Decoder batches whose CTAs of 256 messages span exactly 24 575, 24 576 or 24 577 bytes from `lo & ~15` (the
shared-memory stage window, kWireStage in fpx_wire.cuh, and one byte either side), with leading bytes that belong
to no message and a total that is not a multiple of 16; encoder records past tile_offsets_kernel's first chunk of
4096 tiles; and values whose lengths take every varint width."""
import numpy as np

STAGE = 24 * 1024           # kWireStage: bytes of a decoder CTA's span staged in shared memory
CTA = 256                   # messages per decoder CTA (kWireDecThreads = kRwThreads)
ENC_TILE = 1024             # records per encoder tile (kWireEncTile)
SCAN_CHUNK = 4096           # counters per pass of tile_offsets_kernel's loop
EDGE_SPANS = (STAGE - 1, STAGE, STAGE + 1)
# CTA k starts at lo % 16 = (span of CTA k-1) % 16, i.e. 15, 0 or 1 after 24 575, 24 576, 24 577.  This order holds
# every ordered pair of the three spans once (a de Bruijn sequence), so every span meets every lo % 16.
SPAN_ORDER = (STAGE - 1, STAGE - 1, STAGE, STAGE - 1, STAGE + 1, STAGE, STAGE, STAGE + 1, STAGE + 1, STAGE - 1)
LEAD = 33                   # bytes before message 0 (offsets[0]); 33 % 16 = 1
PAD_FIELD = 15              # the padding's field number: above every member of every decoded oneof
# the large batches past the first scan chunk
BIG_N = (SCAN_CHUNK * ENC_TILE, SCAN_CHUNK * ENC_TILE + ENC_TILE + 1)
# value lengths of every length-varint width, around each width's edge
VALUE_LENS = (0, 1, 127, 128, 16383, 16384, (1 << 21) - 1, 1 << 21)


def venc(v):
    """base-128 varint; a negative int32 is sign-extended to ten bytes"""
    v = int(v)
    if v < 0:
        v &= (1 << 64) - 1
    out = bytearray()
    while True:
        b = v & 0x7f
        v >>= 7
        out.append(b | (0x80 if v else 0))
        if not v:
            return bytes(out)


def fint(f, v):
    return venc(f << 3) + venc(v)


def fbytes(f, b):
    return venc(f << 3 | 2) + venc(len(b)) + bytes(b)


def pad(msg, size):
    """msg with an unknown top-level length-delimited field appended so that it is exactly `size` bytes"""
    need = size - len(msg)
    if need == 0:
        return msg
    for p in range(need - 2, -1, -1):
        if 1 + len(venc(p)) + p == need:
            return msg + fbytes(PAD_FIELD, bytes(p))
    raise ValueError(f"cannot pad {len(msg)} bytes to {size}")


def truncated(msg, size):
    """`size` bytes of a message that ends one byte short: its padding field runs past the end"""
    return pad(msg, size + 1)[:size]


def fill(msgs, total):
    """msgs padded to `total` bytes in all, the padding spread evenly"""
    extra = total - sum(len(m) for m in msgs)
    q, r = divmod(extra, len(msgs))
    assert q >= 2 and q + 1 < 130, (q, total)      # every pad takes >= 2 bytes; 130 is not a field's size
    return [pad(m, len(m) + q + (k < r)) for k, m in enumerate(msgs)]


def pack(msgs, lead=0):
    """`lead` bytes that belong to no message (0xff: a malformed varint if anything parsed them), then the messages
    back to back -> (buf with 16 spare bytes, offsets[n+1])"""
    offs = np.zeros(len(msgs) + 1, dtype=np.int64)
    offs[0] = lead
    offs[1:] = lead + np.cumsum([len(m) for m in msgs])
    buf = b"\xff" * lead + b"".join(msgs) + bytes(16)
    return np.frombuffer(buf, dtype=np.uint8).copy(), offs.astype(np.int32)


def cta_spans(offs):
    """[(lo, hi, span from lo & ~15, staged)] of each decoder CTA, as wire_stage_span computes them"""
    n = len(offs) - 1
    out = []
    for m0 in range(0, n, CTA):
        lo, hi = int(offs[m0]), int(offs[min(n, m0 + CTA)])
        span = hi - (lo & ~15)
        out.append((lo, hi, span, span <= STAGE))
    return out


def stage_batch(make, g, spans=SPAN_ORDER, lead=LEAD, tail=100, cut=None):
    """Messages make(g) in full CTAs whose spans from lo & ~15 are `spans`, after `lead` bytes that belong to no
    message, then `tail` messages ending at a total that is not a multiple of 16.  cut = k: the batch ends with CTA
    k, whose last message is truncated.  -> (buf, offs)"""
    msgs, pos = [], lead
    for k, span in enumerate(spans):
        size = (pos & ~15) + span - pos
        cta = fill([make(g) for _ in range(CTA)], size)
        if cut == k:
            cta[-1] = truncated(cta[-1][:0], len(cta[-1]))
        msgs += cta
        pos += size
        if cut == k:
            return pack(msgs, lead)
    if tail:
        t = [make(g) for _ in range(tail)]
        size = sum(len(m) for m in t) + 3 * tail
        size += (7 - (pos + size)) % 16                 # total % 16 == 7
        msgs += fill(t, size)
    return pack(msgs, lead)


def rand_i32(g):
    """an int32 of any varint width, negatives (ten bytes) included"""
    r = g.random()
    if r < 0.1:
        return int(g.integers(-(1 << 31), 0))
    return int(g.integers(0, 1 << int(g.integers(1, 32))))


def rand_bytes(g, lo, hi):
    return bytes(g.integers(0, 256, size=int(g.integers(lo, hi)), dtype=np.uint8))


# -- messages of each decoder (every one well formed, each under 90 bytes so that a CTA fits 24 575 bytes)
def inbound_message(inbound):
    """make(g) of ProxyLeaderInbound / AcceptorInbound (0, 1) and their Mencius forms (2, 3)"""
    def p2a(g):
        return fint(1, rand_i32(g)) + fint(2, rand_i32(g)) + fbytes(3, rand_bytes(g, 0, 24))

    def ints(g, k):
        return b"".join(fint(f, rand_i32(g)) for f in range(1, k + 1))

    def make(g):
        if inbound == 0:
            return fbytes(1, p2a(g)) if g.random() < 0.5 else fbytes(2, ints(g, 4))
        if inbound == 1:
            return fbytes(2, p2a(g)) if g.random() < 0.6 else fbytes(int(g.choice((1, 3, 4))), rand_bytes(g, 0, 20))
        which = int(g.integers(1, 6 if inbound == 2 else 4))
        if which == 1:
            return fbytes(1, rand_bytes(g, 0, 20))                        # a member carried opaque
        if which == 2:
            return fbytes(2, p2a(g))
        if which == 3:
            return fbytes(3, ints(g, 3))
        if which == 4:
            return fbytes(4, ints(g, 3))
        return fbytes(5, fint(1, int(g.integers(0, 4))) + fint(2, int(g.integers(0, 4))) +
                      fint(3, rand_i32(g)) + fint(4, rand_i32(g)) + fint(5, rand_i32(g)))
    return make


def vm_message(g):
    """a vanilla Mencius ServerInbound of any member"""
    which = int(g.integers(1, 10))
    ints = lambda k: b"".join(fint(f, rand_i32(g)) for f in range(1, k + 1))   # noqa: E731
    value = lambda: fbytes(2, b"") if g.random() < 0.2 else fbytes(1, rand_bytes(g, 0, 20))   # noqa: E731
    if which == 1:
        return fbytes(1, fbytes(1, rand_bytes(g, 0, 20)))
    if which == 4:
        return fbytes(4, ints(3) + fbytes(4, value()))
    if which in (5, 6):
        return fbytes(which, ints(3))
    if which == 7:
        return fbytes(7, ints(1) + fbytes(2, value()) + fint(3, int(g.integers(0, 2))))
    if which == 9:
        return fbytes(9, ints(2))
    return fbytes(which, rand_bytes(g, 0, 20))


def ep_message(G, n):
    """make(g) of a random EPaxos ReplicaInbound of at most 90 bytes over n replicas"""
    import wire_ep_oracle as W

    def make(g):
        while True:
            raw = W.random_message(G, g, n).SerializeToString()
            if len(raw) <= 90:
                return raw
    return make


def command(g):
    """a MultiPaxos Command {command_id {client_address, client_pseudonym, client_id}, command}"""
    cid = fbytes(1, rand_bytes(g, 0, 6)) + fint(2, rand_i32(g)) + fint(3, rand_i32(g))
    return fbytes(1, cid) + fbytes(2, rand_bytes(g, 0, 6))


def replica_message(kinds):
    """make(g) of a MultiPaxos ReplicaInbound whose member is drawn from `kinds` (0: no member)"""
    def make(g):
        k = int(g.choice(kinds))
        if k == 0:
            return b""
        if k == 1:
            return fbytes(1, fint(1, rand_i32(g)) + fbytes(2, rand_bytes(g, 0, 24)))
        if k in (2, 3):
            return fbytes(k, fint(1, rand_i32(g)) + fbytes(2, command(g)))
        if k == 4:
            return fbytes(4, fbytes(1, command(g)))
        cmds = b"".join(fbytes(2 if k != 7 else 1, command(g)) for _ in range(int(g.integers(0, 3))))
        return fbytes(k, (fint(1, rand_i32(g)) if k != 7 else b"") + cmds)
    return make


def reads_message(batcher):
    """make(g) of a ClientInbound (batcher False) or ReadBatcherInbound"""
    def make(g):
        which = int(g.integers(1, 5 if batcher else 6))
        if which != 4:
            return fbytes(which, rand_bytes(g, 0, 20))                     # not parsed: any body
        if batcher:
            return fbytes(4, b"".join(fint(f, rand_i32(g)) for f in range(1, 5)))
        cid = fbytes(1, rand_bytes(g, 0, 6)) + fint(2, rand_i32(g)) + fint(3, rand_i32(g))
        return fbytes(4, fbytes(1, cid) + fint(2, int(g.integers(0, 4))) + fint(3, int(g.integers(0, 4))) +
                      fint(4, rand_i32(g)))
    return make


def split_batch(g, staged):
    """A ReplicaInbound batch of edge CTAs whose first Chosen, followed by a read, falls in the middle of a staged
    (staged True) or unstaged CTA; every message before it is a read or carries no member. -> (buf, offs, index)"""
    spans = (STAGE, STAGE + 1, STAGE - 1)
    k = 0 if staged else 1
    at = k * CTA + 100
    i = [0]
    reads, chosen = replica_message((0, 2, 3, 4, 5, 6, 7)), replica_message((1,))

    def make(g):
        j = i[0]
        i[0] += 1
        return chosen(g) if j == at else reads(g) if j != at + 1 else replica_message((2,))(g)
    buf, offs = stage_batch(make, g, spans=spans)
    return buf, offs, at


def value_arena(lens, g):
    """values of the given lengths back to back -> (arena, value_offsets)"""
    vals = [bytes(g.integers(0, 256, size=n, dtype=np.uint8)) for n in lens]
    offs = np.zeros(len(vals) + 1, dtype=np.int32)
    offs[1:] = np.cumsum([len(v) for v in vals])
    return np.frombuffer(b"".join(vals) + bytes(16), dtype=np.uint8)[:offs[-1]].copy(), offs


def body_len_widths(out, offs):
    """widths of the body-length varints (after the one-byte outer tag) of the non-empty encoded messages"""
    widths = set()
    for i in range(len(offs) - 1):
        lo, hi = int(offs[i]), int(offs[i + 1])
        if hi > lo:
            w = 1
            while out[lo + w] & 0x80:
                w += 1
            widths.add(w)
    return widths


def window_batch(msgs):
    """msgs laid out for a decoder so that each is parsed from a staged CTA when it fits the window and again from
    an unstaged one: CTAs of at most STAGE - 15 bytes (staged wherever lo falls) padded to 256 messages with
    zero-length ones, then all of msgs (<= 256, one over the window) in one CTA.
    -> (buf, offs, src): src[j] = the index in msgs of batch message j, -1 for a zero-length filler"""
    assert len(msgs) <= CTA and sum(len(m) for m in msgs) > STAGE
    groups, cur, size = [], [], 0
    for k, m in enumerate(msgs):
        if len(m) > STAGE - 15:
            continue
        if size + len(m) > STAGE - 15:
            groups.append(cur)
            cur, size = [], 0
        cur.append(k)
        size += len(m)
    groups.append(cur)
    src = []
    for grp in groups:
        src += grp + [-1] * (CTA - len(grp))
    src += list(range(len(msgs)))
    buf, offs = pack([msgs[k] if k >= 0 else b"" for k in src])
    return buf, offs, np.array(src)


def body_width(msg):
    """bytes of the body-length varint after a one-byte outer tag"""
    w = 1
    while msg[w] & 0x80:
        w += 1
    return w
