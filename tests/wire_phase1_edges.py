"""Batch builders of the Phase 1 wire paths' edge tests (tests/test_wire_phase1_edges_*.py).  TEST INFRASTRUCTURE.

The leader's walk (p1_walk_kernel) stages a message P1_WINDOW bytes at a time from `lo & ~15` and restages when a
field header (a tag and a varint: at most HEADER_MAX bytes) may cross the window's end; these builders put a chosen
header at a chosen distance from that end, in canonical or padded varints.  The other builders make the oneof
sequences the walk merges or resets, batches of minimal 8-byte infos packed as tightly as protobuf allows, and
Phase1bs whose entry counts, slots and row counts sit on the per-entry passes' grid strides.  The constants mirror
the kernels'; tests/test_wire_phase1_edges_oracle.py reads them back from the sources."""
import numpy as np

from wire_mencius_phase1_cases import VALUES as VALUE_BYTES
from wire_edges import ENC_TILE, PAD_FIELD, SCAN_CHUNK, VALUE_LENS, body_len_widths, fbytes, fint, pack, venc  # noqa: F401

# -- fpx_wire_phase1.cuh / fpx_engine_wire_phase1.inc
P1_WINDOW = 16 * 1024       # kP1Window: bytes of a message staged per step of the walk
P1_THREADS = 256            # kP1Threads
P1_MIN_INFO = 8             # kP1MinInfo: bytes of the smallest info field; one entry per 8 bytes of the batch
HEADER_MAX = 20             # the walk restages when fewer bytes than this are left in the window
PARSE_CTAS = 1024           # p1_parse / p1_max / p1_first: grid (1024, min(n, 65535))
GRID_Y = 65535
PARSE_STRIDE = PARSE_CTAS * P1_THREADS          # 262 144 entries per grid-stride step of one message
EMIT_CTAS = 4096            # p1_emit: at most 4096 CTAs
EMIT_STRIDE = EMIT_CTAS * P1_THREADS            # 2^20 rows per grid-stride step
P1A_TILE = 1024             # kP1aTile: slots per p1a_count / p1a_fill CTA
P1A_MAX_N = 65535           # the acceptor call's record limit (gridDim.y of count and fill)
# -- fpx_vm_revoke.cuh
VM_P1A_THREADS = 256        # kVmP1aThreads: slots per chunk of vm_p1a_apply's walk
# the boundary values
PARSE_EDGES = (PARSE_STRIDE - 1, PARSE_STRIDE, PARSE_STRIDE + 1)
EMIT_EDGES = (EMIT_STRIDE - 1, EMIT_STRIDE, EMIT_STRIDE + 1)
SCAN_EDGES = (SCAN_CHUNK - 1, SCAN_CHUNK, SCAN_CHUNK + 1)
BIG_P2A = SCAN_CHUNK * ENC_TILE + ENC_TILE + 1  # Phase2a records past the encoder's first scan chunk
# a header starting d bytes before the window's end, d = P1_WINDOW - (offset from lo & ~15): every byte of a
# 20-byte header on either side of the end, and headers wholly inside or wholly past it
WINDOW_DISTANCES = (-3, 0, 1, 2, 5, 9, 10, 11, 15, 19, 20, 21, 22, 40)
INT_MIN, INT_MAX = -(1 << 31), (1 << 31) - 1
NOOP = -(1 << 31)           # FPX_VALUE_NOOP
# include/fpx.h's statuses the edges meet
ERR_INVALID_ARG, ERR_BAD_ACCEPTOR, ERR_SLOT_RANGE, ERR_CHECK_FAILED, ERR_WIRE = -1, -5, -6, -14, -15
EMPTY_VALUE = b""           # a vote_value of no bytes: the smallest info
VALUES = tuple(VALUE_BYTES)  # canonical CommandBatchOrNoops: Noop, an empty batch, one command


def pvenc(v, width):
    """v as a varint of exactly `width` bytes: the canonical bytes with continuation bits and zero 7-bit groups
    appended (protobuf decoders accept this; the protobuf runtime accepts tags of up to 5 bytes).  None: canonical."""
    b = bytearray(venc(v))
    width = width or len(b)
    assert len(b) <= width <= 10, (v, width)
    while len(b) < width:
        b[-1] |= 0x80
        b.append(0)
    return bytes(b)


def read_varint(b, p):
    """-> (value, position after it), 64-bit"""
    v, s = 0, 0
    while True:
        c = b[p]
        p += 1
        v |= (c & 0x7f) << s
        s += 7
        if not c & 0x80:
            return v, p


def info_body(slot, vote_round, value):
    return fint(1, slot) + fint(2, vote_round) + fbytes(3, value)


def field(f, body, tag_w=1, len_w=None):
    """a length-delimited field with its tag and length padded to tag_w / len_w bytes"""
    return pvenc(f << 3 | 2, tag_w) + pvenc(len(body), len_w or len(venc(len(body)))) + bytes(body)


def info(slot, vote_round, value, tag_w=1, len_w=None):
    return field(4, info_body(slot, vote_round, value), tag_w, len_w)


def scalars(group, acceptor, round_):
    return fint(1, group) + fint(2, acceptor) + fint(3, round_)


def pad_field(size):
    """an unknown field (PAD_FIELD) of exactly `size` >= 2 bytes, or two when one cannot take that size"""
    for p in range(size - 2, -1, -1):
        if 1 + len(venc(p)) + p == size:
            return fbytes(PAD_FIELD, bytes(p))
    return fbytes(PAD_FIELD, b"") + pad_field(size - 2)


def phase1b(group, acceptor, round_, infos, member=1):
    """LeaderInbound{phase1b {group_index, acceptor_index, round, info...}} (member 1), infos [(slot, vr, value)]"""
    return field(member, scalars(group, acceptor, round_) + b"".join(info(*x) for x in infos))


def tail_to(pos, mod=7):
    """a message that belongs to no member (an unknown field only) ending the batch at total % 16 == mod"""
    return pad_field(2 + (mod - (pos + 2)) % 16)


# --------------------------------------------------------------------------- the walk's window end
def window_message(lo, d, target, tag_w, len_w, group, acceptor, round_, infos_before, target_info, infos_after):
    """A LeaderInbound starting at buffer offset lo whose `target` header starts d bytes before the end of the walk's
    first window, (lo & ~15) + P1_WINDOW:
      'info'    the header of info target_info (tag padded to tag_w bytes, length to len_w);
      'scalar'  the Phase1b's round (tag to tag_w bytes, the value to len_w), after every info but the later ones;
      'member'  a second phase1b member (tag to tag_w, length to len_w) that merges target_info and infos_after.
    An unknown field before the target positions it.  -> (message bytes, target offset from lo, target header)"""
    want = (lo & ~15) + P1_WINDOW - d - lo                  # the target's offset within the message
    pre = fint(1, group) + fint(2, acceptor) + (b"" if target == "scalar" else fint(3, round_))
    pre += b"".join(info(*x) for x in infos_before)
    after = b"".join(info(*x) for x in infos_after)
    if target == "member":
        head = pvenc(0x0a, tag_w) + pvenc(len(info(*target_info)) + len(after), len_w)
        tgt = head + info(*target_info) + after
        body1 = pre + pad_field(want - 4 - len(pre))        # member 1's tag and a 3-byte length, then pre and pad
        msg = field(1, body1, len_w=3) + tgt
    else:
        if target == "info":
            head = pvenc(0x22, tag_w) + pvenc(len(info_body(*target_info)), len_w)
            tgt = head + info_body(*target_info)
            rest = after + fint(3, round_)
        else:
            head = pvenc(0x18, tag_w) + pvenc(round_, len_w)
            tgt = head
            rest = info(*target_info) + after
        body = pre + pad_field(want - 4 - len(pre)) + tgt + rest
        msg = field(1, body, len_w=3)
    assert msg[want: want + len(head)] == head, (d, target)
    return msg, want, head


def window_batch(d, target, tag_w, len_w, lead, g, round_=9):
    """[an empty Phase1b of acceptor 1, the window-edge message of acceptor 0, a tail to total % 16 == 7] after
    `lead` bytes; the edge message completes the quorum of one group of three.  -> (buf, offs, edge index, target
    position in buf, header, infos [(slot, vr, value)] the edge message carries in order)"""
    def infos(k, base):
        return [(int(base + i), int(g.integers(0, round_)), VALUES[int(g.integers(0, len(VALUES)))]) for i in range(k)]
    before, after = infos(3, 0), infos(12, 10)
    tgt = infos(1, 5)[0]
    first = phase1b(0, 1, round_, [])
    lo = lead + len(first)
    msg, off, head = window_message(lo, d, target, tag_w, len_w, 0, 0, round_, before, tgt, after)
    msgs = [first, msg, tail_to(lo + len(msg))]
    buf, offs = pack(msgs, lead)
    return buf, offs, 1, lo + off, head, before + [tgt] + after


# --------------------------------------------------------------------------- the walk's oneof handling
def oneof_cases(round_=9, nack=6):
    """{name: (the message of acceptor 0, its expected Phase1b: (group, acceptor, round, infos) or None when it is not
    a Phase1b, or 'bad' when it fails to parse)}.  nack: LeaderInbound's nack member (MultiPaxos 6, Mencius 7)."""
    A = [(0, 3, VALUES[1]), (2, 4, VALUES[2])]
    B = [(1, 5, VALUES[0]), (3, 1, b"")]
    short = field(4, fint(1, 7) + fint(2, 1))                       # a 4-byte info: no vote_value
    S = scalars(0, 0, round_)
    inf = lambda xs: b"".join(info(*x) for x in xs)                 # noqa: E731
    nk = field(nack, fint(1, round_ + 3))
    return {
        "merge": (field(1, S + inf(A)) + field(1, inf(B)), (0, 0, round_, A + B)),
        "merge_scalars_last_win": (field(1, scalars(0, 2, round_ - 4) + inf(A)) + field(1, fint(2, 0) + fint(3, round_)
                                   + inf(B)), (0, 0, round_, A + B)),
        "merge_required_split": (field(1, fint(1, 0) + inf(A)) + field(1, fint(2, 0)) + field(1, fint(3, round_) + inf(B)),
                                 (0, 0, round_, A + B)),
        "reset_by_nack": (field(1, S + inf(A)) + nk + field(1, S + inf(B)), (0, 0, round_, B)),
        "reset_loses_scalars": (field(1, S + inf(A)) + nk + field(1, inf(B)), "bad"),
        "replaced_by_nack": (field(1, S + inf(A)) + nk, None),
        "scalars_after_infos": (field(1, inf(A) + fint(3, round_) + fint(2, 0) + fint(1, 0)), (0, 0, round_, A)),
        "scalars_between_infos": (field(1, inf(A[:1]) + S + inf(A[1:])), (0, 0, round_, A)),
        "short_info": (field(1, S + short + inf(A)), "bad"),
        "empty_info": (field(1, S + field(4, b"") + inf(A)), "bad"),
        "short_info_reset": (field(1, S + short) + nk + field(1, S + inf(B)), (0, 0, round_, B)),
        "short_info_merged": (field(1, S + short) + field(1, inf(B)), "bad"),
        "unknown_fields": (field(1, S + bytes([0x29]) + bytes(8) + inf(A) + bytes([0x35]) + bytes(4) + fint(9, 1 << 40))
                           + fint(12, 3) + bytes([0x6d]) + bytes(4), (0, 0, round_, A)),
    }


def oneof_batch(msg, round_=9):
    """the oneof message of acceptor 0 after an empty Phase1b of acceptor 1, 33 bytes in (lo % 16 == 1)"""
    return pack([phase1b(0, 1, round_, []), msg], 33)


# --------------------------------------------------------------------------- tight 8-byte infos
def tight_message(group, acceptor, round_, slots, vote_rounds):
    """a Phase1b made only of minimal 8-byte infos (one-byte slot and vote_round, an empty vote_value)"""
    assert all(0 <= s < 128 for s in slots) and all(0 <= r < 128 for r in vote_rounds)
    return phase1b(group, acceptor, round_, [(s, r, EMPTY_VALUE) for s, r in zip(slots, vote_rounds)])


def tight_batch(lead, g, round_=9, per_group=5, quorum=3):
    """Messages of minimal infos back to back after `lead` bytes, held and stale ones alternating, whose starts take
    every offs[m] % 8: the layout where one message's entries could run into the next one's.  The last held
    message completes the quorum.  -> (buf, offs)"""
    msgs, held = [], 0
    k = 0
    while held < quorum:
        stale = k % 2 == 0
        n_info = int(g.integers(1, 15)) + 16 * int(g.integers(0, 2))
        slots = np.sort(g.choice(120, size=n_info, replace=False))
        vr = g.integers(0, round_, size=n_info)
        if stale:
            msgs.append(tight_message(0, per_group - 1, round_ - 1, slots, vr))
        else:
            msgs.append(tight_message(0, held, round_, slots, vr))
            held += 1
        k += 1
    buf, offs = pack(msgs, lead)
    return buf, offs


# --------------------------------------------------------------------------- grid strides
def many_infos(acceptor, round_, slots, g, n_values=64):
    """one Phase1b of acceptor (group 0) with one info per slot, values one of n_values short byte strings"""
    vals = [bytes(g.integers(0, 256, int(k), np.uint8)) for k in g.integers(0, 12, n_values)]
    vr = g.integers(0, round_, size=len(slots))
    pick = g.integers(0, n_values, size=len(slots))
    body = bytearray(scalars(0, acceptor, round_))
    for s, r, p in zip(slots.tolist(), vr.tolist(), pick.tolist()):
        body += info(s, r, vals[p])
    return field(1, bytes(body))


def emit_batch(count, cw, round_=9):
    """Phase1bs of acceptors 0 and 1 (group 0) whose infos put max_slot at cw + count - 1: count rows to emit, a
    few of them voted (at the stride edges)."""
    top = cw + count - 1
    marks = sorted({cw, cw + 1, cw + EMIT_STRIDE - 1, cw + EMIT_STRIDE, top} & set(range(cw, top + 1)))
    a = phase1b(0, 0, round_, [(s, 1, bytes([s & 0xff])) for s in marks])
    b = phase1b(0, 1, round_, [(s, 2, bytes([1, s & 0xff])) for s in marks[::2]])
    return pack([a, b], 5)


def p2a_chunk_batch(count, round_=9):
    """two Phase1bs whose max_slot is count - 1 (chosen_watermark 0): count Phase2a records to encode"""
    return emit_batch(count, 0, round_)


# --------------------------------------------------------------------------- Phase1b bodies of each varint width
def phase1b_value_len(body, group, acceptor, round_, slot, vote_round):
    """the value length that makes an acceptor's Phase1b of one info {slot, vote_round, value} `body` bytes long"""
    head = 3 + len(venc(group)) + len(venc(acceptor)) + len(venc(round_ & 0xffffffffffffffff if round_ < 0 else round_))
    for vlen in range(max(0, body - head - 40), body):
        ib = 2 + len(venc(slot)) + len(venc(vote_round)) + 1 + len(venc(vlen)) + vlen
        if head + 1 + len(venc(ib)) + ib == body:
            return vlen
    return None


def vm_phase1b_value_len(body, server, round_, start, stop, slot, vote_round):
    """the value length that makes a vanilla Mencius Phase1b of one pending info `body` bytes long"""
    head = 4 + sum(len(venc(x)) for x in (server, round_, start, stop))
    for vlen in range(max(0, body - head - 40), body):
        inner = 1 + len(venc(vote_round)) + 1 + len(venc(vlen)) + vlen
        ib = 1 + len(venc(slot)) + 1 + len(venc(inner)) + inner
        if head + 1 + len(venc(ib)) + ib == body:
            return vlen
    return None


BODY_EDGES = (127, 128, 16383, 16384, (1 << 21) - 1, 1 << 21)
ROUND_EDGES = (0, 127, 128, 16383, 16384, (1 << 21) - 1, 1 << 21, (1 << 28) - 1, 1 << 28, INT_MAX)


def width_of(n):
    return len(venc(n))


# --------------------------------------------------------------------------- the reference's fill-in
def python_fill_in(msgs, parse, groups, per_group, f, round_, cw, lgroups=1, leader_group=0, recover_slot=None):
    """Leader.handlePhase1b (MultiPaxos, or Mencius with lgroups > 1 / recover_slot) over Phase1bs parsed by
    `parse(raw) -> (kind, group, acceptor, round, [(slot, vote_round, value bytes)])` (kind 'bad' on a parse error):
    (status, index, None) or (0, complete, (max_slot, next_slot, [(slot, value or None)]))."""
    held = [dict() for _ in range(groups)]
    for i, raw in enumerate(msgs):
        kind, grp, acc, rnd, infos = parse(raw)
        if kind == "bad":
            return -15, i, None
        if kind != 1:
            continue
        if rnd != round_:
            if rnd > round_:
                return -14, i, None
            continue
        if not (0 <= grp < groups and 0 <= acc < per_group):
            return -5, i, None
        held[grp][acc] = infos
        if not all(len(h) >= f + 1 for h in held):
            continue
        mx = max(max((s for s, _, _ in p), default=-1) for h in held for p in h.values())
        if recover_slot is not None:
            mx = max(mx, recover_slot)
            if mx != -1 and mx % lgroups != leader_group:
                return -14, i, None
        nxt = None
        if recover_slot is not None:
            nxt = leader_group if mx < 0 else (lgroups * (mx // lgroups) + leader_group +
                                                (lgroups if lgroups * (mx // lgroups) + leader_group <= mx else 0))
            if nxt > INT_MAX:
                return -6, i, None
        s0 = cw + (leader_group - cw % lgroups) % lgroups
        out = []
        for s in range(s0, mx + 1, lgroups):
            best = None
            for a in sorted(held[(s // lgroups) % groups]):
                x = next((x for x in held[(s // lgroups) % groups][a] if x[0] == s), None)
                if x is not None and (best is None or x[1] > best[1]):
                    best = x
            out.append((s, None if best is None else best[2]))
        return 0, i, (mx, nxt, out)
    return 0, -1, None


# --------------------------------------------------------------------------- slots at the int32 edges
def mp_slot_cases(round_=9):
    """{name: (msgs, chosen_watermark)} for one MultiPaxos group of three: negative and INT_MIN info slots (ten-byte
    varints), max_slot = INT_MAX, a watermark at INT_MAX"""
    v = lambda s: (s, 1 + (s & 3), VALUES[s % 3])                 # noqa: E731
    two = lambda a, b: [phase1b(0, 0, round_, [v(s) for s in a]), phase1b(0, 2, round_, [v(s) for s in b])]   # noqa: E731
    return {
        "negative_slots": (two([-1, -5, INT_MIN, 3], [2, -7]), 0),
        "only_int_min": (two([INT_MIN], [INT_MIN, INT_MIN]), 0),
        "int_min_and_empty": (two([INT_MIN], []), 0),
        "max_slot_int32_max": (two([INT_MAX, INT_MAX - 2], [INT_MAX - 1, INT_MAX]), INT_MAX - 3),
        "watermark_int32_max": (two([INT_MAX], [-1]), INT_MAX),
        "watermark_past_max_slot": (two([INT_MAX - 1], [5]), INT_MAX),
    }


MENCIUS_SHAPE = (1, 3, 2, 3)
# the cases of mencius_slot_cases() that are refused: a next_slot past INT32_MAX (DESIGN §7), a max_slot the leader
# group does not own (logger.check)
MENCIUS_SLOT_STATUS = {"next_slot_past_int32": ERR_SLOT_RANGE, "recover_next_slot_past_int32": ERR_SLOT_RANGE,
                       "s0_past_int32_votes": ERR_SLOT_RANGE, "recover_of_another_group": ERR_CHECK_FAILED,
                       "info_of_another_group_above": ERR_CHECK_FAILED}      # f, LG, AG, acceptors per group


def mencius_batch(slots, round_=9, lgroups=3, agroups=2, everywhere=False):
    """f + 1 = 2 Phase1bs in each acceptor group; each carries the given slots its group serves ((s / LG) % AG,
    negative slots in group 0), with vote rounds that differ by acceptor.  everywhere: every Phase1b carries every
    slot, and a group's votes on the slots it does not serve have the higher rounds (safeValue must not read them)."""
    msgs = []
    for ag in range(agroups):
        for a in range(2):
            owner = lambda s: (s // lgroups if s >= 0 else 0) % agroups == ag    # noqa: E731
            mine = [s for s in slots if everywhere or owner(s)]
            msgs.append(phase1b(ag, a, round_, [(s, ((s + a) & 7) + (0 if owner(s) else 8), VALUES[(s + a + ag) % 3])
                                                for s in mine]))
    return msgs


def cross_group_mp(round_=9):
    """MultiPaxos with two groups of three: each group's f + 1 Phase1bs, where group 1's also report group 0's slots
    (s % 2 == 0) with higher vote rounds and other values, up to a max_slot only group 1 reports"""
    own0 = [(s, 1, VALUES[1]) for s in (0, 2, 4)]
    own1 = [(s, 1, VALUES[2]) for s in (1, 3, 5)]
    foreign = [(s, 7, VALUES[0]) for s in (0, 2, 4, 6)]
    return [phase1b(0, 0, round_, own0), phase1b(1, 2, round_, sorted(own1 + foreign)), phase1b(0, 1, round_, own0[1:]),
            phase1b(1, 0, round_, own1[:1] + foreign[:1])]


def mencius_slot_cases():
    """{name: (leader_group, chosen_watermark, recover_slot, msgs)} for LG = 3, AG = 2: s0 past int32, next_slot at
    INT_MAX (accepted) and one step past (FPX_ERR_SLOT_RANGE), recover_slot above every info or of another group"""
    top = INT_MAX                         # 2^31 - 1 = 3 * 715827882 + 1: leader group 1's slot
    return {
        "s0_past_int32": (2, top, -1, mencius_batch([])),
        "s0_past_int32_votes": (2, top, -1, mencius_batch([top - 2])),
        "next_slot_int32_max": (1, top - 9, -1, mencius_batch([top - 3, top - 6])),
        "next_slot_past_int32": (1, top - 9, -1, mencius_batch([top - 6, top])),
        "recover_next_slot_int32_max": (1, top - 9, top - 3, mencius_batch([top - 9])),
        "recover_next_slot_past_int32": (1, top - 9, top, mencius_batch([top - 9])),
        "recover_above_every_info": (0, 0, 30, mencius_batch([0, 3, 6, 9])),
        "recover_of_another_group": (0, 0, 31, mencius_batch([0, 3])),
        "negative_info_slots": (0, 0, -1, mencius_batch([-3, INT_MIN, 6, 12])),
        "info_of_another_group_above": (0, 0, -1, mencius_batch([0, 3, 10])),
        "infos_in_every_acceptor_group": (0, 0, -1, mencius_batch([0, 3, 6, 9, 12, 15], everywhere=True)),
    }
