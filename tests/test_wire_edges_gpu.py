"""The wire codecs at their edges against the CPU oracles: decoder CTAs at the shared-memory stage window (24 575,
24 576 and 24 577 bytes from lo & ~15, lo % 16 in {0, 1, 15}, leading bytes outside every message, a total that is
not a multiple of 16), encoders and the replica-inbound decoder past tile_offsets_kernel's first chunk of 4096
tiles, every encoder at out_capacity = total, total - 1 and 0 in its host and device forms, and values whose
lengths take every varint width."""
import ctypes as C
import itertools

import numpy as np
import pytest
import torch

import wire_edges as E
import wire_ep_oracle as W
import wire_reads_oracle as R
import wire_vm_oracle as V
from frankenpaxos_b200 import (CHOSEN, MENCIUS, NACK, P2A, P2A_RANGE, P2B, READ_SLOT, READS_CLIENT, READS_READ_BATCHER,
                               VANILLA_MENCIUS, Engine, FpxError, Reads)
from frankenpaxos_b200.epaxos import CALL_LEAD, CALL_PREACCEPT, CALL_PREACCEPTOK, CALL_PREPARE, EpaxosReplica
from frankenpaxos_b200.engine import VM_SKIP, VALUE_NOOP
from oracle import fpx_oracle_py as O

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
LG, AG = 3, 3                       # the Mencius engine's leader and acceptor groups
KEY_CAP = 1 << 10
EP_F, EP_N = 1, 3
INVALID_ARG, WIRE = -1, -15
SENTINEL = 0xA5


@pytest.fixture(scope="module")
def H():
    h = {"mp": Engine(1, 2, 3, slot_capacity=1 << 12, max_batch=1 << 12),
         "mencius": Engine(1, AG, 3, num_leaders=2, num_replicas=2, slot_capacity=1 << 12, max_batch=1 << 12,
                           protocol=MENCIUS, num_leader_groups=LG),
         "vm": Engine(1, 1, 3, slot_capacity=1 << 12, max_batch=1 << 12, protocol=VANILLA_MENCIUS),
         "ep": EpaxosReplica(EP_F, 0, 1 << 10, max_batch=1 << 12)}
    h["client"] = Reads(h["mp"], READS_CLIENT, key_capacity=KEY_CAP)
    h["batcher"] = Reads(h["mp"], READS_READ_BATCHER, key_capacity=KEY_CAP)
    yield h
    for k in ("client", "batcher", "mp", "mencius", "vm", "ep"):
        h[k].close()


@pytest.fixture(scope="module")
def G():
    return W.golden_module()


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).to(DEV)


def host(t, dtype):
    return t.cpu().numpy().view(dtype).reshape(-1)


def status_of(fn, *a):
    try:
        return (0, -1), fn(*a)
    except FpxError as e:
        return (e.status, e.index), None


def collect(handle):
    try:
        handle.sync()
        return 0, -1
    except FpxError as e:
        return e.status, e.index


# ---------------------------------------------------------------------------------------------------- decoders
# Each decoder: make (a message), oracle(buf, offs) -> ((status, index), outputs), host / device forms ->
# outputs, and spans(outputs) -> (message index, off, len) of every value span the outputs carry.
def _rec_spans(kinds):
    def spans(out):
        kind, rec = out[0], out[1].view(np.int32).reshape(-1, 4)
        i = np.flatnonzero(np.isin(kind, kinds))
        return i, rec[i, 2], rec[i, 3]
    return spans


def _inbound(inbound, key):
    def oracle(buf, offs):
        st, err, kind, rec = O.wire_decode_inbound(inbound, buf, offs, LG, AG)
        return (st, err), (kind, rec)

    def host_form(H, buf, offs):
        return H[key].wire_decode_inbound(inbound, buf, offs)

    def dev_form(H, d_buf, d_offs, n):
        kind, rec = torch.zeros(n, dtype=torch.int32, device=DEV), torch.zeros((n, 4), dtype=torch.int32, device=DEV)
        H[key].wire_decode_inbound_dev(inbound, d_buf.data_ptr(), d_offs.data_ptr(), n, kind.data_ptr(), rec.data_ptr())
        return collect(H[key]), (host(kind, np.int32), host(rec, np.int32))
    kinds = {0: (1,), 1: (1, 2, 3, 4), 2: (1, 2), 3: (1, 2)}[inbound]
    return E.inbound_message(inbound), oracle, host_form, dev_form, _rec_spans(kinds)


def _vm():
    def oracle(buf, offs):
        st, err, kind, rec, sender = V.decode(buf, offs)
        return (st, err), (kind, rec, sender)

    def host_form(H, buf, offs):
        return H["vm"].wire_decode_vm_server_inbound(buf, offs)

    def dev_form(H, d_buf, d_offs, n):
        kind, rec = torch.zeros(n, dtype=torch.int32, device=DEV), torch.zeros((n, 4), dtype=torch.int32, device=DEV)
        sender = torch.zeros(n, dtype=torch.int32, device=DEV)
        H["vm"].wire_decode_vm_server_inbound_dev(d_buf.data_ptr(), d_offs.data_ptr(), n, kind.data_ptr(),
                                                  rec.data_ptr(), sender.data_ptr())
        return collect(H["vm"]), (host(kind, np.int32), host(rec, np.int32), host(sender, np.int32))
    return E.vm_message, oracle, host_form, dev_form, _rec_spans((1, 2, 3, 4, 7, 8))


def _ep(G):
    def oracle(buf, offs):
        st, err, kind, rows, values = W.decode(buf, offs, EP_N, 7)
        return (st, err), (kind, rows, values)

    def host_form(H, buf, offs):
        return H["ep"].wire_decode(buf, offs, 7)

    def dev_form(H, d_buf, d_offs, n):
        kind = torch.zeros(n, dtype=torch.int32, device=DEV)
        rows = torch.zeros((n, 12 + EP_N), dtype=torch.int32, device=DEV)
        values = torch.zeros((n, 2), dtype=torch.int32, device=DEV)
        H["ep"].wire_decode_dev(d_buf.data_ptr(), d_offs.data_ptr(), n, 7, kind.data_ptr(), rows.data_ptr(),
                                values.data_ptr())
        return collect(H["ep"]), (host(kind, np.int32), host(rows, np.int32), host(values, np.int32))

    def spans(out):
        i = np.flatnonzero(out[1][:, W.VALUE] != -1)
        return i, out[2][i, 0], out[2][i, 1]
    return E.ep_message(G, EP_N), oracle, host_form, dev_form, spans


def _replica(kinds):
    def oracle(buf, offs):
        st, err, *rest = R.decode_replica(buf, offs, 11, 3)
        return (st, err), tuple(rest)

    def host_form(H, buf, offs):
        return H["mp"].wire_decode_replica_inbound(buf, offs, 11, 3)

    def dev_form(H, d_buf, d_offs, n):
        cap = n * 2 + 1
        kind = torch.zeros(n, dtype=torch.int32, device=DEV)
        chosen, cvals = torch.zeros((n, 2), dtype=torch.int32, device=DEV), torch.zeros((n, 2), dtype=torch.int32, device=DEV)
        reads, rcmds = torch.zeros((cap, 2), dtype=torch.int32, device=DEV), torch.zeros((cap, 2), dtype=torch.int32, device=DEV)
        counts = torch.zeros(3, dtype=torch.int32, device=DEV)
        H["mp"].wire_decode_replica_inbound_dev(d_buf.data_ptr(), d_offs.data_ptr(), n, 11, 3, cap, kind.data_ptr(),
                                                chosen.data_ptr(), cvals.data_ptr(), reads.data_ptr(), rcmds.data_ptr(),
                                                counts.data_ptr())
        st = collect(H["mp"])
        nc, nr, split = (int(x) for x in counts.cpu().numpy())
        return st, (host(kind, np.int32), host(chosen, np.int32)[:2 * nc], host(cvals, np.int32)[:2 * nc],
                    host(reads, np.int32)[:2 * nr], host(rcmds, np.int32)[:2 * nr], split)
    return E.replica_message(kinds), oracle, host_form, dev_form, None


def _reads(key):
    batcher = key == "batcher"

    def oracle(buf, offs):
        st, err, *rest = R.decode_reads(buf, offs, batcher, KEY_CAP)
        return (st, err), tuple(rest)

    def host_form(H, buf, offs):
        return H[key].wire_decode(buf, offs)

    def dev_form(H, d_buf, d_offs, n):
        kind, out = torch.zeros(n, dtype=torch.int32, device=DEV), torch.zeros((n, 4), dtype=torch.int32, device=DEV)
        spans = torch.zeros((n, 2), dtype=torch.int32, device=DEV)
        H[key].wire_decode_dev(d_buf.data_ptr(), d_offs.data_ptr(), n, kind.data_ptr(), out.data_ptr(), spans.data_ptr())
        return collect(H[key]), (host(kind, np.int32), host(out, np.int32), host(spans, np.int32))

    def spans(out):
        i = np.flatnonzero(out[0] != 0)
        return i, out[2][i, 0], out[2][i, 1]
    return E.reads_message(batcher), oracle, host_form, dev_form, spans


DECODERS = ["inbound0", "inbound1", "mencius2", "mencius3", "vm", "ep", "replica_reads", "replica_chosen", "client",
            "batcher"]


def decoder(name, G):
    if name.startswith("inbound"):
        return _inbound(int(name[-1]), "mp")
    if name.startswith("mencius"):
        return _inbound(int(name[-1]), "mencius")
    if name == "vm":
        return _vm()
    if name == "ep":
        return _ep(G)
    if name.startswith("replica"):
        return _replica((0, 2, 3, 4, 5, 6, 7) if name == "replica_reads" else (0, 1))
    return _reads(name)


def replica_spans(out, offs, buf):
    """(message index, off, len) of the replica decode's Chosen values and read Commands"""
    kind, chosen, cvals, reads, rcmds = out[:5]
    cv, rc = np.asarray(cvals).reshape(-1, 2), np.asarray(rcmds).reshape(-1, 2)
    ci = np.asarray(chosen).view(np.int32).reshape(-1, 2)[:, 1] - 11
    ri = np.searchsorted(offs, rc[:, 0], side="right") - 1
    return np.concatenate([ci, ri]), np.concatenate([cv[:, 0], rc[:, 0]]), np.concatenate([cv[:, 1], rc[:, 1]])


def same(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        if isinstance(x, (int, np.integer)):
            assert int(x) == int(y)
        else:
            assert np.array_equal(np.asarray(x).view(np.int32).reshape(-1), np.asarray(y).view(np.int32).reshape(-1))


def decode_everywhere(H, dec, buf, offs):
    """host form, device form from a buffer of exactly offsets[n] bytes, and the oracle agree -> oracle's result"""
    _, oracle, host_form, dev_form, _ = dec
    ost, oout = oracle(buf, offs)
    st, out = status_of(host_form, H, buf, offs)
    assert st == ost
    total, n = int(offs[-1]), len(offs) - 1
    dst, dout = dev_form(H, dev(buf[:total]), dev(offs), n)
    assert dst == ost
    if ost[0] == 0:
        same(out, oout)
        same(dout, oout)
    return ost, oout


@pytest.mark.parametrize("name", DECODERS)
def test_stage_window_edges(H, G, name):
    """Every decoder on CTAs of 24 575 / 24 576 / 24 577 bytes at every lo % 16 of {0, 1, 15}: the results, and the
    value spans of staged and unstaged CTAs alike, are the oracle's, from the host and the device form."""
    dec = decoder(name, G)
    g = np.random.Generator(np.random.PCG64(sum(map(ord, name))))
    buf, offs = E.stage_batch(dec[0], g)
    ctas = E.cta_spans(offs)
    assert offs[0] > 0 and offs[-1] % 16 != 0
    assert {(s, lo % 16) for lo, _, s, _ in ctas[:len(E.SPAN_ORDER)]} == \
        {(s, m) for s in E.EDGE_SPANS for m in (0, 1, 15)}
    assert {st for *_, st in ctas} == {True, False} and ctas[-1][3]          # the batch ends in a staged CTA
    (st, _), out = decode_everywhere(H, dec, buf, offs)
    assert st == 0
    i, off, ln = replica_spans(out, offs, buf) if dec[4] is None else dec[4](out)
    assert ((offs[i] <= off) & (off + ln <= offs[i + 1])).all()               # inside its own message
    staged = np.array([c[3] for c in ctas])[i // E.CTA]
    assert staged.any() and (~staged).any()                                   # spans in both kinds of CTA
    for k in np.flatnonzero(ln > 0)[::7]:
        assert bytes(buf[off[k]:off[k] + ln[k]]) in bytes(buf[offs[i[k]]:offs[i[k] + 1]])


@pytest.mark.parametrize("name", DECODERS)
@pytest.mark.parametrize("cut", [2, 3, 4])
def test_truncated_last_message_of_a_cta_ending_the_batch(H, G, name, cut):
    """The batch ends with a staged CTA of 24 576 bytes (ending on a 16-byte boundary) or 24 575 bytes (ending inside
    a 16-byte chunk, which the stage copies byte by byte), or an unstaged one of 24 577 bytes, whose last message is
    cut short: the oracle's error and index, host and device forms."""
    dec = decoder(name, G)
    g = np.random.Generator(np.random.PCG64(cut))
    buf, offs = E.stage_batch(dec[0], g, cut=cut)
    lo, hi, span, staged = E.cta_spans(offs)[-1]
    assert hi == offs[-1] and span == E.SPAN_ORDER[cut] and staged == (span <= E.STAGE)
    assert (hi % 16 == 0) == (cut == 2)            # cut 3: a staged CTA ending inside a 16-byte chunk
    (st, idx), _ = decode_everywhere(H, dec, buf, offs)
    assert (st, idx) == (WIRE, len(offs) - 2)


@pytest.mark.parametrize("staged", [True, False])
def test_replica_split_inside_an_edge_cta(H, staged):
    dec = _replica(())
    buf, offs, at = E.split_batch(np.random.Generator(np.random.PCG64(staged)), staged)
    assert E.cta_spans(offs)[at // E.CTA][3] == staged
    (st, _), out = decode_everywhere(H, dec, buf, offs)
    assert st == 0 and out[5] == at + 1


# ------------------------------------------------------------------------------------ past the first scan chunk
def rand_i32(g, n):
    return (g.integers(-(1 << 31), 1 << 31, size=n) >> g.integers(0, 32, size=n)).astype(np.int32)


def short_values(g):
    return R.pack([bytes(g.integers(0, 256, size=k, dtype=np.uint8)) for k in range(6)])


@pytest.mark.parametrize("n", E.BIG_N)
def test_encoders_past_the_first_scan_chunk(H, n):
    assert -(-n // E.ENC_TILE) >= E.SCAN_CHUNK and (n == E.BIG_N[0] or -(-n // E.ENC_TILE) > E.SCAN_CHUNK)
    g = np.random.Generator(np.random.PCG64(n))
    arena, voffs = short_values(g)
    arena = arena[:voffs[-1]]
    vid = np.where(g.integers(0, 5, size=n) == 0, VALUE_NOOP, g.integers(0, 6, size=n)).astype(np.int32)
    p2b = np.zeros(n, dtype=P2B)
    for f in P2B.names:
        p2b[f] = rand_i32(g, n)
    # MultiPaxos and Mencius Phase2b, Nack (the small encoders: a CTA sums the tiles before it)
    out, offs = H["mp"].wire_encode_phase2b(p2b)
    oout, ooffs = O.wire_encode_phase2b(p2b)
    assert np.array_equal(offs, ooffs) and np.array_equal(out, oout)
    kind, rec = H["mp"].wire_decode_inbound(0, out, offs)
    assert (kind == 2).all() and np.array_equal(rec.view(np.int32), p2b.view(np.int32))
    out, offs = H["mencius"].wire_encode_phase2b(p2b)
    oout, ooffs = O.wire_encode_mencius_phase2b(p2b)
    assert np.array_equal(offs, ooffs) and np.array_equal(out, oout)
    nk = np.zeros(n, dtype=NACK); nk["round"] = p2b["round"]
    out, offs = H["mp"].wire_encode_nack(nk)
    oout, ooffs = O.wire_encode_nack(nk)
    assert np.array_equal(offs, ooffs) and np.array_equal(out, oout)
    sk = np.zeros(n, dtype=VM_SKIP); sk["server"], sk["slot_start"], sk["slot_stop"] = p2b["group"], p2b["slot"], p2b["round"]
    out, offs = H["vm"].wire_encode_vm_skip(sk)
    st, _, oout, ooffs = V.encode("skip", sk, servers=3)
    assert st == 0 and np.array_equal(offs, ooffs) and np.array_equal(out, oout)
    del sk, nk
    # MultiPaxos Chosen, decoded back by the replica
    ch = np.zeros(n, dtype=CHOSEN); ch["slot"] = p2b["slot"]; ch["value_id"] = np.where(vid < 0, 0, vid)
    out, offs = H["mp"].wire_encode_chosen(ch, arena, voffs)
    st, _, oout, ooffs = O.wire_encode_chosen(ch, arena, voffs)
    assert st == 0 and np.array_equal(offs, ooffs) and np.array_equal(out, oout)
    kind, chosen, cvals, reads, _, split = H["mp"].wire_decode_replica_inbound(out, offs, 0, 0, 0)
    assert (kind == 1).all() and split == n and len(reads) == 0
    assert np.array_equal(chosen["slot"], ch["slot"]) and np.array_equal(chosen["value_id"], np.arange(n))
    assert np.array_equal(cvals[:, 1], np.diff(voffs)[ch["value_id"]])
    del chosen, cvals, kind
    # the vanilla Mencius value-gathering encoders, decoded back
    reps = p2b.copy(); reps["group"] = g.integers(0, 4, size=n); reps["round"] = np.where(reps["group"] == 2, vid, reps["round"])
    pa = np.zeros(n, dtype=P2A); pa["slot"], pa["round"], pa["value_id"] = p2b["slot"], p2b["round"], vid
    vc = ch.copy(); vc["value_id"] = vid
    for what, fn, recs in (("replies", H["vm"].wire_encode_vm_replies, reps), ("chosen", H["vm"].wire_encode_vm_chosen, vc),
                           ("phase2a", H["vm"].wire_encode_vm_phase2a, pa)):
        out, offs = fn(recs, arena, voffs)
        st, _, oout, ooffs = V.encode(what, recs, arena, voffs, servers=3)
        assert st == 0 and np.array_equal(offs, ooffs) and np.array_equal(out, oout), what
        kind, rec, _ = H["vm"].wire_decode_vm_server_inbound(out, offs)
        st, _, okind, orec, _ = V.decode(out, offs)
        assert st == 0 and np.array_equal(kind, okind) and np.array_equal(rec.view(np.int32), orec.view(np.int32))
    del reps, pa, vc, out, oout, rec, orec


@pytest.mark.parametrize("n", E.BIG_N)
def test_read_path_encoders_past_the_first_scan_chunk(H, n):
    assert -(-n // E.ENC_TILE) >= E.SCAN_CHUNK
    g = np.random.Generator(np.random.PCG64(n + 1))
    # MaxSlotReply: every record answers one of a few MaxSlotRequests of a small request batch
    reqs = [E.fbytes(3, E.fbytes(1, E.fbytes(1, bytes(k)) + E.fint(2, 7 * k) + E.fint(3, -k))) for k in range(5)]
    buf, roffs = R.pack(reqs)
    kind0, rec0 = H["mp"].wire_decode_inbound(1, buf, roffs)
    j = g.integers(0, 5, size=n)
    recs = rec0[j].copy()
    recs["a"] = g.integers(0, 2, size=n) << 16 | g.integers(0, 3, size=n)
    recs["b"] = rand_i32(g, n)
    kind = kind0[j]
    out, offs = H["mp"].wire_encode_max_slot_replies(buf[:roffs[-1]], kind, recs)
    st, _, oout, ooffs = R.encode_max_slot_replies(buf[:roffs[-1]], kind, recs, 2, 3)
    assert st == 0 and np.array_equal(offs, ooffs) and np.array_equal(out, oout)
    k2, rep, _ = H["client"].wire_decode(out, offs)
    assert (k2 == 4).all() and np.array_equal(rep["slot"], recs["b"])
    assert np.array_equal(rep["voter"], recs["a"])
    del out, oout, rep, recs
    # ReadRequest and ReadRequestBatch, decoded back by the replica
    cmd = lambda k: E.fbytes(2, E.command(np.random.Generator(np.random.PCG64(k))))   # noqa: E731
    arena, voffs = R.pack([cmd(0), b"", cmd(1) + cmd(2), cmd(3)])
    arena = arena[:voffs[-1]]
    rs = np.zeros(n, dtype=READ_SLOT); rs["key"] = g.integers(0, 4, size=n); rs["slot"] = rand_i32(g, n)
    for r, batcher in ((H["client"], False), (H["batcher"], True)):
        out, offs = r.wire_encode_read_requests(rs, arena, voffs)
        st, _, oout, ooffs = R.encode_read_requests(rs, batcher, arena, voffs)
        assert st == 0 and np.array_equal(offs, ooffs) and np.array_equal(out, oout)
        if batcher:
            kind, chosen, _, reads, _, split = H["mp"].wire_decode_replica_inbound(out, offs)
            ncmd = np.array([1, 0, 2, 1])[rs["key"]]
            assert (kind == 5).all() and split == n and len(chosen) == 0
            assert np.array_equal(reads["slot"], np.repeat(rs["slot"], ncmd))


def ep_expected(G, call, in_rows, out_rows, me, entries, cmd_value=None):
    return W.expected_encode(G, call, in_rows, out_rows, EP_N, me, cmd_value, entries)


def ep_encode(H, call, in_rows, out_rows, arena, voffs, cap):
    """fpx_epaxos_wire_encode into a buffer of `cap` bytes -> (bytes, offsets)"""
    in_rows = np.ascontiguousarray(in_rows, dtype=np.int32)
    rows = None if out_rows is None else np.ascontiguousarray(out_rows, dtype=np.int32)
    out = np.zeros(max(cap, 1), dtype=np.uint8)
    offs = np.zeros(len(in_rows) + 1, dtype=np.int32)
    H["ep"]._host_call(H["ep"]._L.fpx_epaxos_wire_encode, call, in_rows.ctypes.data, None if rows is None else rows.ctypes.data,
                       len(in_rows), arena.ctypes.data, voffs.ctypes.data, len(voffs) - 1, out.ctypes.data, cap,
                       offs.ctypes.data)
    return out[:offs[-1]], offs


def ep_lead_rows(g, m, vids):
    rows = np.zeros((m, 8 + EP_N), dtype=np.int32)
    rows[:, 0] = 0; rows[:, 1] = g.integers(0, 1 << 20, size=m); rows[:, 2] = g.integers(0, 300, size=m)
    rows[:, 3] = g.integers(0, 3, size=m); rows[:, 4] = vids; rows[:, 5] = rand_i32(g, m)
    rows[:, 8:] = rand_i32(g, m * EP_N).reshape(m, EP_N)
    return rows


@pytest.mark.parametrize("n", E.BIG_N)
def test_epaxos_encoder_past_the_first_scan_chunk(H, G, n):
    """lead -> PreAccept and handlePreAccept's replies at n records: the records repeat with a period of 7 (prime to
    the tile), so the runtime serialises one period and the whole output is that period repeated."""
    assert -(-n // E.ENC_TILE) >= E.SCAN_CHUNK
    g = np.random.Generator(np.random.PCG64(n + 2))
    arena, voffs = W.value_arena(8)
    entries = W.split(arena, voffs)
    P = 7
    lead = ep_lead_rows(g, P, [0, 1, VALUE_NOOP, 3, 4, 5, 6])
    replies = np.zeros((P, 4 + EP_N), dtype=np.int32)
    replies[:, 0] = [1, 2, 1, 0, 1, 2, 1]; replies[:, 1:] = rand_i32(g, P * (3 + EP_N)).reshape(P, -1)
    pa = np.zeros((P, 6 + 2 * EP_N), dtype=np.int32); pa[:, :4] = lead[:, :4]
    for call, in_rows, out_rows in ((CALL_LEAD, lead, None), (CALL_PREACCEPT, pa, replies)):
        period = ep_expected(G, call, in_rows, out_rows, 0, entries)
        reps = -(-n // P)
        big_in = np.tile(in_rows, (reps, 1))[:n]
        big_out = None if out_rows is None else np.tile(out_rows, (reps, 1))[:n]
        lens = np.tile([len(m) for m in period], reps)[:n]
        out, offs = ep_encode(H, call, big_in, big_out, arena, voffs, int(lens.sum()))
        assert np.array_equal(offs, np.concatenate([[0], np.cumsum(lens)]))
        whole = np.frombuffer(b"".join(period), dtype=np.uint8)
        k = n // P
        assert np.array_equal(out[:k * len(whole)].reshape(k, -1), np.broadcast_to(whole, (k, len(whole))))
        assert bytes(out[k * len(whole):]) == b"".join(period[:n - k * P])
        if call == CALL_LEAD:
            kind, rows, _ = H["ep"].wire_decode(out, offs)
            assert (kind == 2).all() and np.array_equal(rows[:, W.SEQ], big_in[:, 5])
            assert np.array_equal(rows[:, W.DEPS:], big_in[:, 8:])


def test_replica_decode_past_the_first_scan_chunk(H):
    """n = 4096 * 256 + 257 ReplicaInbound messages, twice: the first Chosen in tile 4096 with a read after it in the
    same tile, and the first Chosen in tile 0 with every read after tile 4096."""
    n = E.SCAN_CHUNK * E.CTA + E.CTA + 1
    g = np.random.Generator(np.random.PCG64(3))
    reads = [E.replica_message((2, 3, 4, 5, 6, 7))(g) for _ in range(16)]
    chosen = [E.replica_message((1,))(g) for _ in range(16)]
    nothing = E.pad(b"", 5)
    for first_chosen, first_read in ((E.SCAN_CHUNK * E.CTA + 9, None), (5, E.SCAN_CHUNK * E.CTA + 100)):
        j, pick = g.integers(0, 16, size=n), g.integers(0, 3, size=n)
        anything = lambda i: (reads, chosen, [nothing] * 16)[pick[i]][j[i]]       # noqa: E731
        msgs = []
        for i in range(n):
            if i == first_chosen:
                msgs.append(chosen[j[i]])
            elif first_read is None:           # reads before the first Chosen, one right after it, then anything
                msgs.append((reads[j[i]] if pick[i] else nothing) if i < first_chosen else
                            reads[j[i]] if i == first_chosen + 1 else anything(i))
            else:                              # Chosen from tile 0 on, no read before tile 4096
                msgs.append(nothing if i < first_chosen else reads[j[i]] if i == first_read else
                            (chosen[j[i]] if pick[i] else nothing) if i < first_read else anything(i))
        buf, offs = R.pack(msgs)
        assert -(-n // E.CTA) > E.SCAN_CHUNK
        o = R.decode_replica(buf, offs, 11, 3)
        st, got = status_of(H["mp"].wire_decode_replica_inbound, buf, offs, 11, 3)
        assert st == (o[0], o[1]) == (0, -1)
        kind, ch, cvals, rd, rcmds, split = got
        assert split == o[7] == (first_chosen + 1 if first_read is None else first_read)
        assert split // E.CTA >= E.SCAN_CHUNK
        for x, y in zip((kind, ch, cvals, rd, rcmds), o[2:7]):
            assert np.array_equal(np.asarray(x).view(np.int32), np.asarray(y).view(np.int32))
        assert len(ch) > 0 and (len(rd) > 0) == (first_read is None)     # records of [0, split) only


# ------------------------------------------------------------------------------------------------ out_capacity
def encoders(H, G, n):
    """(name, handle, host fn, host args before out, dev fn or None, dev args before d_out, oracle bytes, offsets)"""
    g = np.random.Generator(np.random.PCG64(n))
    L = H["mp"]._L
    arena, voffs = short_values(g)
    arena = arena[:voffs[-1]].copy()
    nv = len(voffs) - 1
    vid = np.where(g.integers(0, 5, size=n) == 0, VALUE_NOOP, g.integers(0, nv, size=n)).astype(np.int32)
    p2b = np.zeros(n, dtype=P2B)
    for f in P2B.names:
        p2b[f] = rand_i32(g, n)
    nk = np.zeros(n, dtype=NACK); nk["round"] = p2b["round"]
    ch = np.zeros(n, dtype=CHOSEN); ch["slot"] = p2b["slot"]; ch["value_id"] = np.where(vid < 0, 0, vid)
    vc = ch.copy(); vc["value_id"] = vid
    reps = p2b.copy(); reps["group"] = g.integers(0, 4, size=n); reps["round"] = np.where(reps["group"] == 2, vid, reps["round"])
    pa = np.zeros(n, dtype=P2A); pa["slot"], pa["round"], pa["value_id"] = p2b["slot"], p2b["round"], vid
    sk = np.zeros(n, dtype=VM_SKIP); sk["server"], sk["slot_start"], sk["slot_stop"] = p2b["group"], p2b["slot"], p2b["round"]
    ep_arena, ep_voffs = W.value_arena(8)
    lead = ep_lead_rows(g, n, np.where(vid < 0, VALUE_NOOP, vid % 8))
    reqs = [E.fbytes(3, E.fbytes(1, E.fbytes(1, bytes(k)) + E.fint(2, k) + E.fint(3, k))) for k in range(3)]
    rbuf, roffs = R.pack(reqs)
    rbuf = rbuf[:roffs[-1]].copy()
    kind0, rec0 = H["mp"].wire_decode_inbound(1, rbuf, roffs)
    msr = rec0[g.integers(0, 3, size=n)].copy(); msr["a"] = g.integers(0, 3, size=n); msr["b"] = rand_i32(g, n)
    mkind = np.full(n, 3, dtype=np.int32)
    rarena, rvoffs = R.pack([E.fbytes(2, E.command(g)) for _ in range(3)])
    rarena = rarena[:rvoffs[-1]].copy()
    rs = np.zeros(n, dtype=READ_SLOT); rs["key"] = g.integers(0, 3, size=n); rs["slot"] = rand_i32(g, n)
    keep = [arena, voffs, p2b, nk, ch, vc, reps, pa, sk, ep_arena, ep_voffs, lead, rbuf, kind0, msr, mkind, rarena,
            rvoffs, rs]
    d = {id(a): dev(a) for a in keep}
    P = lambda a: a.ctypes.data                      # noqa: E731
    D = lambda a: d[id(a)].data_ptr()                # noqa: E731
    out = []

    def add(name, handle, fn, hargs, dfn, dargs, oracle):
        st, _, ob, oo = oracle
        assert st == 0
        out.append((name, handle, fn, hargs, dfn, dargs, np.asarray(ob, dtype=np.uint8), oo))
    ob, oo = O.wire_encode_phase2b(p2b)
    add("phase2b", "mp", L.fpx_wire_encode_phase2b, (P(p2b), n), L.fpx_wire_encode_phase2b_dev, (D(p2b), n), (0, 0, ob, oo))
    ob, oo = O.wire_encode_mencius_phase2b(p2b)
    add("mencius_phase2b", "mencius", L.fpx_wire_encode_phase2b, (P(p2b), n), L.fpx_wire_encode_phase2b_dev, (D(p2b), n),
        (0, 0, ob, oo))
    ob, oo = O.wire_encode_nack(nk)
    add("nack", "mp", L.fpx_wire_encode_nack, (P(nk), n), None, None, (0, 0, ob, oo))
    add("chosen", "mp", L.fpx_wire_encode_chosen, (P(ch), n, P(arena), P(voffs), nv), None, None,
        O.wire_encode_chosen(ch, arena, voffs))
    for what, recs, fn, dfn in (("replies", reps, L.fpx_wire_encode_vm_replies, L.fpx_wire_encode_vm_replies_dev),
                                ("chosen", vc, L.fpx_wire_encode_vm_chosen, L.fpx_wire_encode_vm_chosen_dev),
                                ("phase2a", pa, L.fpx_wire_encode_vm_phase2a, L.fpx_wire_encode_vm_phase2a_dev)):
        add("vm_" + what, "vm", fn, (P(recs), n, P(arena), P(voffs), nv), dfn, (D(recs), n, D(arena), D(voffs), nv),
            V.encode(what, recs, arena, voffs, servers=3))
    add("vm_skip", "vm", L.fpx_wire_encode_vm_skip, (P(sk), n), L.fpx_wire_encode_vm_skip_dev, (D(sk), n),
        V.encode("skip", sk, servers=3))
    ep_bytes = ep_expected(G, CALL_LEAD, lead, None, 0, W.split(ep_arena, ep_voffs))
    ep_offs = np.concatenate([[0], np.cumsum([len(m) for m in ep_bytes])]).astype(np.int32)
    add("epaxos", "ep", L.fpx_epaxos_wire_encode, (CALL_LEAD, P(lead), None, n, P(ep_arena), P(ep_voffs), 8),
        L.fpx_epaxos_wire_encode_dev, (CALL_LEAD, D(lead), None, n, D(ep_arena), D(ep_voffs), 8),
        (0, 0, np.frombuffer(b"".join(ep_bytes), np.uint8), ep_offs))
    add("max_slot_replies", "mp", L.fpx_wire_encode_max_slot_replies, (P(rbuf), len(rbuf), P(mkind), P(msr), n),
        L.fpx_wire_encode_max_slot_replies_dev, (D(rbuf), len(rbuf), D(mkind), D(msr), n),
        R.encode_max_slot_replies(rbuf, mkind, msr, 2, 3))
    add("read_requests", "client", L.fpx_reads_wire_encode_read_requests, (P(rs), n, P(rarena), P(rvoffs), 3),
        L.fpx_reads_wire_encode_read_requests_dev, (D(rs), n, D(rarena), D(rvoffs), 3),
        R.encode_read_requests(rs, False, rarena, rvoffs))
    return out, (keep, d)


CALLS = itertools.count()


def handler_call(H, key):
    """one handler call of the handle whose encode was refused: it must succeed"""
    k = next(CALLS)
    if key == "mp":
        H["mp"].replica_chosen(np.array([(k, 0)], dtype=CHOSEN))
    elif key == "mencius":
        H["mencius"].mencius_arm_range(np.array([(400 + 2 * k, 401 + 2 * k, 0, -1)], dtype=P2A_RANGE))
    elif key == "vm":
        H["vm"].vm_client_request(np.array([(600 + k, 0, 700 + k, (600 + k) % 3)], dtype=P2A))
    elif key == "ep":
        H["ep"].lead(np.array([[0, k, 0, 0, 5, 1, 0, 0] + [0] * EP_N], dtype=np.int32))
    else:
        H[key].open([k], [k])


@pytest.mark.parametrize("n", [100, 3 * E.ENC_TILE + 5])
def test_out_capacity_refusals(H, G, n):
    """Every encoder, host and device form: capacity = total succeeds with the oracle's bytes; total - 1 and 0 are
    refused with FPX_ERR_INVALID_ARG at index 0, nothing is written at or past out_capacity (the host form leaves
    the caller's buffer untouched), and the handle's next encode and handler call succeed."""
    specs, _keep = encoders(H, G, n)
    for name, key, fn, hargs, dfn, dargs, ob, oo in specs:
        total = len(ob)
        h = H[key].h
        for cap in (total, total - 1, 0):
            buf = np.full(cap + 256, SENTINEL, dtype=np.uint8)
            offs = np.zeros(n + 1, dtype=np.int32)
            err = C.c_int64(-1)
            st = fn(h, *hargs, buf.ctypes.data, cap, offs.ctypes.data, C.byref(err))
            if cap == total:
                assert (st, err.value) == (0, -1), name
                assert np.array_equal(offs, oo) and np.array_equal(buf[:total], ob), name
                assert (buf[total:] == SENTINEL).all(), name
            else:
                assert (st, err.value) == (INVALID_ARG, 0), (name, cap)
                assert (buf == SENTINEL).all(), (name, cap)
                handler_call(H, key)
            if dfn is None:
                continue
            d_out = torch.full((cap + 256,), SENTINEL, dtype=torch.uint8, device=DEV)
            d_offs = torch.zeros(n + 1, dtype=torch.int32, device=DEV)
            H[key]._check(dfn(h, *dargs, d_out.data_ptr(), cap, d_offs.data_ptr()))
            got = collect(H[key])
            tail = d_out[cap:].cpu().numpy()
            assert (tail == SENTINEL).all(), (name, cap)          # the guard region
            if cap == total:
                assert got == (0, -1), name
                assert np.array_equal(d_offs.cpu().numpy(), oo) and np.array_equal(d_out[:total].cpu().numpy(), ob)
            else:
                assert got == (INVALID_ARG, 0), (name, cap)
                handler_call(H, key)
        # nothing latched: the same encode succeeds again
        buf = np.zeros(total + 16, dtype=np.uint8)
        offs = np.zeros(n + 1, dtype=np.int32)
        err = C.c_int64(-1)
        assert fn(h, *hargs, buf.ctypes.data, total, offs.ctypes.data, C.byref(err)) == 0, name
        assert np.array_equal(buf[:total], ob)


# ------------------------------------------------------------------------------------------- length-varint widths
def varint_lens():
    """every width's edge, and lengths that take a message body across 127/128 and 16 383/16 384 with the other
    fields' widths"""
    return [0, 1, 5, 127, 128] + list(range(110, 131)) + [16383, 16384] + list(range(16360, 16390)) + \
        [(1 << 21) - 1, 1 << 21]


def varint_records(g, nvalues):
    """value ids: every value twice, a few Noops; slots of every width"""
    ids = np.concatenate([np.arange(nvalues), np.arange(nvalues), np.full(6, VALUE_NOOP)]).astype(np.int32)
    slots = np.array([E.rand_i32(g) for _ in range(len(ids))], dtype=np.int32)
    return ids, slots


def through_both_paths(out, offs, decode):
    """The encoded messages re-laid by E.window_batch and decoded: decode(buf, offs) -> value length per batch
    message (-1: none).  Asserts that body lengths and value lengths of widths 1-3 are parsed in staged CTAs and of
    widths 1-4 in unstaged ones; returns (src, value lengths)."""
    msgs = W.split(out, offs)
    buf, boffs, src = E.window_batch(msgs)
    staged = np.array([c[3] for c in E.cta_spans(boffs)])[np.arange(len(src)) // E.CTA]
    vlen = decode(buf, boffs)
    real = src >= 0
    for cls, want in ((True, {1, 2, 3}), (False, {1, 2, 3, 4})):
        sel = [j for j in np.flatnonzero(real & (staged == cls)) if len(msgs[src[j]])]
        assert {E.body_width(msgs[src[j]]) for j in sel} == want
        assert {len(E.venc(vlen[j])) for j in sel if vlen[j] >= 0} == want
    return src, vlen


def test_value_length_varint_widths(H, G):
    g = np.random.Generator(np.random.PCG64(21))
    lens = varint_lens()
    arena, voffs = E.value_arena(lens, g)
    ids, slots = varint_records(g, len(lens))
    vl = np.where(ids == VALUE_NOOP, 2, np.diff(voffs)[np.where(ids < 0, 0, ids)])
    # MultiPaxos Chosen (no Noop), decoded back by the replica
    ch = np.zeros(len(ids), dtype=CHOSEN); ch["slot"] = slots; ch["value_id"] = np.where(ids < 0, 0, ids)
    out, offs = H["mp"].wire_encode_chosen(ch, arena, voffs)
    st, _, oout, ooffs = O.wire_encode_chosen(ch, arena, voffs)
    assert st == 0 and np.array_equal(offs, ooffs) and np.array_equal(out, oout)

    def replica_chosen(buf, boffs):
        o = R.decode_replica(buf, boffs)
        got = H["mp"].wire_decode_replica_inbound(buf, boffs)
        assert o[0] == 0
        for x, y in zip(got[:5], o[2:7]):
            assert np.array_equal(np.asarray(x).view(np.int32), np.asarray(y).view(np.int32))
        v = np.full(len(boffs) - 1, -1)
        v[got[1]["value_id"]] = got[2][:, 1]
        assert np.array_equal(got[2].sum(axis=1), boffs[got[1]["value_id"] + 1])     # the value ends its message
        return v
    src, v = through_both_paths(out, offs, replica_chosen)
    assert np.array_equal(v[src >= 0], np.diff(voffs)[ch["value_id"]][src[src >= 0]])
    # vanilla Mencius Chosen, Phase2a and the reply stream, decoded back
    vc = ch.copy(); vc["value_id"] = ids
    pa = np.zeros(len(ids), dtype=P2A); pa["slot"] = slots; pa["round"] = slots[::-1]; pa["value_id"] = ids
    reps = np.zeros(len(ids), dtype=P2B); reps["group"] = 2; reps["slot"] = slots; reps["round"] = ids

    def vm(buf, boffs):
        kind, rec, _ = H["vm"].wire_decode_vm_server_inbound(buf, boffs)
        st, _, okind, orec, _ = V.decode(buf, boffs)
        assert st == 0 and np.array_equal(kind, okind) and np.array_equal(rec.view(np.int32), orec.view(np.int32))
        return np.where(kind != 0, rec["d"], -1)
    for what, fn, recs in (("chosen", H["vm"].wire_encode_vm_chosen, vc), ("phase2a", H["vm"].wire_encode_vm_phase2a, pa),
                           ("replies", H["vm"].wire_encode_vm_replies, reps)):
        out, offs = fn(recs, arena, voffs)
        st, _, oout, ooffs = V.encode(what, recs, arena, voffs, servers=3)
        assert st == 0 and np.array_equal(offs, ooffs) and np.array_equal(out, oout), what
        src, v = through_both_paths(out, offs, vm)
        assert np.array_equal(v[src >= 0], vl[src[src >= 0]]), what
    # ReadRequest / ReadRequestBatch whose Command takes every length width, decoded back by the replica
    commands = [E.fbytes(1, E.fbytes(1, b"") + E.fint(2, 0) + E.fint(3, 0)) + E.fbytes(2, bytes(k)) for k in lens]
    clen = np.array([len(c) for c in commands])
    rarena, rvoffs = R.pack([E.fbytes(2, c) for c in commands])
    rarena = rarena[:rvoffs[-1]]
    keep = ids >= 0
    rs = np.zeros(int(keep.sum()), dtype=READ_SLOT); rs["key"] = ids[keep]; rs["slot"] = slots[keep]

    def replica_reads(buf, boffs):
        o = R.decode_replica(buf, boffs)
        got = H["mp"].wire_decode_replica_inbound(buf, boffs)
        assert o[0] == 0 and got[5] == len(boffs) - 1
        for x, y in zip(got[:5], o[2:7]):
            assert np.array_equal(np.asarray(x).view(np.int32), np.asarray(y).view(np.int32))
        v = np.full(len(boffs) - 1, -1)
        v[np.searchsorted(boffs, got[4][:, 0], side="right") - 1] = got[4][:, 1]
        return v
    for r, batcher in ((H["client"], False), (H["batcher"], True)):
        out, offs = r.wire_encode_read_requests(rs, rarena, rvoffs)
        st, _, oout, ooffs = R.encode_read_requests(rs, batcher, rarena, rvoffs)
        assert st == 0 and np.array_equal(offs, ooffs) and np.array_equal(out, oout)
        src, v = through_both_paths(out, offs, replica_reads)
        assert np.array_equal(v[src >= 0], clen[rs["key"]][src[src >= 0]])


def ep_value_entries(G, lens):
    """CommandOrNoop{command{client_address of `len` bytes, 0, 0, ""}} per length (0: an empty CommandOrNoop)"""
    entries = []
    for k in lens:
        m = G.cls("CommandOrNoop")()
        if k:
            m.command.client_address = bytes(k); m.command.client_pseudonym = 0
            m.command.client_id = 0; m.command.command = b""
        entries.append(m.SerializeToString())
    arena, voffs = R.pack(entries)
    return entries, arena[:voffs[-1]].copy(), voffs


def test_epaxos_value_length_varint_widths(H, G):
    """PreAccept (lead), PrepareOk / Commit (handlePrepare's replies), and Accept / Commit (handlePreAcceptOk's
    events, whose value the encoder reads from the cmdLog) with CommandOrNoops of every length width"""
    g = np.random.Generator(np.random.PCG64(22))
    entries, arena, voffs = ep_value_entries(G, varint_lens())
    ids, slots = varint_records(g, len(entries))
    m = len(ids)
    lead = ep_lead_rows(g, m, ids)
    prep_in = np.zeros((m, 4), dtype=np.int32); prep_in[:, :2] = lead[:, :2]
    prep = np.zeros((m, 9 + EP_N), dtype=np.int32)
    prep[:, 0] = np.where(g.integers(0, 2, size=m) == 0, 1, 3)            # OK (PrepareOk) or COMMIT
    prep[:, 2:6] = g.integers(0, 300, size=(m, 4)); prep[:, 6] = g.integers(1, 3, size=m)
    prep[:, 7] = ids; prep[:, 8] = slots; prep[:, 9:] = rand_i32(g, m * EP_N).reshape(m, EP_N)
    # the events of handlePreAcceptOk for instances (0, 0 .. m-1), whose values a lead call puts in the cmdLog
    with EpaxosReplica(EP_F, 0, 1 << 10, max_batch=1 << 12) as ep:
        ep.lead(np.array([[0, i, 0, 0, int(v), 1, 0, 0] + [0] * EP_N for i, v in enumerate(ids)], dtype=np.int32))
        ok_in = np.zeros((m, 6 + EP_N), dtype=np.int32); ok_in[:, 1] = np.arange(m)
        ok_in[:, 2:6] = g.integers(0, 300, size=(m, 4)); ok_in[:, 6:] = rand_i32(g, m * EP_N).reshape(m, EP_N)
        events = np.zeros((m, 2 + EP_N), dtype=np.int32)
        events[:, 0] = np.where(g.integers(0, 3, size=m) == 0, 1, 2)        # FAST_COMMIT (Commit) or SLOW_ACCEPT (Accept)
        events[:, 1:] = rand_i32(g, m * (1 + EP_N)).reshape(m, -1)
        expected = ep_expected(G, CALL_PREACCEPTOK, ok_in, events, 0, entries, lambda rep, num: int(ids[num]))
        out, offs = ep_encode({"ep": ep}, CALL_PREACCEPTOK, ok_in, events, arena, voffs, sum(len(x) for x in expected))
        assert W.split(out, offs) == expected
        assert {W.ACCEPT, W.COMMIT} <= {x[0] >> 3 for x in expected}
    encoded = [(out, offs)]
    for call, in_rows, out_rows in ((CALL_LEAD, lead, None), (CALL_PREPARE, prep_in, prep)):
        expected = ep_expected(G, call, in_rows, out_rows, 0, entries)
        out, offs = ep_encode(H, call, in_rows, out_rows, arena, voffs, sum(len(x) for x in expected))
        assert W.split(out, offs) == expected
        encoded.append((out, offs))

    def ep_decode(buf, boffs):
        kind, rows, values = H["ep"].wire_decode(buf, boffs, 5)
        st, _, okind, orows, ovalues = W.decode(buf, boffs, EP_N, 5)
        assert st == 0 and np.array_equal(kind, okind) and np.array_equal(rows, orows) and np.array_equal(values, ovalues)
        return np.where(rows[:, W.VALUE] != -1, values[:, 1], -1)
    el = np.array([len(e) if v != VALUE_NOOP else 2 for e, v in zip([entries[max(v, 0)] for v in ids], ids)])
    for out, offs in encoded:
        src, v = through_both_paths(out, offs, ep_decode)
        assert np.array_equal(v[src >= 0], el[src[src >= 0]])
