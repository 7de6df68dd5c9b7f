"""The batch builders of tests/test_wire_edges_gpu.py against the CPU oracles, without a device: padded and unpadded
messages decode to the same records, the CTAs span the stage window's edges as intended, the truncated and split
batches fail and split where intended, and the batches past the first scan chunk fit their memory budget."""
import numpy as np
import pytest

import wire_edges as E
import wire_reads_oracle as R
import wire_vm_oracle as V
from oracle import fpx_oracle_py as O


def decode(name, buf, offs):
    """(status, index, kind, the records as int32) of the oracle of decoder `name`"""
    if name.startswith("inbound"):
        st, err, kind, rec = O.wire_decode_inbound(int(name[-1]), buf, offs, 3, 3)
        return st, err, kind, rec.view(np.int32).reshape(-1, 4)
    if name == "vm":
        st, err, kind, rec, sender = V.decode(buf, offs)
        return st, err, kind, np.column_stack([rec.view(np.int32).reshape(-1, 4), sender])
    if name == "replica":
        st, err, kind, chosen, cvals, reads, rcmds, split = R.decode_replica(buf, offs)
        return st, err, kind, (chosen.view(np.int32), cvals[:, 1], reads["slot"], rcmds[:, 1], split)
    st, err, kind, out, spans = R.decode_reads(buf, offs, name == "batcher", 64)
    return st, err, kind, np.column_stack([out.view(np.int32).reshape(-1, 4), spans[:, 1]])


MAKE = {"inbound0": E.inbound_message(0), "inbound1": E.inbound_message(1), "inbound2": E.inbound_message(2),
        "inbound3": E.inbound_message(3), "vm": E.vm_message, "replica": E.replica_message((0, 1, 2, 3, 4, 5, 6, 7)),
        "client": E.reads_message(False), "batcher": E.reads_message(True)}


def without_spans(name, res):
    """the records with the value offsets dropped (they move with the padding), lengths kept"""
    if name == "replica":
        return res
    r = np.array(res, copy=True)
    if name.startswith("inbound") or name == "vm":
        r[:, 2] = 0
    return r


@pytest.mark.parametrize("name", sorted(MAKE))
def test_padded_messages_decode_to_the_same_records(name):
    g = np.random.Generator(np.random.PCG64(1))
    msgs = [MAKE[name](g) for _ in range(600)]
    padded = [E.pad(m, len(m) + int(k)) for m, k in zip(msgs, g.choice([0, 2, 50, 129, 131, 400], size=len(msgs)))]
    a, b = decode(name, *E.pack(msgs)), decode(name, *E.pack(padded, lead=E.LEAD))
    assert a[:2] == b[:2] == (0, -1)
    assert np.array_equal(a[2], b[2]) and len(set(a[2].tolist())) > 1
    x, y = without_spans(name, a[3]), without_spans(name, b[3])
    if name == "replica":
        for u, v in zip(x, y):
            assert np.array_equal(u, v)
    else:
        assert np.array_equal(x, y)


@pytest.mark.parametrize("name", sorted(MAKE))
def test_stage_batches_span_the_window_edges(name):
    g = np.random.Generator(np.random.PCG64(2))
    buf, offs = E.stage_batch(MAKE[name], g)
    ctas = E.cta_spans(offs)
    assert offs[0] == E.LEAD and offs[-1] % 16 == 7 and len(buf) >= offs[-1]
    assert [c[2] for c in ctas[:len(E.SPAN_ORDER)]] == list(E.SPAN_ORDER)
    assert {(c[2], c[0] % 16) for c in ctas[:len(E.SPAN_ORDER)]} == {(s, m) for s in E.EDGE_SPANS for m in (0, 1, 15)}
    assert [c[3] for c in ctas[:len(E.SPAN_ORDER)]] == [s <= E.STAGE for s in E.SPAN_ORDER]
    assert ctas[-1][3]
    assert decode(name, buf, offs)[:2] == (0, -1)
    for cut in (2, 3, 4):
        buf, offs = E.stage_batch(MAKE[name], g, cut=cut)
        assert len(offs) - 1 == (cut + 1) * E.CTA and E.cta_spans(offs)[-1][2] == E.SPAN_ORDER[cut]
        assert decode(name, buf, offs)[:2] == (-15, len(offs) - 2)


def test_value_spans_point_into_their_own_message():
    """the oracle's spans of a stage batch lie inside the message that carries them (what the GPU test checks of
    both kinds of CTA)"""
    g = np.random.Generator(np.random.PCG64(3))
    buf, offs = E.stage_batch(E.vm_message, g)
    st, _, kind, rec, _ = V.decode(buf, offs)
    assert st == 0
    i = np.flatnonzero(np.isin(kind, (1, 2, 3, 4, 7, 8)))
    off, ln = rec["c"][i], rec["d"][i]
    assert ((offs[i] <= off) & (off + ln <= offs[i + 1])).all()
    staged = np.array([c[3] for c in E.cta_spans(offs)])[i // E.CTA]
    assert staged.any() and (~staged).any()


@pytest.mark.parametrize("staged", [True, False])
def test_split_batches_split_inside_the_intended_cta(staged):
    buf, offs, at = E.split_batch(np.random.Generator(np.random.PCG64(4)), staged)
    st, err, kind, chosen, *_, split = R.decode_replica(buf, offs)
    assert (st, err) == (0, -1) and split == at + 1 and kind[at] == 1 and kind[at + 1] == 2
    assert E.cta_spans(offs)[at // E.CTA][3] == staged


def test_large_batches_fit_their_budget():
    """past the first scan chunk: more than 4096 tiles, and outputs around 100 MB with short values"""
    for n in E.BIG_N:
        assert -(-n // E.ENC_TILE) >= E.SCAN_CHUNK
    assert -(-E.BIG_N[1] // E.ENC_TILE) == E.SCAN_CHUNK + 2
    n = 1 << 16                                        # bytes per record of the largest message shapes, scaled up
    g = np.random.Generator(np.random.PCG64(5))
    recs = np.zeros(n, dtype=V.P2A)
    recs["slot"] = g.integers(-(1 << 31), 1 << 31, size=n) >> g.integers(0, 32, size=n)
    recs["round"] = recs["slot"][::-1]
    recs["value_id"] = g.integers(0, 6, size=n)
    arena, voffs = R.pack([bytes(k) for k in range(6)])
    st, _, out, _ = V.encode("phase2a", recs, arena, voffs, servers=3)
    assert st == 0 and len(out) / n * E.BIG_N[1] < 160e6


def test_value_lengths_take_every_varint_width():
    assert sorted({len(E.venc(k)) for k in E.VALUE_LENS}) == [1, 2, 3, 4]
    arena, voffs = E.value_arena(E.VALUE_LENS, np.random.Generator(np.random.PCG64(6)))
    ch = np.zeros(len(E.VALUE_LENS), dtype=O.np.dtype([("slot", "<i4"), ("value_id", "<i4")]))
    ch["slot"] = [0, 1, 127, 128, 16384, -1, 1 << 21, 5]
    ch["value_id"] = np.arange(len(E.VALUE_LENS))
    st, _, out, offs = O.wire_encode_chosen(ch, arena, voffs)
    assert st == 0 and E.body_len_widths(out, offs) == {1, 2, 3, 4}
