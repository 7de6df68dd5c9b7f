"""The EPaxos wire oracle (tests/wire_ep_oracle.cc) against tests/golden/wire_epaxos.json (bytes written by Google's
Python protobuf runtime from S/epaxos/EPaxos.proto's shapes) and against that runtime on random and mutated
messages."""
import json
import os

import numpy as np
import pytest

import wire_ep_oracle as W

HERE = os.path.dirname(os.path.abspath(__file__))
CASES = json.load(open(os.path.join(HERE, "golden", "wire_epaxos.json")))["cases"]
DEFAULT_ROW = [-1, -1, -1, -1, 0, -1, -1, 0, -1, 0, 0, 0]


def decode_one(c):
    raw = bytes.fromhex(c["hex"])
    buf, offs = W.pack([raw])
    return raw, W.decode(buf, offs, c["n"], c["value_id_base"])


def test_golden_decode():
    assert len(CASES) > 100
    for c in CASES:
        raw, (st, err, kind, rows, values) = decode_one(c)
        name = c.get("name", c["type"])
        assert st == c["status"], name
        if st != W.OK:
            assert err == 0 and kind[0] == 0 and list(rows[0]) == DEFAULT_ROW + [0] * c["n"], name
            continue
        assert kind[0] == c["kind"], name
        assert list(rows[0]) == (c["row"] if c.get("row") else DEFAULT_ROW + [0] * c["n"]), name
        off, ln = values[0]
        assert raw[off:off + ln].hex() == c.get("value_hex", ""), name


def test_golden_covers_the_issue_cases():
    names = {c.get("name") for c in CASES}
    types = {c["type"] for c in CASES}
    assert {"pre_accept", "pre_accept_ok", "accept", "accept_ok", "commit", "prepare", "prepare_ok", "nack",
            "client_request", "prepare_ok.not_seen", "pre_accept.overflow_packed"} <= types
    assert {"instance twice (merge)", "unknown fields at every level", "missing instance_number", "overlong varint",
            "truncated nested length", "numReplicas != n", "set count != n", "command_or_noop twice",
            "unknown status"} <= names


def test_golden_batch_offsets_and_first_error():
    """all cases in one batch: spans are batch offsets, the first failing message is reported"""
    n = 3
    raws = [bytes.fromhex(c["hex"]) for c in CASES]
    buf, offs = W.pack(raws)
    st, err, kind, rows, values = W.decode(buf, offs, n, 0)
    first_bad = next(i for i, c in enumerate(CASES) if c["status"] != W.OK)
    assert st == CASES[first_bad]["status"] and err == first_bad
    for i, c in enumerate(CASES):
        if c["status"] == W.OK and c["kind"]:
            off, ln = values[i]
            assert bytes(buf[off:off + ln]).hex() == c["value_hex"]
            assert rows[i, W.VALUE] in (i, W.VALUE_NOOP, -1)


def test_robustness_agrees_with_the_protobuf_runtime():
    G = W.golden_module()
    for c in CASES:
        if c["type"] != "robustness":
            continue
        st, _ = W.runtime_status(G, bytes.fromhex(c["hex"]), c["n"])
        assert st == c["status"], c["name"]


def test_oracle_against_the_protobuf_runtime_on_random_messages():
    G = W.golden_module()
    g = np.random.Generator(np.random.PCG64(7))
    for n in (3, 5, 7):
        msgs = [W.random_message(G, g, n) for _ in range(300)]
        raws = [m.SerializeToString() for m in msgs]
        buf, offs = W.pack(raws)
        st, err, kind, rows, values = W.decode(buf, offs, n, 100)
        assert st == W.OK, err
        for i, m in enumerate(msgs):
            assert kind[i] == G.MEMBERS[m.WhichOneof("request")]
            assert list(rows[i]) == G.expected_row(m, n, 100 + i)
            off, ln = values[i]
            assert bytes(buf[off:off + ln]).hex() == G.expected_value(m)


def test_mutations_accept_and_reject_like_the_runtime():
    G = W.golden_module()
    g = np.random.Generator(np.random.PCG64(11))
    n = 3
    seen = set()
    for _ in range(4000):
        m = W.random_message(G, g, n)
        raw = W.mutate(m.SerializeToString(), g)
        want, pm = W.runtime_status(G, raw, n)
        buf, offs = W.pack([raw])
        st, err, kind, rows, values = W.decode(buf, offs, n, 0)
        seen.add(want)
        assert st == want, raw.hex()
        if st == W.OK and pm is not None and pm.WhichOneof("request"):
            assert list(rows[0]) == G.expected_row(pm, n, 0), raw.hex()
    assert seen == {W.OK, W.WIRE, W.UNSUPPORTED}


@pytest.mark.parametrize("n", [3, 7])
def test_pack_layouts(n):
    G = W.golden_module()
    g = np.random.Generator(np.random.PCG64(n))
    msgs = [W.random_message(G, g, n) for _ in range(400)]
    buf, offs = W.pack([m.SerializeToString() for m in msgs])
    st, _, kind, rows, _ = W.decode(buf, offs, n, 0)
    assert st == W.OK
    calls = {2: W.CALL_PREACCEPT, 4: W.CALL_ACCEPT, 3: W.CALL_PREACCEPTOK, 5: W.CALL_ACCEPTOK, 6: W.CALL_COMMIT,
             9: W.CALL_NACK, 7: W.CALL_PREPARE, 8: W.CALL_PREPAREOK}
    for k, call in calls.items():
        idx = np.nonzero(kind == k)[0]
        for i in idx[:20]:
            ld = np.arange(n, dtype=np.int32) + 5
            st, err, out = W.pack_rows(call, kind, rows, int(i), 1, n, ld if call == W.CALL_PREACCEPT else None)
            assert st == W.OK
            r, o = rows[i], list(out[0])
            head = [r[W.IREP], r[W.INUM]]
            deps = list(r[W.DEPS:])
            if call == W.CALL_PREACCEPT:
                assert o == head + [r[W.BORD], r[W.BREP], r[W.VALUE], r[W.SEQ]] + list(ld) + deps
            elif call == W.CALL_ACCEPT:
                assert o == head + [r[W.BORD], r[W.BREP], r[W.VALUE], r[W.SEQ]] + deps
            elif call == W.CALL_PREACCEPTOK:
                assert o == head + [r[W.BORD], r[W.BREP], r[W.REPLICA], r[W.SEQ]] + deps
            elif call == W.CALL_ACCEPTOK:
                assert o == head + [r[W.BORD], r[W.BREP], r[W.REPLICA], 0]
            elif call == W.CALL_COMMIT:
                assert o == head + [r[W.VALUE], r[W.SEQ]] + deps
            elif call in (W.CALL_NACK, W.CALL_PREPARE):
                assert o == head + [r[W.BORD], r[W.BREP]]
            else:
                v = r[W.VALUE] if r[W.STATUS] else 0
                assert o == head + [r[W.BORD], r[W.BREP], r[W.REPLICA], r[W.VBORD], r[W.VBREP], r[W.STATUS], v]
        # a row of another kind
        other = np.nonzero(kind != k)[0][0]
        st, err, _ = W.pack_rows(call, kind, rows, int(other), 1, n)
        assert (st, err) == (W.INVALID_ARG, other)


def test_pack_refuses_sparse_sets_and_other_calls():
    c = next(c for c in CASES if c["type"] == "pre_accept.overflow_packed")
    raw, (st, _, kind, rows, _) = decode_one(c)
    assert st == W.OK and rows[0, W.OVERFLOW] == 3
    assert W.pack_rows(W.CALL_PREACCEPT, kind, rows, 0, 1, 3)[:2] == (W.UNSUPPORTED, 0)
    for call in (W.CALL_LEAD, W.CALL_PREPARE_PHASE, W.CALL_SLOW_PATH_TIMER):
        assert W.pack_rows(call, kind, rows, 0, 1, 3)[0] == W.INVALID_ARG
