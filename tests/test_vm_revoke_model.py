"""Hand cases of the vanilla Mencius server model the revocation GPU tests compare against (no GPU)."""
from vm_revoke_model import NOOP, Server


def test_nack_keeps_the_raise_of_the_slots_before_it():
    s = Server(1, 3)
    s.phase2a(6, 0, 5)
    s.phase2a(9, 7, 8)                       # above the Phase1a's round
    reply, skip = s.phase1a(4, 0, 12)        # slots 0, 3, 6, 9
    assert reply == ("nack", 0, 12, 7) and skip is None
    assert s.log[0] == ("voteless", 4) and s.log[3] == ("voteless", 4)
    assert s.log[6] == ("pending", 4, 0, 5) and s.log[9] == ("pending", 7, 7, 8)


def test_raised_entry_nacks_a_lower_phase2a_and_keeps_its_vote():
    s = Server(2, 3)
    s.phase2a(0, 0, 11)
    assert s.phase1a(5, 0, 1)[0] == ("phase1b", 5, 0, 1, [(0, "pending", 0, 11)])
    assert s.phase2a(0, 0, 12) == ("nack", 5)
    assert s.phase1a(6, 0, 1)[0] == ("phase1b", 6, 0, 1, [(0, "pending", 0, 11)])
    assert s.phase2a(0, 6, 13) == ("phase2b", 6)
    assert s.entry_row(0) == (2, 6, 6, 13, 0)


def test_self_revocation_fills_before_the_walk():
    s = Server(1, 3, next_slot=4)
    s.phase2a(1, 0, 3)
    reply, skip = s.phase1a(4, 1, 11)        # slots 1, 4, 7, 10 of server 1
    assert skip == (4, 11) and s.next_slot == 13
    assert reply == ("phase1b", 4, 1, 11, [(1, "pending", 0, 3), (4, "chosen", NOOP, False),
                                           (7, "chosen", NOOP, False), (10, "chosen", NOOP, False)])


def test_empty_range_and_chosen_with_revocation():
    s = Server(1, 3)
    assert s.phase1a(3, 6, 6)[0] == ("phase1b", 3, 6, 6, [])
    s.choose(6, 9, True)
    s.choose(6, 9, False)
    assert s.phase2a(6, 0, 1) == ("chosen", 9, True)
    assert s.phase1a(3, 6, 7)[0] == ("phase1b", 3, 6, 7, [(6, "chosen", 9, True)])


# the steady-state handlers agree with tests/scala_transcription.py's VanillaServer over random traces
from hypothesis import given, settings, strategies as st  # noqa: E402

from scala_transcription import VanillaServer  # noqa: E402

OPS = st.lists(st.tuples(st.sampled_from(["phase2a", "chosen"]), st.integers(0, 11), st.integers(0, 6),
                         st.integers(0, 4)), max_size=60)


@settings(max_examples=200, deadline=None)
@given(OPS)
def test_model_agrees_with_the_transcription_without_revocation(ops):
    m, t = Server(1, 3), VanillaServer(1, 1)
    for op, slot, rnd, v in ops:
        if op == "phase2a":
            a, b = m.phase2a(slot, rnd, v), t.handle_phase2a(slot, rnd, v)
            assert a[0] == b[0] and (a[1] == b[2])
        else:
            m.choose(slot, v, False); t.handle_chosen(slot, v)
    for slot in range(12):
        e, te = m.log.get(slot), t.log.get(slot)
        assert (e is None) == (te is None)
        if e is not None:
            assert e[0] == te[0] and (e[1:] == te[1:] if e[0] == "pending" else e[1] == te[1])
