"""CPU: the poison catalogue (tests/poison_cases.py) accounts for every entry point of include/borb.h - each BORB_API name is driven
by a case or carries the reason it needs none - and borb_debug_set_poison checks its argument without touching a device."""
from tests import poison_cases as P
from tests.test_cabi import declared_symbols, lib  # noqa: F401  (module fixture)


def test_every_entry_point_is_in_exactly_one_table():
    names = set(declared_symbols())
    assert not set(P.COVERED) & set(P.NOT_COVERED)
    assert set(P.COVERED) | set(P.NOT_COVERED) == names, (sorted(names - set(P.COVERED) - set(P.NOT_COVERED)),
                                                          sorted(set(P.COVERED) | set(P.NOT_COVERED) - names))
    for name, cases in P.COVERED.items():
        assert cases and set(cases) <= set(P.CASES), name
    assert all(reason.strip() for reason in P.NOT_COVERED.values())


def test_every_case_drives_an_entry_point():
    assert set(P.CASES) == set().union(*P.COVERED.values())


def test_poison_switch_checks_its_argument(lib):
    so = lib.load()
    try:
        for byte in (-1, 0, 255, 0x7F):
            assert so.borb_debug_set_poison(byte) == 0, byte
        for byte in (-2, 256, 1 << 30, -(1 << 31)):
            assert so.borb_debug_set_poison(byte) == 1, byte
            assert b"poison byte" in so.borb_last_error()
    finally:
        assert so.borb_debug_set_poison(-1) == 0
