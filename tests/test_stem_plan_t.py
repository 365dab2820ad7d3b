"""CPU: which stem convolutions take the transposed four-row instance (b2_stemconv.cuh, kT), through the host-only view of the
launcher's choice.  The rule: the four-row instance runs where it did before (BN = 64, a temporal filter, not pair mode, three ring
stages fit, i.e. kh <= 7), and it is the transposed one when an output row has at most 112 columns.  The force knob selects
(4 | 16) or refuses (4) the transposed instance wherever the four-row one is eligible."""
import ctypes

import pytest

FORCE_T = 4 | 16


@pytest.fixture(scope="module")
def lib():
    from pretorched_x_b200 import _lib
    lib = _lib.load()
    lib.b2_debug_stem_plan.argtypes = [ctypes.c_int] * 5 + [ctypes.POINTER(ctypes.c_int)]
    lib.b2_debug_set_stem_rows.argtypes = [ctypes.c_int]
    lib.b2_debug_set_stem_rows(-1)
    yield lib
    lib.b2_debug_set_stem_rows(-1)


def plan(lib, K, kt, kh, Wo, pair, force=-1):
    out = (ctypes.c_int * 2)()
    lib.b2_debug_set_stem_rows(force)
    try:
        assert lib.b2_debug_stem_plan(K, kt, kh, Wo, int(pair), out) == 0
    finally:
        lib.b2_debug_set_stem_rows(-1)
    return out[0], bool(out[1])


RULE_CASES = [
    # K, kt, kh, Wo, pair -> (G, transposed)
    ((64, 7, 7, 112, False), (4, True)),       # resnet3d50 / nonlocal50 stem at 224²
    ((64, 7, 7, 32, False), (4, True)),
    ((64, 7, 7, 111, False), (4, True)),
    ((64, 7, 7, 113, False), (4, False)),      # rows up to 120 columns keep the 128-row tile
    ((64, 7, 7, 120, False), (4, False)),
    ((64, 7, 7, 250, False), (4, False)),      # several column tiles
    ((8, 5, 7, 32, False), (4, True)),         # SlowFast fast-path stem, 8 channels
    ((40, 3, 3, 56, False), (4, True)),
    ((64, 2, 7, 112, False), (4, True)),
    ((64, 1, 7, 112, False), (2, False)),      # 2-D stem: one tap per item
    ((64, 1, 7, 28, True), (2, False)),        # pair mode
    ((64, 7, 8, 112, False), (2, False)),      # kh = 8: no room for three ring stages
    ((64, 3, 13, 32, False), (2, False)),
    ((110, 7, 7, 112, False), (1, False)),     # BN = 128
    ((256, 7, 7, 56, False), (1, False)),
]


@pytest.mark.parametrize("args,want", RULE_CASES, ids=["K%d_kt%d_kh%d_Wo%d_pair%d" % c[0] for c in RULE_CASES])
def test_rule(lib, args, want):
    assert plan(lib, *args) == want


@pytest.mark.parametrize("args", [(64, 7, 7, 112, False), (8, 5, 7, 32, False), (64, 1, 7, 112, False), (64, 7, 7, 120, False)])
def test_force_four_rows_refuses_transposed(lib, args):
    assert plan(lib, *args, force=4) == (4, False)


def test_force_transposed(lib):
    assert plan(lib, 64, 7, 7, 112, False, force=FORCE_T) == (4, True)
    assert plan(lib, 64, 1, 7, 112, False, force=FORCE_T) == (4, True)       # 2-D stem, on request
    assert plan(lib, 64, 7, 7, 120, False, force=FORCE_T) == (4, False)      # wider than 112: the four-row instance
    assert plan(lib, 64, 1, 7, 28, True, force=FORCE_T) == (2, False)        # not eligible for four rows
    assert plan(lib, 64, 7, 8, 112, False, force=FORCE_T) == (2, False)
    assert plan(lib, 110, 7, 7, 112, False, force=FORCE_T) == (1, False)


def test_force_two_rows(lib):
    assert plan(lib, 64, 7, 7, 112, False, force=2) == (2, False)
