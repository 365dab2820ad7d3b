"""CPU: the stem convolution's row plan (b2_stemconv.cuh, stem_row_plan) behind a debug entry point.  Slab row i feeds local
output rows g_lo..g_hi through taps dh = i - 2g, read from consecutive weight-image slots starting at the slot of dh(g_lo).  Every
(output row, dh) pair must be covered exactly once, and each output row must see its taps in ascending dh order (slab rows are
issued in ascending order), which is what keeps the G = 1, 2 and 4 instances bit-identical."""
import ctypes

import pytest


def stem_slot(dh, kh):
    emax = ((kh - 1) // 2) * 2
    n_even = emax // 2 + 1
    omax = ((kh - 2) // 2) * 2 + 1 if kh >= 2 else -1
    return (emax - dh) // 2 if dh % 2 == 0 else n_even + (omax - dh) // 2


@pytest.fixture(scope="module")
def plan():
    from pretorched_x_b200 import _lib
    lib = _lib.load()
    lib.b2_debug_stem_row_plan.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_int)]

    def get(G, kh):
        out = (ctypes.c_int * 48)()
        rows = lib.b2_debug_stem_row_plan(G, kh, out)
        return rows, [tuple(out[3 * i:3 * i + 3]) for i in range(max(rows, 0))]
    return get


@pytest.mark.parametrize("G", [1, 2, 4])
@pytest.mark.parametrize("kh", range(1, 8))
def test_every_tap_once_in_ascending_order(plan, G, kh):
    rows, p = plan(G, kh)
    assert rows == 2 * (G - 1) + kh
    seen = {g: [] for g in range(G)}
    for i, (g_lo, g_hi, slot) in enumerate(p):
        if g_lo > g_hi:
            continue
        assert 0 <= g_lo <= g_hi < G
        for g in range(g_lo, g_hi + 1):
            dh = i - 2 * g
            assert 0 <= dh < kh
            assert stem_slot(dh, kh) == slot + (g - g_lo)      # the stacked taps are consecutive slots of the image
            seen[g].append(dh)
    for g in range(G):
        assert seen[g] == list(range(kh))                       # every tap once, ascending


def test_plan_refuses_too_many_slab_rows(plan):
    assert plan(4, 11)[0] == -1                                  # 2 * 3 + 11 > 16 slab rows
    assert plan(4, 10)[0] == 16
