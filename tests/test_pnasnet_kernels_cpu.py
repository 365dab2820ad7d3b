"""CPU: the PNASNet-5 kernels' contracts (no GPU needed).

1. The fp64 references of tests/pnasnet_kernel_ref.py against the reference model's own formulation, module by module
   (pnasnet.py:33-146): a branch's ZeroPad2d((1, 0, 1, 0)) -> depthwise convolution at padding K/2 -> [1:, 1:] crop is the
   depthwise convolution at pad = K/2 - 1 with the ceil extent; the zero-pad max-pool is the ceil-extent pool with padding 0;
   FactorizedReduction's two paths are the offset gathers at offsets 0 and 1; a 54-channel tensor stored at pitch 56 with zero
   taps in the pad channels gives the same result and zero pad channels.
2. The C entries' declarations, ctypes bindings, argument checks and spill-free sm_90a instances; the wrappers' argument checks.
"""
import os
import re

import pytest
import torch
import torch.nn as nn

from pretorched_x_b200 import _lib, ops, ops_pnasnet
from tests import pnasnet_kernel_ref as PR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _signed(shape, seed):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed), dtype=torch.float64)


# ---------------------------------------------------------------------------------------------
# 1. the decompositions, in fp64
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", (3, 5, 7))
@pytest.mark.parametrize("hw", (42, 21, 13))
def test_zero_pad_branch_is_the_convolution_at_pad_k_half_minus_one(k, hw):
    """relu_1 -> ZeroPad2d((1, 0, 1, 0)) -> depthwise_conv2d (stride 2, padding k // 2) -> [1:, 1:] (pnasnet.py:86-92)."""
    C = 8
    x = _signed((2, C, hw, hw), k * 100 + hw)
    conv = nn.Conv2d(C, C, k, stride=2, padding=k // 2, groups=C, bias=False).double()
    with torch.no_grad():
        conv.weight.copy_(_signed((C, 1, k, k), 7))
        want = conv(nn.ZeroPad2d((1, 0, 1, 0))(torch.relu(x)))[:, :, 1:, 1:]
    Ho = want.shape[2]
    assert Ho == hw // 2                                   # 42 -> 21, not the 22 the convolution computes before the crop
    wk = conv.weight.detach().reshape(C, k * k).t()
    got, _ = PR.dw_kxk_relu_in_ref(x.permute(0, 2, 3, 1), wk, k, 2, k // 2 - 1, Ho, Ho)
    assert torch.allclose(got, want.permute(0, 2, 3, 1).reshape(-1, C), rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("k,stride,hw", [(3, 1, 11), (5, 1, 21), (7, 1, 42), (3, 2, 165), (5, 2, 83), (7, 2, 21), (7, 2, 9)])
def test_branch_convolution_is_the_kxk_reference(k, stride, hw):
    C = 8
    x = _signed((1, C, hw, hw), k + hw)
    conv = nn.Conv2d(C, C, k, stride=stride, padding=k // 2, groups=C, bias=False).double()
    with torch.no_grad():
        conv.weight.copy_(_signed((C, 1, k, k), 3))
        want = conv(torch.relu(x))
    Ho = want.shape[2]
    got, A = PR.dw_kxk_relu_in_ref(x.permute(0, 2, 3, 1), conv.weight.detach().reshape(C, k * k).t(), k, stride, k // 2, Ho, Ho)
    assert torch.allclose(got, want.permute(0, 2, 3, 1).reshape(-1, C), rtol=1e-12, atol=1e-12)
    assert torch.all(A >= got.abs() - 1e-12)


@pytest.mark.parametrize("hw", (42, 21, 83))
def test_zero_pad_max_pool_is_the_ceil_pool_without_padding(hw):
    """MaxPool(3, stride 2, zero_pad=True) (pnasnet.py:33-46) is nn.MaxPool2d(3, 2, 0, ceil_mode=True), the pool the slice kernel
    runs with the extent of ops.ceil_pool_dim."""
    x = _signed((2, 8, hw, hw), hw)
    want = nn.MaxPool2d(3, stride=2, padding=1)(nn.ZeroPad2d((1, 0, 1, 0))(x))[:, :, 1:, 1:]
    got = nn.MaxPool2d(3, stride=2, padding=0, ceil_mode=True)(x)
    assert torch.equal(got, want)
    assert want.shape[2] == ops.ceil_pool_dim(hw, 3, 2, 0)


@pytest.mark.parametrize("hw", (165, 83, 42, 21))
def test_factorized_reduction_paths_are_offset_gathers(hw):
    """path_1: AvgPool2d(1, 2) reads x[2i, 2j]; path_2: ZeroPad2d((0, 1, 0, 1)) -> [1:, 1:] -> AvgPool2d(1, 2) reads x[2i + 1, 2j + 1],
    zero past the far edge of an odd map (pnasnet.py:117-146)."""
    C = 8
    x = torch.relu(_signed((2, C, hw, hw), hw))
    p1 = nn.AvgPool2d(1, stride=2, count_include_pad=False)(x)
    p2 = nn.AvgPool2d(1, stride=2, count_include_pad=False)(nn.ZeroPad2d((0, 1, 0, 1))(x)[:, :, 1:, 1:])
    xl = x.permute(0, 2, 3, 1)
    for path, off in ((p1, 0), (p2, 1)):
        assert torch.equal(PR.gather_offset_ref(xl, 2, off), path.permute(0, 2, 3, 1).reshape(-1, C))
    if hw % 2:
        assert torch.all(p2[:, :, -1, :] == 0) and torch.all(p2[:, :, :, -1] == 0)


def test_padded_slice_with_zero_taps_matches_and_keeps_pad_channels_zero():
    """A 54-channel tensor at pitch 56 (CellStem0's slices), pad channels zero, through the depthwise pass with zero taps there."""
    k, hw = 5, 21
    x = _signed((2, hw, hw, 54), 5)
    w = _signed((k * k, 54), 6)
    want, _ = PR.dw_kxk_relu_in_ref(x, w, k, 1, 2, hw, hw)
    xp = torch.cat([x, torch.zeros(2, hw, hw, 2, dtype=x.dtype)], -1)
    wp = torch.cat([w, torch.zeros(k * k, 2, dtype=w.dtype)], -1)
    got, _ = PR.dw_kxk_relu_in_ref(xp, wp, k, 1, 2, hw, hw)
    assert torch.equal(got[:, :54], want) and torch.all(got[:, 54:] == 0)


def test_network_cases_cover_every_map_and_width():
    cases = PR.network_cases()
    assert {c[3] for c in cases} == {56, 96, 112, 216, 432, 864}
    assert {(c[1], c[4], c[5]) for c in cases} == {(1, 83, 83), (1, 42, 42), (1, 21, 21), (1, 11, 11), (2, 165, 83), (2, 83, 42),
                                                  (2, 42, 21), (2, 21, 11)}
    for k, s, p, C, hw, Ho in cases:
        x = torch.zeros(1, 1, hw, hw)
        zp = s == 2 and p == k // 2 - 1
        conv = nn.Conv2d(1, 1, k, stride=s, padding=k // 2, bias=False)
        out = conv(nn.ZeroPad2d((1, 0, 1, 0))(x))[:, :, 1:, 1:] if zp else conv(x)
        assert out.shape[2] == Ho, (k, s, p, hw)


# ---------------------------------------------------------------------------------------------
# 2. the C entries and their wrappers
# ---------------------------------------------------------------------------------------------
def test_entries_are_declared_and_bound():
    with open(os.path.join(ROOT, "include", "b2_pretorched.h")) as f:
        header = f.read()
    assert re.search(r"int b2_dwconv_kxk_relu_in_ndhwc\(const void\* x, int ldx, const float\* w, void\* y, int ldy, int N, int H, "
                     r"int W, int C, int K, int stride,\s+int pad, int Ho, int Wo, void\* stream\);", header)
    assert re.search(r"int b2_shortcut_a_offset_ndhwc\(const void\* x, void\* y, int N, int H, int W, int C, int stride, int offset, "
                     r"int relu, int Cout,\s+void\* stream\);", header)
    for name, nargs in (("b2_dwconv_kxk_relu_in_ndhwc", 15), ("b2_shortcut_a_offset_ndhwc", 11)):
        assert len(_lib.SYMBOLS[name][1]) == nargs


def test_kxk_instances_compile_for_sm90a_without_spills():
    from pretorched_x_b200.csrc import build
    build.build()
    with open(os.path.join(os.path.dirname(build.LIB), "build.log")) as f:
        log = f.read()
    for k, s, r in ((3, 1, 6), (5, 1, 4), (7, 1, 4), (3, 2, 2), (5, 2, 2), (7, 2, 2)):
        inst = "ILi%dELi%dELi%dEE" % (k, s, r)
        m = re.search(r"Compiling entry function '_ZN2b217dwconv_kxk_kernel%s[^']*' for 'sm_90a'\n[^\n]*\n\s*(\d+) bytes stack frame, "
                      r"(\d+) bytes spill stores, (\d+) bytes spill loads" % inst, log)
        assert m, "dwconv_kxk_kernel %s not in the build log" % inst
        assert m.groups() == ("0", "0", "0"), (inst, m.groups())


def test_dwconv_entry_refuses_bad_arguments():
    lib = _lib.load()
    buf = torch.zeros(1 << 16, dtype=torch.float32)
    p = buf.data_ptr()
    y = p + 4096 * 16                                      # far enough past x for the small shapes below
    ok = (p, 8, p, y, 8, 1, 4, 4, 8, 3, 1, 1, 4, 4, None)

    def call(**kw):
        names = ("x", "ldx", "w", "y", "ldy", "N", "H", "W", "C", "K", "stride", "pad", "Ho", "Wo", "stream")
        args = dict(zip(names, ok))
        args.update(kw)
        return lib.b2_dwconv_kxk_relu_in_ndhwc(*[args[n] for n in names])

    assert call(x=None) == -1 and "null" in _lib.last_error()
    for bad in (dict(K=4), dict(K=9), dict(K=1)):
        assert call(**bad) == -1 and "kernel size" in _lib.last_error()
    assert call(stride=3) == -1 and "stride" in _lib.last_error()
    assert call(C=12, ldx=16, ldy=16) == -1 and "multiple of 8" in _lib.last_error()
    assert call(ldx=12) == -1 and "pitch" in _lib.last_error()
    assert call(C=16, ldx=16, ldy=8) == -1 and "pitch" in _lib.last_error()
    assert call(pad=2) == -1 and "padding" in _lib.last_error()
    assert call(pad=-1) == -1 and "padding" in _lib.last_error()
    assert call(Ho=6) == -1 and "past" in _lib.last_error()
    assert call(Ho=0) == -1 and "empty" in _lib.last_error()
    assert call(y=p + 4) == -1 and "aligned" in _lib.last_error()
    assert call(y=p + 16 * 8) == -1 and "overlaps" in _lib.last_error()


def test_gather_entry_refuses_bad_arguments():
    lib = _lib.load()
    buf = torch.zeros(4096, dtype=torch.float32)
    p = buf.data_ptr()
    assert lib.b2_shortcut_a_offset_ndhwc(None, p, 1, 4, 4, 8, 2, 1, 0, 8, None) == -1
    assert lib.b2_shortcut_a_offset_ndhwc(p, p + 8192, 1, 4, 4, 8, 2, 2, 0, 8, None) == -1 and "offset" in _lib.last_error()
    assert lib.b2_shortcut_a_offset_ndhwc(p, p + 8192, 1, 4, 4, 8, 3, 1, 0, 8, None) == -1 and "stride" in _lib.last_error()
    assert lib.b2_shortcut_a_offset_ndhwc(p, p + 8192, 1, 4, 4, 12, 2, 1, 0, 16, None) == -1
    assert lib.b2_shortcut_a_offset_ndhwc(p + 4, p + 8192, 1, 4, 4, 8, 2, 1, 0, 8, None) == -1 and "aligned" in _lib.last_error()


def test_wrappers_validate_their_arguments():
    a = ops.Act(torch.zeros((2 * 5 * 5, 56), dtype=torch.float16), 2, 1, 5, 5, 56)
    w = torch.zeros((25, 56), dtype=torch.float32)
    with pytest.raises(RuntimeError, match="CUDA"):
        ops_pnasnet.dwconv_kxk_relu_in(a, w, 5, 1, 2, 5, 5)
    with pytest.raises(ValueError, match="k in"):
        ops_pnasnet.dwconv_kxk_relu_in(a, w, 4, 1, 2, 5, 5)
    with pytest.raises(ValueError, match="stride 1 or 2"):
        ops_pnasnet.dwconv_kxk_relu_in(a, w, 5, 3, 2, 5, 5)
    bad = ops.Act(torch.zeros((50, 56), dtype=torch.float16), 2, 1, 5, 5, 54)
    with pytest.raises(ValueError, match="C % 8 == 0"):
        ops_pnasnet.dwconv_kxk_relu_in(bad, torch.zeros((25, 54)), 5, 1, 2, 5, 5)
    for w_bad in (torch.zeros((56, 25)), torch.zeros((25, 56), dtype=torch.float64), torch.zeros((25, 112))[:, ::2],
                  torch.zeros((9, 56))):
        with pytest.raises(ValueError, match=r"fp32 \[25\]\[56\]"):
            ops_pnasnet.dwconv_kxk_relu_in(a, w_bad, 5, 1, 2, 5, 5)
    clip = ops.Act(torch.zeros((100, 56), dtype=torch.float16), 2, 2, 5, 5, 56)
    with pytest.raises(ValueError, match="images"):
        ops_pnasnet.gather_offset(clip, 2, 1)
    with pytest.raises(RuntimeError, match="CUDA"):
        ops_pnasnet.gather_offset(a, 2, 1)
