"""CPU: the grouped-convolution surface that needs no device -- the three C-ABI entries, the packed-filter size arithmetic, and
the route ``engine.packed_conv`` takes for a grouped convolution (group-aware pack inside the kernel's contract, block-diagonal
dense filter outside it), decided from the shape alone."""
import pytest
import torch.nn as nn

import pretorched_x_b200 as P
from pretorched_x_b200 import _lib, engine, ops


def test_library_exports_grouped_entries_and_keeps_abi():
    lib = _lib.load()
    for name in ("b2_pack_grouped_conv_weight_elems", "b2_pack_grouped_conv_weight", "b2_conv_grouped_ndhwc_fprop"):
        assert hasattr(lib, name) and name in _lib.SYMBOLS
    assert lib.b2_version() == 103


@pytest.mark.parametrize("kt", [1, 3])
@pytest.mark.parametrize("cg", [4, 8, 16, 32])
def test_packed_elems(cg, kt):
    lib = _lib.load()
    K = 32 * cg
    block = 32 if cg == 32 else 16
    assert lib.b2_pack_grouped_conv_weight_elems(K, cg, 32, kt, 3, 3) == K * block * kt * 9


def test_packed_elems_outside_contract_is_zero():
    lib = _lib.load()
    assert lib.b2_pack_grouped_conv_weight_elems(64, 2, 32, 3, 3, 3) == 0        # 2 channels per group
    assert lib.b2_pack_grouped_conv_weight_elems(96, 8, 12, 3, 3, 3) == 0        # K not a multiple of 64
    assert lib.b2_pack_grouped_conv_weight_elems(128, 4, 16, 3, 3, 3) == 0       # cg * groups != K
    assert lib.b2_pack_grouped_conv_weight_elems(128, 4, 32, 3, 1, 1) == 0       # not 3x3 in plane
    assert lib.b2_pack_grouped_conv_weight_elems(128, 4, 32, 5, 3, 3) == 0


def test_resnext3d50_conv2_takes_the_grouped_route():
    m = P.resnext3d50(num_classes=10)
    convs = [blk.conv2 for ln in ("layer1", "layer2", "layer3", "layer4") for blk in getattr(m, ln)]
    assert len(convs) == 16 and {c.weight.shape[1] for c in convs} == {4, 8, 16, 32}
    assert all(engine.grouped_route(c) for c in convs)
    assert not any(engine.grouped_route(c) for c in m.modules() if isinstance(c, nn.Conv3d) and c.groups == 1)


def test_grouped_convolutions_outside_the_contract_stay_dense():
    assert engine.grouped_route(nn.Conv3d(128, 128, 3, 2, 1, groups=32, bias=False))
    assert engine.grouped_route(nn.Conv2d(256, 256, 3, 1, 1, groups=32, bias=False))      # 2-D 3x3: kt = 1
    assert engine.grouped_route(nn.Conv3d(512, 512, (1, 3, 3), 1, (0, 1, 1), groups=32, bias=False))
    for conv in (nn.Conv3d(128, 256, 3, 1, 1, groups=32, bias=False),          # C != K
                 nn.Conv3d(64, 64, 3, 1, 1, groups=32, bias=False),            # 2 channels per group
                 nn.Conv3d(96, 96, 3, 1, 1, groups=12, bias=False),            # C % 64 != 0
                 nn.Conv3d(128, 128, 1, 1, 0, groups=32, bias=False),          # grouped 1x1x1
                 nn.Conv3d(128, 128, 3, 1, 0, groups=32, bias=False),          # no padding
                 nn.Conv3d(128, 128, 3, (1, 2, 1), 1, groups=32, bias=False),  # unequal in-plane strides
                 nn.Conv3d(128, 128, 3, 1, 1, bias=False)):                    # not grouped
        assert not engine.grouped_route(conv), conv
    assert not ops.grouped_pack_applies(128, 128, 32, (3, 3, 3), (3, 3, 3), (1, 1, 1))
