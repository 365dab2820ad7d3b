"""CPU: which consecutive bottlenecks the engine chains (engine._chains / _chained_pairs: the closing 1x1x1 GEMM of one block also
computes the next block's conv1, b2_gemm_chain_f16).  Unit 0 is the stem, units 1..3 are layer1."""
import pytest
import torch.nn as nn

import pretorched_x_b200 as P
from pretorched_x_b200 import engine


def pairs(model, simt=False):
    return sorted(engine._chained_pairs(engine._trunk_units(model), simt))


@pytest.mark.parametrize("name", ["resnet3d50", "resnet3d101", "nonlocalresnet3d50"])
def test_layer1_pairs_chain_3d(name):
    """layer1.0 -> 1.1 -> 1.2 -> layer2.0: the only closing GEMMs of at most 256 columns."""
    assert pairs(getattr(P, name)(num_classes=10, pretrained=None)) == [1, 2, 3]


def test_layer1_pairs_chain_2d():
    assert pairs(P.resnet50(num_classes=10, pretrained=None)) == [1, 2, 3]


def test_no_chain_under_simt():
    assert pairs(P.resnet3d50(num_classes=10, pretrained=None), simt=True) == []


def test_no_chain_for_basic_blocks_or_preactivation():
    assert pairs(P.resnet3d18(num_classes=10, pretrained=None)) == []
    assert pairs(P.preact_resnet3d50(num_classes=10)) == []


def test_no_chain_after_a_nonlocal_block():
    model = P.nonlocalresnet3d50(num_classes=10, pretrained=None)
    blk, nxt = model.layer1[1], model.layer1[2]
    assert engine._chains(blk, nxt)
    blk.nonlocal_layer = True
    blk.nonlocalblock = nn.Identity()
    assert not engine._chains(blk, nxt)
    assert pairs(model) == [1, 3]


def test_no_chain_into_a_biased_or_strided_conv1():
    model = P.resnet3d50(num_classes=10, pretrained=None)
    nxt = model.layer1[1]
    nxt.conv1 = nn.Conv3d(256, 64, kernel_size=1, bias=True)
    assert pairs(model) == [2, 3]
    nxt.conv1 = nn.Conv3d(256, 64, kernel_size=1, stride=2, bias=False)
    assert pairs(model) == [2, 3]


def test_no_chain_across_a_depth_first_segment(monkeypatch):
    """run_trunk hands each segment to _run_units on its own: a pair split by a segment boundary never chains."""
    model = P.resnet3d50(num_classes=10, pretrained=None)
    units = engine._trunk_units(model)
    assert sorted(engine._chained_pairs(units[:3], False)) == [1]          # stem, 1.0, 1.1 | 1.2, ...
    assert sorted(engine._chained_pairs(units[3:], False)) == [0]          # 1.2 -> 2.0


def test_frozen_prefix_of_finetune_chains_but_not_into_trainable_blocks():
    """run_trunk_finetune: the frozen prefix runs through _run_units (its inner pairs chain); its last unit has no successor in
    that list, so a block that goes through BlockTrainFunction never receives a chained h1."""
    model = P.resnet3d50(num_classes=10, pretrained=None)
    units = engine._trunk_units(model)
    n_frozen = 1 + len(model.layer1)                                       # fine_tune(2): stem + layer1 frozen
    assert sorted(engine._chained_pairs(units[:n_frozen], False)) == [1, 2]
