"""CPU: fine-tuning surface of the 2-D ResNets and of TRN -- parameter groups, requires_grad split, refused k and backbones,
TRN.get_optim_policies against the reference's groups (tests/golden/trn_optim_policies.pt), the torchvision blocks the
backward accepts, and the host-side plan of the (kt, kh, kw) weight-gradient entry point."""
import os

import pytest
import torch
import torch.nn as nn
import torchvision.models.resnet as tvresnet

import pretorched_x_b200 as P
from pretorched_x_b200 import _lib, engine
from pretorched_x_b200.models import resnet3d

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "trn_optim_policies.pt")

# (trainable, lr = 0) group counts per ft_begin_index, written out from the architectures.  resnet18 has 62 parameters: stem 3;
# BasicBlock 6, 9 with its 1x1 projection; layer1 = 12, layer2..4 = 15 each; head 2.  resnet50 has 161: stem 3; Bottleneck 9,
# 12 with its projection; layer1..4 = 30, 39, 57, 30; head 2 (the same counts as resnet3d50).
EXPECTED_COUNTS = {
    "resnet18": {1: (59, 3), 2: (47, 15), 3: (32, 30), 4: (17, 45), 5: (2, 60)},
    "resnet50": {1: (158, 3), 2: (128, 33), 3: (89, 72), 4: (32, 129), 5: (2, 159)},
}


def _expected_trainable(name, k):
    stage = name.split('.')[0]
    return stage == 'last_linear' or (stage.startswith('layer') and int(stage[5:]) >= k)


@pytest.mark.parametrize("arch", ["resnet18", "resnet50"])
@pytest.mark.parametrize("k", [1, 2, 3, 4, 5])
def test_2d_fine_tuning_groups_and_split(arch, k):
    model = getattr(P, arch)(num_classes=11, pretrained=None)
    groups = resnet3d.get_fine_tuning_parameters(model, k)
    named = list(model.named_parameters())
    assert len(groups) == len(named)
    assert (sum(set(g) == {'params'} for g in groups), sum('lr' in g for g in groups)) == EXPECTED_COUNTS[arch][k]
    for grp, (n, p) in zip(groups, named):
        assert grp['params'] is p, n
        trainable = _expected_trainable(n, k)
        assert p.requires_grad == trainable, n
        assert set(grp) == ({'params'} if trainable else {'params', 'lr'}), n
    assert model.ft_begin_index == k
    torch.optim.SGD(groups, lr=1e-3, momentum=0.9)


@pytest.mark.parametrize("arch", ["resnet18", "resnet50"])
def test_2d_fine_tune_refuses_stem_and_bad_index(arch):
    model = getattr(P, arch)(num_classes=5, pretrained=None)
    with pytest.raises(NotImplementedError, match="stem"):
        model.fine_tune(0)
    with pytest.raises(ValueError):
        model.fine_tune(6)
    assert model.ft_begin_index is None
    assert all(p.requires_grad for p in model.parameters())


@pytest.mark.parametrize("arch", ["resnet34", "resnet101", "resnet152"])
def test_other_2d_depths_are_accepted(arch):
    getattr(P, arch)(num_classes=5, pretrained=None).fine_tune(1)


def test_torchvision_blocks_outside_the_backward_are_refused():
    grouped = tvresnet.Bottleneck(256, 64, groups=32, base_width=4)                   # ResNeXt-style 3x3
    dilated = tvresnet.Bottleneck(256, 64, dilation=2)
    biased = tvresnet.BasicBlock(64, 64)
    biased.conv1 = nn.Conv2d(64, 64, 3, padding=1, bias=True)
    pooled = tvresnet.BasicBlock(64, 128, stride=2, downsample=nn.Sequential(nn.AvgPool2d(2), nn.Conv2d(64, 128, 1, bias=False),
                                                                              nn.BatchNorm2d(128)))
    for blk in (grouped, dilated, biased, pooled):
        with pytest.raises(NotImplementedError, match=type(blk).__name__):
            engine.check_trainable_block(blk)
    engine.check_trainable_block(tvresnet.Bottleneck(256, 128, stride=2, downsample=nn.Sequential(
        nn.Conv2d(256, 512, 1, stride=2, bias=False), nn.BatchNorm2d(512))))


def _trn(consensus="MSTRN", arch="resnet18", **kw):
    kw = kw or dict(frame_bottleneck_dim=128, video_feature_dim=64)
    return P.TRN(10, num_segments=8, arch=arch, consensus=consensus, pretrained=None, **kw)


@pytest.mark.parametrize("consensus", ["TRN", "HTRN", "MSTRN"])
@pytest.mark.parametrize("k", [3, 4])
def test_trn_fine_tune_split(consensus, k):
    model = _trn(consensus).fine_tune(k)
    for n, p in model.named_parameters():
        parts = n.split('.')
        if parts[0] == 'base_model':
            trainable = parts[1].startswith('layer') and int(parts[1][5:]) >= k
        else:
            trainable = parts[0] in ('temporal_relation', 'last_linear')
        assert p.requires_grad == trainable, n
    assert model.base_model.ft_begin_index == k


def test_trn_fine_tune_refuses_backbone_without_fine_tune():
    model = _trn("TRN", arch="mobilenetv2")
    with pytest.raises(NotImplementedError, match="mobilenetv2"):
        model.fine_tune(4)


def _named(model, groups):
    names = {id(p): n for n, p in model.named_parameters()}
    return [dict(name=g['name'], lr_mult=g['lr_mult'], decay_mult=g['decay_mult'], params=[names[id(p)] for p in g['params']])
            for g in groups]


def _policy_cases():
    return sorted(torch.load(GOLDEN, weights_only=False)["cases"])


@pytest.mark.parametrize("case", _policy_cases())
@pytest.mark.parametrize("pbn", [True, False])
def test_trn_optim_policies_match_reference(case, pbn):
    fx = torch.load(GOLDEN, weights_only=False)["cases"][case]
    model = P.TRN(10, num_segments=fx["segments"], arch=fx["arch"], consensus=fx["consensus"], pretrained=None, **fx["kwargs"])
    model.partialBN(pbn)
    got = _named(model, model.get_optim_policies())
    assert got == fx["policies"][pbn]
    if not pbn:                                          # with partial BN off every parameter is in exactly one group
        listed = [n for g in got for n in g["params"]]
        assert sorted(listed) == sorted(n for n, _ in model.named_parameters())


def test_trn_optim_policies_refuse_unknown_leaf_module():
    model = _trn("TRN")
    model.temporal_relation.extra = nn.PReLU()
    with pytest.raises(ValueError, match="PReLU"):
        model.get_optim_policies()


def test_wgrad_thw_symbols_exported_and_abi_unchanged():
    lib = _lib.load()
    for name in ("b2_conv_wgrad_thw", "b2_conv_wgrad_thw_workspace_elems"):
        assert name in _lib.SYMBOLS and hasattr(lib, name)
    assert lib.b2_version() == 103


@pytest.mark.parametrize("shape", [(2, 1, 14, 14, 256, 256), (3, 4, 13, 9, 64, 128), (1, 8, 56, 56, 64, 64)])
def test_wgrad_thw_workspace(shape):
    """The cubic entry's plan is the (k, k, k) plan of the new one; a (1, 3, 3) filter needs a third of the 3x3x3 workspace."""
    lib = _lib.load()
    for k, s in ((1, 1), (1, 2), (3, 1), (3, 2)):
        assert lib.b2_conv_wgrad_workspace_elems(*shape, k, s, k // 2) == \
            lib.b2_conv_wgrad_thw_workspace_elems(*shape, k, k, k, s, s, k // 2, k // 2)
    if shape[1] == 1:
        assert 3 * lib.b2_conv_wgrad_thw_workspace_elems(*shape, 1, 3, 3, 1, 1, 0, 1) == \
            lib.b2_conv_wgrad_thw_workspace_elems(*shape, 3, 3, 3, 1, 1, 1, 1)
