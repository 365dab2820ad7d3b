"""CPU: the fine-tuning surface of the 3-D ResNets (parameter groups, requires_grad split, refused block families) and the
index algebra of the strided backward (zero insertion / shortcut-A adjoint) that the GPU kernels implement."""
import pytest
import torch
import torch.nn.functional as F

import pretorched_x_b200 as P
from pretorched_x_b200 import engine
from pretorched_x_b200.models import resnet3d


# (trainable, lr = 0) group counts per ft_begin_index, written out from the architectures: resnet3d50 has 161 parameters
# (stem 3; Bottleneck 9, 12 with its type-B projection; layer1..4 = 30, 39, 57, 30; head 2), resnet3d18 with type-A shortcuts
# has 53 (stem 3; BasicBlock 6; 12 per stage; head 2).  The reference's substring rule would put the 2 head parameters
# (named last_linear after modify_resnets) in the lr = 0 column as well.
EXPECTED_COUNTS = {
    "resnet3d50": {1: (158, 3), 2: (128, 33), 3: (89, 72), 4: (32, 129), 5: (2, 159)},
    "resnet3d18": {1: (50, 3), 2: (38, 15), 3: (26, 27), 4: (14, 39), 5: (2, 51)},
}


def _expected_trainable(name, k):
    stage = name.split('.')[0]
    return stage == 'last_linear' or (stage.startswith('layer') and int(stage[5:]) >= k)


@pytest.mark.parametrize("arch", ["resnet3d18", "resnet3d50"])
@pytest.mark.parametrize("k", [1, 2, 3, 4, 5])
def test_get_fine_tuning_parameters_matches_reference_layout(arch, k):
    model = getattr(P, arch)(num_classes=11, pretrained=None)
    groups = resnet3d.get_fine_tuning_parameters(model, k)
    named = list(model.named_parameters())
    assert len(groups) == len(named)
    assert (sum(set(g) == {'params'} for g in groups), sum('lr' in g for g in groups)) == EXPECTED_COUNTS[arch][k]
    for grp, (n, p) in zip(groups, named):
        assert grp['params'] is p, n
        trainable = _expected_trainable(n, k)
        if trainable:
            assert set(grp) == {'params'}, n
        else:
            assert set(grp) == {'params', 'lr'} and grp['lr'] == 0.0, n
    # the head is trainable here, where the reference's 'fc' test would freeze last_linear
    assert all(set(g) == {'params'} for g, (n, _) in zip(groups, named) if n.startswith('last_linear.'))
    assert model.ft_begin_index == k
    torch.optim.SGD(groups, lr=1e-3, momentum=0.9)          # the groups are a valid optimizer argument


@pytest.mark.parametrize("k", [1, 3, 4, 5])
def test_fine_tune_sets_requires_grad(k):
    model = P.resnet3d50(num_classes=5, pretrained=None).fine_tune(k)
    for n, p in model.named_parameters():
        stage = n.split('.')[0]
        trainable = stage == 'last_linear' or (stage.startswith('layer') and int(stage[5:]) >= k)
        assert p.requires_grad == trainable, n


def test_fine_tune_refuses_stem_and_bad_index():
    model = P.resnet3d18(num_classes=5, pretrained=None)
    with pytest.raises(NotImplementedError):
        model.fine_tune(0)
    with pytest.raises(NotImplementedError):
        resnet3d.get_fine_tuning_parameters(model, 0)
    with pytest.raises(ValueError):
        model.fine_tune(6)
    assert model.ft_begin_index is None
    assert all(p.requires_grad for p in model.parameters())


def _unsupported_models():
    return {
        "preact_resnet3d18": lambda: P.preact_resnet3d18(num_classes=5),
        "r2plus1d18": lambda: P.r2plus1d18(num_classes=5),
        "resnext3d50": lambda: P.resnext3d50(num_classes=5),
        "nonlocalresnet3d50": lambda: P.nonlocalresnet3d50(pretrained=None),
        "slowfast18": lambda: P.slowfast.resnet18(mode="sf", num_classes=5),
    }


@pytest.mark.parametrize("family", sorted(_unsupported_models()))
def test_unsupported_block_families_raise(family):
    model = _unsupported_models()[family]()
    blocks = [m for m in model.modules() if m is not model and hasattr(m, "conv1") and hasattr(m, "conv2")]   # residual blocks
    assert blocks, family
    for blk in blocks:
        with pytest.raises(NotImplementedError, match=type(blk).__name__):
            engine.check_trainable_block(blk)
    if hasattr(model, "fine_tune"):
        with pytest.raises(NotImplementedError):
            model.fine_tune(4)


def test_plain_blocks_are_accepted():
    for arch in ("resnet3d10", "resnet3d18", "resnet3d34", "resnet3d50", "resnet3d101", "resneti3d50"):
        model = getattr(P, arch)(num_classes=5, pretrained=None) if arch != "resnet3d10" else P.resnet3d10(num_classes=5)
        model.fine_tune(1)
    P.resnet3d18(num_classes=5, pretrained=None, shortcut_type='B').fine_tune(1)
    P.resnet3d50(num_classes=5, pretrained=None, shortcut_type='A').fine_tune(1)


# ---------------------------------------------------------------------------------------------
# index algebra of the strided backward (what b2_zero_insert_ndhwc + a stride-1 convolution compute)
# ---------------------------------------------------------------------------------------------
def zero_insert(g, size, stride, channels=None):
    """y[:, :, s*t, s*h, s*w] = g[:, :channels, t, h, w] on the full-resolution grid ``size``, zeros elsewhere (NCDHW)."""
    N, C = g.shape[:2]
    C = C if channels is None else channels
    y = g.new_zeros((N, C) + tuple(size))
    To, Ho, Wo = ((n - 1) // stride + 1 for n in size)
    assert tuple(g.shape[2:]) == (To, Ho, Wo)
    y[:, :, ::stride, ::stride, ::stride] = g[:, :C]
    return y


SIZES = [(1, 7, 7), (2, 7, 7), (3, 14, 14), (1, 5, 9), (4, 28, 28)]


@pytest.mark.parametrize("size", SIZES)
def test_strided_dgrad_is_zero_insert_then_flipped_stride1_conv(size):
    torch.manual_seed(0)
    Cin, Cout = 5, 6
    x = torch.randn((2, Cin) + size, dtype=torch.float64)
    w = torch.randn((Cout, Cin, 3, 3, 3), dtype=torch.float64)
    y = F.conv3d(x, w, stride=2, padding=1)
    g = torch.randn_like(y)
    want = torch.nn.grad.conv3d_input(x.shape, w, g, stride=2, padding=1)
    z = zero_insert(g, size, 2)
    got = F.conv3d(z, w.flip(2, 3, 4).transpose(0, 1), padding=1)
    assert got.shape == want.shape
    assert torch.allclose(got, want, atol=1e-10)


@pytest.mark.parametrize("size", SIZES)
def test_zero_insert_is_adjoint_of_shortcut_a(size):
    torch.manual_seed(1)
    from oracle import functional as OF
    x = torch.randn((2, 4) + size, dtype=torch.float64)
    ya = OF.shortcut_a(x, 8, 2)
    g = torch.randn_like(ya)
    lhs = (ya * g).sum()
    rhs = (x * zero_insert(g, size, 2, channels=4)).sum()
    assert torch.allclose(lhs, rhs)


@pytest.mark.parametrize("size", SIZES)
def test_strided_projection_dgrad_is_zero_insert_of_low_res_product(size):
    torch.manual_seed(2)
    x = torch.randn((2, 6) + size, dtype=torch.float64)
    w = torch.randn((10, 6, 1, 1, 1), dtype=torch.float64)
    g = torch.randn_like(F.conv3d(x, w, stride=2))
    want = torch.nn.grad.conv3d_input(x.shape, w, g, stride=2)
    low = torch.einsum('nkthw,kc->ncthw', g, w[:, :, 0, 0, 0])
    assert torch.allclose(zero_insert(low, size, 2), want, atol=1e-10)
