"""GPU (-m gpu): the slab kernel's 128-wide transposed form (b2_slab_t128.cuh) against fp64 and against the slab kernel.

Every case forces the form (b2_debug_set_slab_t128(1): small shapes fall below the rule's item count) and pins the launch by its
kernel id and plan; it is held to the kernel-matrix bound of tests/kernel_ref.py, must leave the NaN sentinel rows around its out=
rows untouched and repeat bitwise, and its output must be bitwise the slab kernel's with the form off (same accumulation order per
element, same epilogue expression).  Shapes with several rounds of items per CTA exercise the persistent path (staging-tile
hand-over, ring phases and slab prefetch across items).  A resnet3d50 forward, eager and graph-replayed, is bitwise the same with
the form on and off, with the form's stride-1 and stride-2 launches recorded."""
import ctypes
import os

import pytest
import torch

from oracle import functional as OF
from tests.conftest import has_h100
from tests.test_gpu_kernel_matrix import KNOB_ENV, SLAB, assert_within, last_kernel, make

pytestmark = [
    pytest.mark.gpu,
    pytest.mark.skipif(not has_h100(), reason="needs an H100"),
    pytest.mark.skipif(any(os.environ.get(e) for e in KNOB_ENV),
                       reason="a dispatch override is set in the environment (%s)" % ", ".join(KNOB_ENV)),
]

SLAB_T128 = 15                     # KID_SLAB_T128 of csrc/b2_host.h


@pytest.fixture(autouse=True)
def lib():
    from pretorched_x_b200 import _lib
    lib = _lib.load()
    lib.b2_debug_set_slab_t128.argtypes = [ctypes.c_int]
    try:
        yield lib
    finally:
        lib.b2_debug_set_slab_t128(-1)
        lib.b2_debug_set_densem(-1, 0)


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


K3, K2 = (3, 3, 3), (1, 3, 3)
P3, P2 = (1, 1, 1), (0, 1, 1)
# name, N, Cin, pitch, T, H, W, K, kernel, stride, padding, (NP, rows per item)
CASES = [
    ("s1_t4_28x28_k128", 1, 128, 128, 4, 28, 28, 128, K3, (1, 1, 1), P3, (216, 7)),
    ("s1_t2_14x14_k256", 2, 256, 256, 2, 14, 14, 256, K3, (1, 1, 1), P3, (224, 14)),
    ("s1_t1_14x14_k512_centre_tap", 1, 128, 128, 1, 14, 14, 512, K3, (1, 1, 1), P3, (224, 14)),
    ("s2_t4_56_to_28_k128", 1, 128, 128, 4, 56, 56, 128, K3, (2, 2, 2), P3, (216, 7)),
    ("s2_t2_28_to_14_k256", 2, 256, 256, 2, 28, 28, 256, K3, (2, 2, 2), P3, (216, 14)),
    ("s2_spatial_only_t4_28_to_14_k128", 1, 192, 192, 4, 28, 28, 128, K3, (1, 2, 2), P3, (216, 14)),
    ("2d_28x28_k128", 3, 128, 128, 1, 28, 28, 128, K2, (1, 1, 1), P2, (216, 7)),
    ("2d_14x14_k256", 3, 256, 256, 1, 14, 14, 256, K2, (1, 1, 1), P2, (224, 14)),
    ("2d_s2_28_to_14_k512", 2, 64, 64, 1, 28, 28, 512, K2, (1, 2, 2), P2, (216, 14)),
    ("np256_13x17_k128", 2, 64, 64, 2, 13, 17, 128, K3, (1, 1, 1), P3, (256, 13)),
    ("ragged_rows_15x28_k128", 1, 128, 128, 3, 15, 28, 128, K3, (1, 1, 1), P3, (256, 8)),
]


def conv_out(lib, pb, relu):
    """fp16 output through ops.conv into rows [pad, pad + M) of a NaN-filled buffer: (buffer, out rows, (kernel id, info))."""
    from pretorched_x_b200 import ops
    pad = 3
    buf = torch.full((pb.M + 2 * pad, pb.ldy), float("nan"), dtype=torch.float16, device=pb.a.data.device)
    out = buf[pad:pad + pb.M]
    ops.conv(pb.a, pb.pc, relu=relu, out=out)
    torch.cuda.synchronize()
    return buf, out, last_kernel(lib)


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
@pytest.mark.parametrize("relu", [True, False], ids=["relu", "affine"])
def test_slab_t128_against_fp64_and_slab(dev, lib, case, relu):
    lib.b2_debug_set_densem(0, 0)                          # small planes: keep them off the dense-M kernel
    lib.b2_debug_set_slab_t128(1)
    pb = make(dev, case[:11])
    buf, got, (kid, info) = conv_out(lib, pb, relu)
    assert kid == SLAB_T128 and info[:4] == case[11] + (128, case[9][1]), (kid, info)
    ref, A = pb.ref(relu=relu)
    assert_within("slab_t128 %s%s" % (pb.name, " relu" if relu else ""), got[:, :pb.K], ref, A, True)
    assert torch.isnan(buf[:3].float()).all() and torch.isnan(buf[3 + pb.M:].float()).all(), "rows outside out= were written"
    _, again, _ = conv_out(lib, pb, relu)
    assert torch.equal(again.view(torch.int16), got.view(torch.int16)), "two identical calls differ"
    lib.b2_debug_set_slab_t128(0)
    _, want, (kid0, _) = conv_out(lib, pb, relu)
    assert kid0 == SLAB
    assert torch.equal(got.view(torch.int16), want.view(torch.int16)), "the transposed form differs from the slab kernel"


# name, N, Cin, pitch, T, H, W, K, kernel, stride, padding, (NP, rows per item): more than two items per SM
PERSISTENT = [
    ("persistent_s1_28x28_k256", 16, 128, 128, 4, 28, 28, 256, K3, (1, 1, 1), P3, (216, 7)),
    ("persistent_s2_56_to_28_k256", 12, 128, 128, 8, 56, 56, 256, K3, (2, 2, 2), P3, (216, 7)),
]


@pytest.mark.parametrize("case", PERSISTENT, ids=[c[0] for c in PERSISTENT])
def test_slab_t128_persistent_items_bitwise(dev, lib, case):
    """Several items per CTA: every output element bitwise the slab kernel's, and a second call bitwise the first (no fp64
    reference at this size: the small cases above hold the same code to it)."""
    lib.b2_debug_set_densem(0, 0)
    lib.b2_debug_set_slab_t128(1)
    pb = make(dev, case[:11])
    buf, got, (kid, info) = conv_out(lib, pb, True)
    assert kid == SLAB_T128 and info[:4] == case[11] + (128, case[9][1]), (kid, info)
    items = pb.a.N * pb.To * -(-pb.Ho // case[11][1]) * (pb.K // 128)
    assert items > 2 * torch.cuda.get_device_properties(dev).multi_processor_count
    assert torch.isfinite(got.float()).all()
    assert torch.isnan(buf[:3].float()).all() and torch.isnan(buf[3 + pb.M:].float()).all(), "rows outside out= were written"
    _, again, _ = conv_out(lib, pb, True)
    assert torch.equal(again.view(torch.int16), got.view(torch.int16)), "two identical calls differ"
    lib.b2_debug_set_slab_t128(0)
    _, want, (kid0, _) = conv_out(lib, pb, True)
    assert kid0 == SLAB
    assert torch.equal(got.view(torch.int16), want.view(torch.int16)), "the transposed form differs from the slab kernel"


def test_resnet3d50_forward_bitwise_with_form_on_and_off(dev, lib, monkeypatch):
    """The dense-M kernel is off (at this size it would take the strided and layer3-4 convolutions), so the form runs at stride 1 and
    2; every convolution's kernel id is recorded through ops.conv."""
    import pretorched_x_b200 as P
    from pretorched_x_b200 import ops
    from pretorched_x_b200.graph import GraphedForward
    launched = []
    conv = ops.conv

    def recording_conv(*args, **kw):
        y = conv(*args, **kw)
        launched.append(last_kernel(lib))
        return y
    monkeypatch.setattr(ops, "conv", recording_conv)
    lib.b2_debug_set_densem(0, 0)
    torch.manual_seed(0)
    m = OF.randomize_bn_(P.resnet3d50(num_classes=400, pretrained=None), 1).eval().to(dev)
    x = OF.seeded_input((2, 3, 16, 112, 112), 5).to(dev)
    outs = {}
    for mode in (1, 0):
        lib.b2_debug_set_slab_t128(mode)
        launched.clear()
        with torch.no_grad():
            eager = m(x).clone()
        t128 = {info[3] for kid, info in launched if kid == SLAB_T128}
        assert t128 == ({1, 2} if mode else set()), launched
        g = GraphedForward(m, x)
        outs[mode] = (eager, g(x).clone())
        del g
    assert torch.isfinite(outs[1][0]).all()
    assert torch.equal(outs[1][0], outs[0][0]) and torch.equal(outs[1][1], outs[0][1]) and torch.equal(outs[1][0], outs[1][1])
