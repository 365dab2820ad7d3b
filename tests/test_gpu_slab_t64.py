"""GPU (-m gpu): the slab kernel's 64-wide transposed form (slab_t_kernel<64, NP>, b2_slab_t128.cuh) against fp64 and against the
slab kernel's 64-wide tile.

Every case forces the form (b2_debug_set_slab_t64(1): small shapes fall below the rule's item count) and pins the launch by its
kernel id and its plan ({NP, items, R} from the host-only plan view); it is held to the kernel-matrix bound of tests/kernel_ref.py,
must leave the NaN sentinel rows around its out= rows untouched, write zeros into the padding columns [K, ldy), repeat bitwise,
and its output must be bitwise the slab kernel's with the form off (same accumulation order per element, same epilogue
expression).  The planes are chosen so that the last item of a plane ends inside the second warpgroup's half, or leaves that half
wholly past the plane.  A resnet3d50 forward, eager and graph-replayed, is bitwise the same with the form on and off."""
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

SLAB_T64 = 16                      # KID_SLAB_T64 of csrc/b2_host.h
NP = 168


@pytest.fixture(autouse=True)
def lib():
    from pretorched_x_b200 import _lib
    lib = _lib.load()
    lib.b2_debug_set_slab_t64.argtypes = [ctypes.c_int]
    lib.b2_debug_slab_t64_plan.argtypes = [ctypes.POINTER(_lib.ConvArgs), ctypes.POINTER(ctypes.c_int)]
    try:
        yield lib
    finally:
        lib.b2_debug_set_slab_t64(-1)
        lib.b2_debug_set_densem(-1, 0)


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


K3, K2 = (3, 3, 3), (1, 3, 3)
P3, P2 = (1, 1, 1), (0, 1, 1)
# name, N, Cin, pitch, T, H, W, K, kernel, stride, padding
CASES = [
    # 56 x 58 = 3248 padded positions: nine items of 336 and one of 224 (the second warpgroup's half partly past the plane)
    ("t3_56x56", 1, 64, 64, 3, 56, 56, 64, K3, (1, 1, 1), P3),
    # 28 x 30 = 840: two items and one of 168 (the second warpgroup's half wholly past the plane)
    ("2d_28x28", 3, 64, 64, 1, 28, 28, 64, K2, (1, 1, 1), P2),
    # 20 x 24 = 480 = 336 + 144: the last item ends inside the first warpgroup's half
    ("t3_20x22", 2, 64, 64, 3, 20, 22, 64, K3, (1, 1, 1), P3),
    ("c128_two_chunks", 1, 128, 128, 3, 14, 15, 64, K3, (1, 1, 1), P3),
    ("k44_ldy48", 1, 64, 64, 3, 16, 18, 44, K3, (1, 1, 1), P3),
    ("k48_2d", 2, 64, 64, 1, 30, 31, 48, K2, (1, 1, 1), P2),
    ("s2_t4_33_to_17", 1, 64, 64, 4, 33, 33, 64, K3, (2, 2, 2), P3),
    ("valid_2d_30x30", 2, 64, 64, 1, 30, 30, 64, K2, (1, 1, 1), (0, 0, 0)),
]


def host_plan(lib, pb, out):
    """The plan view's {taken, applies, NP, R, items, ...} for the problem's convolution into out."""
    a = pb.args(out)
    plan = (ctypes.c_int * 9)()
    assert lib.b2_debug_slab_t64_plan(ctypes.byref(a), plan) == 0
    return list(plan)


def conv_out(lib, pb, relu):
    """fp16 output through ops.conv into rows [pad, pad + M) of a NaN-filled buffer: (buffer, out rows, (kernel id, info))."""
    from pretorched_x_b200 import ops
    pad = 3
    buf = torch.full((pb.M + 2 * pad, pb.ldy), float("nan"), dtype=torch.float16, device=pb.a.data.device)
    out = buf[pad:pad + pb.M]
    ops.conv(pb.a, pb.pc, relu=relu, out=out)
    torch.cuda.synchronize()
    return buf, out, last_kernel(lib)


def check_launch(lib, pb, out, kid, info):
    """The launch is the form's, with the plan the host-only view reports: NP, items of 2 NP padded positions, slab rows."""
    plan = host_plan(lib, pb, out)
    assert plan[1] == 1 and plan[2] == NP, plan
    P = pb.Ho * (pb.Wo + (2 if pb.s[2] == 1 else 1))       # padded positions of a plane: two halo columns, one at stride 2
    assert plan[4] == pb.a.N * pb.To * -(-P // (2 * NP)), (plan, P)
    assert kid == SLAB_T64 and info[:3] == (plan[2], plan[4], plan[3]), (kid, info, plan)


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
@pytest.mark.parametrize("relu", [True, False], ids=["relu", "affine"])
def test_slab_t64_against_fp64_and_slab(dev, lib, case, relu):
    lib.b2_debug_set_densem(0, 0)                          # small planes: keep them off the dense-M kernel
    lib.b2_debug_set_slab_t64(1)
    pb = make(dev, case)
    buf, got, (kid, info) = conv_out(lib, pb, relu)
    check_launch(lib, pb, got, kid, info)
    ref, A = pb.ref(relu=relu)
    assert_within("slab_t64 %s%s" % (pb.name, " relu" if relu else ""), got[:, :pb.K], ref, A, True)
    if pb.ldy > pb.K:
        assert torch.all(got[:, pb.K:].cpu() == 0), "padding columns [K, ldy) not zero"
    assert torch.isnan(buf[:3].float()).all() and torch.isnan(buf[3 + pb.M:].float()).all(), "rows outside out= were written"
    _, again, _ = conv_out(lib, pb, relu)
    assert torch.equal(again.view(torch.int16), got.view(torch.int16)), "two identical calls differ"
    lib.b2_debug_set_slab_t64(0)
    _, want, (kid0, _) = conv_out(lib, pb, relu)
    assert kid0 == SLAB
    assert torch.equal(got.view(torch.int16), want.view(torch.int16)), "the transposed form differs from the slab kernel"


# more than two items per SM: the staging-tile hand-over, ring phases and slab prefetch across items
PERSISTENT = [
    ("persistent_t3_56x56", 4, 64, 64, 8, 56, 56, 64, K3, (1, 1, 1), P3),
    ("persistent_2d_56x56_k48", 48, 64, 64, 1, 56, 56, 48, K2, (1, 1, 1), P2),
]


@pytest.mark.parametrize("case", PERSISTENT, ids=[c[0] for c in PERSISTENT])
def test_slab_t64_persistent_items_bitwise(dev, lib, case):
    """Several items per CTA: every output element bitwise the slab kernel's, and a second call bitwise the first (no fp64
    reference at this size: the small cases above hold the same code to it)."""
    lib.b2_debug_set_densem(0, 0)
    lib.b2_debug_set_slab_t64(1)
    pb = make(dev, case)
    buf, got, (kid, info) = conv_out(lib, pb, True)
    check_launch(lib, pb, got, kid, info)
    assert info[1] > 2 * torch.cuda.get_device_properties(dev).multi_processor_count
    assert torch.isfinite(got.float()).all()
    if pb.ldy > pb.K:
        assert torch.all(got[:, pb.K:].cpu() == 0), "padding columns [K, ldy) not zero"
    assert torch.isnan(buf[:3].float()).all() and torch.isnan(buf[3 + pb.M:].float()).all(), "rows outside out= were written"
    _, again, _ = conv_out(lib, pb, True)
    assert torch.equal(again.view(torch.int16), got.view(torch.int16)), "two identical calls differ"
    lib.b2_debug_set_slab_t64(0)
    _, want, (kid0, _) = conv_out(lib, pb, True)
    assert kid0 == SLAB
    assert torch.equal(got.view(torch.int16), want.view(torch.int16)), "the transposed form differs from the slab kernel"


def test_resnet3d50_forward_bitwise_with_form_on_and_off(dev, lib, monkeypatch):
    """Layer1's conv2 runs on the form when forced and on the slab kernel when off; every convolution's kernel id is recorded
    through ops.conv."""
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
        lib.b2_debug_set_slab_t64(mode)
        launched.clear()
        with torch.no_grad():
            eager = m(x).clone()
        n64 = sum(kid == SLAB_T64 for kid, _ in launched)
        assert n64 == (3 if mode else 0), launched
        g = GraphedForward(m, x)
        outs[mode] = (eager, g(x).clone())
        del g
    assert torch.isfinite(outs[1][0]).all()
    assert torch.equal(outs[1][0], outs[0][0]) and torch.equal(outs[1][1], outs[0][1]) and torch.equal(outs[1][0], outs[1][1])
