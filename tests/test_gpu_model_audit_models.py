"""GPU (-m gpu): every library launch of the engine's other model forwards -- the ones bench.py does not time -- at the batch the
project measures them at, held element by element to the fp64 bound of tests/kernel_ref.py (tests/model_audit.py), and the
audited eager output equal bit for bit to a CUDA-graph replay.

The kernel files test these models' kernels at hand-picked shapes with a few images; the dispatch rules pick kernels and tile
plans from batch and item counts (the slice convolution's runtime-N, 128-column and narrow 32 / 48 tiles, the split GEMM's 64-
and 128-wide instances, the persistent schedules), so at the measured batch other plans run.  Batches:
  * 2-D models at 256 images, as tools/bench_densenet.py, bench_inception.py, bench_bninception.py, bench_senet.py and
    mobilenet_bench.py measure them (299^2 for the Inception-v4 family, 224^2 otherwise);
  * TRN at 16 videos x 8 segments, with the consensus of the golden fixtures (MSTRN; TRN on mobilenetv2);
  * 3-D models as tools/bench_groupconv.py and bench_others.py run them (resnext3d50 8 x 16 x 224^2, SlowFast-R50 8 x 64 x 224^2),
    and preact_resnet3d50 at 8 x 16 x 224^2 and resnet3d18 (type-A shortcuts) at 32 x 16 x 112^2, which no bench tool fixes.
Each model is freshly built (torch.manual_seed(0), BatchNorm statistics randomised by oracle.functional.randomize_bn_ so that BN
scales vary and some are small) and nothing runs before the audit, so every pack is recorded.  A per-launch table and the
distinct (kernel, plan) pairs are printed (pytest -s)."""
import functools
import os
import time

import numpy as np
import pytest
import torch

import pretorched_x_b200 as P
from oracle import functional as OF
from tests.conftest import has_h100
from tests.model_audit import audit
from tests.test_gpu_model_audit import KNOB_ENV, _assert_clean, _report

pytestmark = [
    pytest.mark.gpu,
    pytest.mark.skipif(not has_h100(), reason="needs an H100"),
    pytest.mark.skipif(any(os.environ.get(e) for e in KNOB_ENV),
                       reason="a dispatch override is set in the environment (%s)" % ", ".join(KNOB_ENV)),
]

TRN_KW = dict(frame_bottleneck_dim=128, video_feature_dim=64)


def _trn(arch, consensus):
    return lambda: P.TRN(10, num_segments=8, arch=arch, consensus=consensus, pretrained=None, **TRN_KW)


def _image(arch):
    return lambda: P.__dict__[arch](pretrained=None)


# (case, constructor, input shape)
CASES = [(a, _image(a), (256, 3, 224, 224)) for a in ("mobilenetv2", "se_resnet50", "se_resnext50_32x4d", "bninception", "densenet121",
                                                      "densenet161", "densenet169", "densenet201")] + \
        [(a, _image(a), (256, 3, 299, 299)) for a in ("inceptionv4", "inceptionresnetv2")] + \
        [("trn_%s_%s" % (a, c), _trn(a, c), (16, 8, 3, s, s)) for a, c, s in (
            ("bninception", "MSTRN", 224), ("inceptionv4", "MSTRN", 299), ("inceptionresnetv2", "MSTRN", 299),
            ("densenet121", "MSTRN", 224), ("se_resnext50_32x4d", "MSTRN", 224), ("mobilenetv2", "TRN", 224))] + \
        [("resnext3d50", lambda: P.resnext3d50(num_classes=400), (8, 3, 16, 224, 224)),
         ("slowfast_resnet50_sf", lambda: P.slowfast.resnet50(mode="sf", num_classes=400), (8, 3, 64, 224, 224)),
         ("preact_resnet3d50", lambda: P.preact_resnet3d50(num_classes=400), (8, 3, 16, 224, 224)),
         ("resnet3d18_typeA", lambda: P.resnet3d18(num_classes=400, pretrained=None, shortcut_type="A"), (32, 3, 16, 112, 112))]


def _build(make, shape):
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    torch.manual_seed(0)
    model = make()
    OF.randomize_bn_(model, 1)
    model = model.eval().to(dev)
    # TRN's relation consensus draws its frame tuples per forward; pin one draw so the audited forward and the captured one match
    for mod in model.modules():
        if hasattr(mod, "sample_tuples"):
            np.random.seed(0)
            picks = mod.sample_tuples()
            mod.sample_tuples = functools.partial(lambda p: p, picks)
    x = torch.randn(shape, generator=torch.Generator().manual_seed(1000)).to(dev)
    return model, x


def _bits(t):
    return t.reshape(-1).view(torch.int32 if t.dtype == torch.float32 else torch.int16)


@pytest.mark.timeout(1800, method="thread")
@pytest.mark.parametrize("name,make,shape", CASES, ids=[c[0] for c in CASES])
def test_forward_every_launch_against_fp64(name, make, shape):
    from pretorched_x_b200.graph import GraphedForward
    model, x = _build(make, shape)
    t0 = time.time()
    rep = audit(lambda: model(x))
    seconds = time.time() - t0
    _report("%s_B%d" % (name, shape[0]), rep, seconds)
    _assert_clean(name, rep)
    want = rep.output.clone()
    rep = None
    graphed = GraphedForward(model, x, warmup=1)
    got = graphed()
    torch.cuda.synchronize()
    assert torch.equal(_bits(got), _bits(want)), "the CUDA-graph replay differs from the audited eager forward"


@pytest.mark.timeout(1800, method="thread")
def test_audit_catches_a_slice_convolution_writing_past_its_slice():
    """densenet121 at 256 images, its 10th slice convolution (a layer in the middle of the second dense block) also writing one
    element into the column right after its slice: the next layer overwrites that column before anything reads it, so the
    logits equal an unfaulted run bit for bit, and the audit fails that launch and only that launch."""
    from pretorched_x_b200 import ops
    model, x = _build(_image("densenet121"), (256, 3, 224, 224))
    real, calls = ops.conv_slice, []

    @functools.wraps(real)
    def faulty(a, pc, y, *args, **kwargs):
        out = real(a, pc, y, *args, **kwargs)
        calls.append(1)
        if len(calls) == 10:
            past = y.as_strided((1,), (1,), y.storage_offset() + (y.shape[0] - 1) * y.stride(0) + y.shape[1])
            past.view(torch.int16).bitwise_not_()
        return out
    ops.conv_slice = faulty
    try:
        rep = audit(lambda: model(x))
    finally:
        ops.conv_slice = real
    bad = rep.failures()
    print("[model-audit] injected fault: %s" % ["#%d %s %s: %s" % (r["index"], r["entry"], r["geometry"], r["where"]) for r in bad])
    slice_rows = [r for r in rep.rows if r["entry"] == "conv_slice"]
    assert [r["index"] for r in bad] == [slice_rows[9]["index"]]
    assert "outside the slice" in bad[0]["where"]
    faulted = rep.output.clone()
    rep = None
    with torch.no_grad():
        clean = model(x)
    torch.cuda.synchronize()
    assert torch.equal(_bits(faulted), _bits(clean)), "the fault reached the logits"
