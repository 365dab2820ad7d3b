"""CPU: BNInception against the reference, as recorded in the fixtures (tests/golden/bninception_b2_224.pt and
trn_bninception_MSTRN.pt, written by oracle/make_golden_bninception.py from the unmodified reference): state_dict keys, shapes and
order, a seeded init bit-identical to the reference's, the registry row, the oracle restatement against the reference's own
stages and logits; TRN on a BNInception backbone; and the split GEMM's host planning and refusals."""
import ctypes
import os

import pytest
import torch

import pretorched_x_b200 as P
from pretorched_x_b200 import _lib, ops
from pretorched_x_b200.models import bninception as PB
from oracle import bninception as OB
from oracle import functional as OF
from oracle.make_golden import sample_of

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
B2_ERR_INVALID = -1


def _load(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


def test_state_dict_layout_and_seeded_init_match_reference():
    fx = _load("bninception_b2_224.pt")
    torch.manual_seed(fx["seeds"]["init"])
    model = P.bninception(pretrained=None, **fx["kwargs"])
    sd = model.state_dict()
    assert len(sd) == 485 and sum(p.numel() for p in model.parameters()) == 11295240
    assert [(k, tuple(v.shape)) for k, v in sd.items()] == [tuple(kv) for kv in fx["keys"]]
    assert OF.digests_match(OF.state_digest(sd), fx["init_digest"])
    assert fx["n_state"] == len(sd)


def test_pretrained_settings_row_matches_reference():
    fx = _load("bninception_b2_224.pt")
    assert P.pretrained_settings["bninception"] == fx["settings"]["bninception"]
    assert "bninception" in P.model_names


def test_block_table_matches_between_package_and_oracle():
    assert PB.BLOCKS == OB.BLOCKS
    assert [PB.block_out_channels(b) for b in PB.BLOCKS] == [256, 320, 576, 576, 576, 608, 608, 1056, 1024, 1024]


def test_oracle_reproduces_reference_stages_and_logits():
    fx = _load("bninception_b2_224.pt")
    model = OB.build_package_model(P, fx)
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    assert OF.digests_match(OF.state_digest(sd), fx["weight_digest"])
    x = OF.seeded_input(fx["input_shape"], fx["seeds"]["input"])
    stages = {}
    with torch.no_grad():
        logits = OB.forward(x, sd, stages)
    assert set(fx["stages"]) == set(OB.STAGES)
    for name, summ in fx["stages"].items():
        assert tuple(stages[name].shape) == tuple(summ["shape"]), name
        s, step = sample_of(stages[name])
        assert step == summ["step"] and torch.equal(s, summ["sample"]), name
    assert torch.equal(logits, fx["logits"])


def test_trn_on_bninception_builds_and_refuses_fine_tune():
    m = P.TRN(10, num_segments=4, arch="bninception", consensus="MSTRN", pretrained=None, frame_bottleneck_dim=128,
              video_feature_dim=64)
    assert m.frame_feature_dim == 1024
    assert (m.input_space, m.mean, m.std, list(m.input_size)) == ("BGR", [104, 117, 128], [1, 1, 1], [224, 224])
    groups = m.get_optim_policies()
    assert sum(len(g["params"]) for g in groups) > 0
    with pytest.raises(NotImplementedError, match="has none"):
        m.fine_tune(4)


@pytest.mark.parametrize("cols,npad,box0", [
    ([64, 64, 64], 192, [0, 1, 2, 3]),          # 3a / 3b: no padding
    ([128, 64], 192, [0, 2, 3]),                # 3c
    ([224, 64, 96], 448, [0, 4, 5, 7]),         # 4a: 384 -> 448
    ([192, 96, 96], 448, [0, 3, 5, 7]),         # 4b
    ([160, 128, 128], 448, [0, 3, 5, 7]),       # 4c: 416 -> 448
    ([96, 128, 160], 448, [0, 2, 4, 7]),        # 4d
    ([128, 192], 320, [0, 2, 5]),               # 4e
    ([352, 192, 160], 768, [0, 6, 9, 12]),      # 5a: 704 -> 768
    ([352, 192, 192], 768, [0, 6, 9, 12]),      # 5b: 736 -> 768
    ([32], 64, [0, 1]),                         # 3a pool projection
    ([8, 8, 8, 8], 256, [0, 1, 2, 3, 4]),
])
def test_split_plan(cols, npad, box0):
    assert ops.split_plan(cols) == (npad, box0)


@pytest.mark.parametrize("cols", [[], [64] * 5, [0], [60], [64, -8]])
def test_split_plan_refusals(cols):
    with pytest.raises(ValueError):
        ops.split_plan(cols)


def _split_call(nd=2, cols=(64, 64), ldy=(64, 64), y_off=(0, 0), N=None, **over):
    """b2_gemm_split_f16 with fake device addresses: every refusal below is decided before any launch."""
    g = _lib.GemmArgs()
    g.a, g.b, g.scale, g.shift = ctypes.c_void_p(0x10000), ctypes.c_void_p(0x20000), ctypes.c_void_p(0x30000), ctypes.c_void_p(0x40000)
    g.M, g.Kd, g.lda, g.ldb, g.relu = 100, 64, 64, 64, 1
    g.N = N if N is not None else ops.split_plan(list(cols)[:nd])[0]
    for k, v in over.items():
        setattr(g, k, v)
    ys = (ctypes.c_void_p * 4)(*[0x100000 + 0x10000 * d + o for d, o in zip(range(4), list(y_off) + [0] * 4)])
    lds = (ctypes.c_int * 4)(*(list(ldy) + [0] * 4)[:4])
    cs = (ctypes.c_int * 4)(*(list(cols) + [0] * 4)[:4])
    rc = _lib.load().b2_gemm_split_f16(ctypes.byref(g), nd, ys, lds, cs, ctypes.c_void_p(0))
    return rc, _lib.last_error()


@pytest.mark.parametrize("case,kw,msg", [
    ("unaligned slice", dict(y_off=(8, 0)), "16-byte"),
    ("pitch below width", dict(ldy=(32, 64)), "pitch"),
    ("pitch not a multiple of 8", dict(ldy=(68, 64)), "pitch"),
    ("width not a multiple of 8", dict(cols=(60, 64), N=128), "multiple of 8"),
    ("N not the packed width", dict(N=128 + 64), "packed width"),
    ("too many destinations", dict(nd=5, cols=(64,) * 5, ldy=(64,) * 5, N=320), "1 to 4"),
    ("residual", dict(residual=ctypes.c_void_p(0x50000), ldr=64), "residual"),
    ("fp32 output", dict(out_f32=1), "fp16"),
    ("plain output pointer", dict(d=ctypes.c_void_p(0x50000), ldd=64), "destinations"),
])
def test_split_gemm_refusals(case, kw, msg):
    rc, err = _split_call(**kw)
    assert rc == B2_ERR_INVALID and msg in err, (case, rc, err)


def _conv_args(**over):
    a = _lib.ConvArgs()
    a.x, a.w, a.scale, a.shift, a.y = (ctypes.c_void_p(v) for v in (0x10000, 0x20000, 0x30000, 0x40000, 0x50000))
    a.N, a.T, a.H, a.W, a.C, a.K, a.ldy = 2, 1, 28, 28, 64, 96, 256
    a.kt, a.kh, a.kw, a.st, a.sh, a.sw, a.pt, a.ph, a.pw = 1, 3, 3, 1, 1, 1, 0, 1, 1
    a.relu, a.mode = 1, _lib.B2_CONV_AUTO
    for k, v in over.items():
        setattr(a, k, v)
    return a


@pytest.mark.parametrize("case,kw", [
    ("stem mode", dict(mode=_lib.B2_CONV_STEM7, C=4, kw=7, kh=7, sw=2, sh=2, pw=3, ph=3)),
    ("mask", dict(mask=ctypes.c_void_p(0x60000), ldm=256, relu=0)),
    ("per-sample affine", dict(aff_ld=96)),
    ("upsample", dict(upsample=1)),
    ("second output", dict(y2=ctypes.c_void_p(0x60000), scale2=ctypes.c_void_p(0x70000), shift2=ctypes.c_void_p(0x80000), aff2_ld=96)),
    ("pool_w", dict(pool_w=1)),
    ("1x1 filter", dict(kh=1, kw=1, ph=0, pw=0)),
    ("unaligned slice", dict(y=ctypes.c_void_p(0x50008))),
])
def test_slice_conv_refusals(case, kw):
    rc = _lib.load().b2_conv_ndhwc_fprop_slice(ctypes.byref(_conv_args(**kw)), ctypes.c_void_p(0))
    assert rc == B2_ERR_INVALID, (case, rc, _lib.last_error())


@pytest.mark.parametrize("case,args", [
    ("pitch below channels", dict(ldx=32)),
    ("unaligned output", dict(y=0x50008)),
    ("window outside the input", dict(Ho=30)),
    ("padding over half the window", dict(ph=2, pw=2)),
    ("bad mode", dict(avg=2)),
])
def test_slice_pool_refusals(case, args):
    a = dict(x=0x10000, ldx=64, y=0x50000, ldy=128, N=2, T=1, H=28, W=28, C=64, kt=1, kh=3, kw=3, st=1, sh=1, sw=1, pt=0, ph=1, pw=1,
             To=1, Ho=28, Wo=28, avg=1)
    a.update(args)
    vals = list(a.values())
    rc = _lib.load().b2_pool_ndhwc_slice(ctypes.c_void_p(vals[0]), vals[1], ctypes.c_void_p(vals[2]), *vals[3:], ctypes.c_void_p(0))
    assert rc == B2_ERR_INVALID, (case, rc, _lib.last_error())
