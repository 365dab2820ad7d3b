"""Generate the MobileNetV2 fixtures tests/golden/mobilenetv2_*.pt and trn_mobilenetv2_TRN.pt from the UNMODIFIED reference
(build container only):

    python -m oracle.make_golden_mobilenet

Same recipe as oracle/make_golden.py: the reference model is built under a fixed seed, its BatchNorms get random statistics
(oracle.functional.randomize_bn_) and are then scaled so that every activation has std 3 (oracle.mobilenet.calibrate_bn_: at
the raw init no ReLU6 reaches 6, so the clamps would go untested); the reference's own CPU fp32 forward runs with hooks on
the block outputs; oracle/mobilenet.py must reproduce every hooked stage bit for bit; logits, strided stage samples and a
weight digest are stored.  The fixtures have kinds of their own ("mobilenetv2", "trn_mobilenetv2"): the ResNet stage walk of
the "model" / "trn" fixture tests does not apply to them.
"""
import contextlib
import io
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import functional as OF            # noqa: E402
from oracle import mobilenet as OM             # noqa: E402
from oracle import reference_loader as RL      # noqa: E402
from oracle.make_golden import GOLDEN_DIR, SEED_BN, SEED_INIT, SEED_INPUT, summarize   # noqa: E402

# block outputs that are stored (the projections of the last block of every stage, and the final 1x1 conv + ReLU6); the
# stem's output is not: the engine stores it without the upper clamp, which its only reader, the depthwise, applies
STAGES = ["features.1", "features.3", "features.6", "features.10", "features.13", "features.16", "features.17", "features.18"]

CASES = {
    # name -> (num_classes, input shape)
    "mobilenetv2_b2_224": (1000, (2, 3, 224, 224)),
    # non-square and not a multiple of 32: stride-2 depthwise layers see odd sizes and 1- / 2-pixel maps
    "mobilenetv2_b2_96x64": (10, (2, 3, 96, 64)),
}


def clamp_shares(taps):
    """{block: (share of expansion outputs at 6, share of depthwise outputs at 6)}."""
    return {i: (float((t['expand'] == 6).double().mean()) if 'expand' in t else None, float((t['dw'] == 6).double().mean()))
            for i, t in taps.items()}


def check_clamps(name, taps):
    shares = clamp_shares(taps)
    both = [i for i, (e, d) in shares.items() if e and d]
    assert len(both) >= 6, "%s: the ReLU6 clamps bind in too few blocks: %s" % (name, shares)
    return shares


def run_case(name, num_classes, shape):
    RL.load()
    torch.manual_seed(SEED_INIT)
    ref = RL.build("mobilenetv2", num_classes=num_classes)
    init_digest = OF.state_digest(ref.state_dict())
    OF.randomize_bn_(ref, SEED_BN)
    ref.eval()
    x = OF.seeded_input(shape, SEED_INPUT)
    factors = OM.calibrate_bn_(ref, x)
    hooked, handles = {}, []
    for st in STAGES:
        handles.append(ref.features[int(st.split('.')[1])].register_forward_hook(
            lambda m, i, o, st=st: hooked.__setitem__(st, o.detach().clone())))
    with torch.no_grad():
        logits = ref(x)
    for h in handles:
        h.remove()
    sd = {k: v.detach().clone() for k, v in ref.state_dict().items()}
    stages, taps = {}, {}
    with torch.no_grad():
        out = OM.forward(x, sd, stages, taps)
    for k, v in hooked.items():
        assert torch.equal(stages[k], v), "oracle restatement differs from the reference at %s/%s" % (name, k)
    assert torch.equal(out, logits)
    shares = check_clamps(name, taps)
    hooked["logits"] = logits
    torch.save(dict(kind="mobilenetv2", arch="mobilenetv2", kwargs=dict(num_classes=num_classes), input_shape=tuple(shape),
                    seeds=dict(init=SEED_INIT, bn=SEED_BN, input=SEED_INPUT), bn_factors=factors, keys=list(sd),
                    init_digest=init_digest, logits=logits.clone(), stages={k: summarize(v) for k, v in hooked.items()},
                    clamp_shares=shares, weight_digest=OF.state_digest(sd), n_state=len(sd), torch_version=torch.__version__),
               os.path.join(GOLDEN_DIR, name + ".pt"))
    print("%-28s logits %s absmax %.4f  clamp shares (expand, dw): %s" % (
        name, tuple(logits.shape), logits.abs().max(), {i: tuple(round(v, 4) if v else v for v in s) for i, s in shares.items()}))


def run_trn_case(name="trn_mobilenetv2_TRN", T=8, B=2, hw=64, kw=dict(frame_bottleneck_dim=128, video_feature_dim=64)):
    """TRN(arch='mobilenetv2', consensus='TRN') through the reference's own TRN.  As in make_golden.run_trn_cases, the only
    patch is to the backbone factory: build it with ``pretrained=None`` and attach the preprocessing attributes
    ``load_pretrained`` would.  The reference's registry (pretorched/models/settings.py) has no mobilenetv2 row, so they come
    from mobilenet.py's own ``pretrained_settings``."""
    trn = RL.load_trn()
    pt = RL.load()
    orig = pt.__dict__["mobilenetv2"]

    def offline(num_classes=1000, pretrained=None):
        m = orig(num_classes=num_classes, pretrained=None)
        for k, v in pt.models.mobilenet.pretrained_settings['mobilenetv2']['imagenet'].items():
            if k in ('input_space', 'input_size', 'input_range', 'mean', 'std'):
                setattr(m, k, v)
        return m
    pt.__dict__["mobilenetv2"] = offline
    try:
        torch.manual_seed(SEED_INIT)
        with contextlib.redirect_stdout(io.StringIO()):
            ref = trn.TRN(10, num_segments=T, arch="mobilenetv2", consensus="TRN", pretrained=None, **kw)
    finally:
        pt.__dict__["mobilenetv2"] = orig
    OF.randomize_bn_(ref, SEED_BN)
    ref.eval()
    x = OF.seeded_input((B, T, 3, hw, hw), SEED_INPUT)
    factors = OM.calibrate_bn_(ref.base_model, x.view((-1, 3, hw, hw)))
    with torch.no_grad():
        feats = ref.features(x)
        logits = ref.logits(feats)
        sd = {k: v.detach().clone() for k, v in ref.state_dict().items()}
        st = {}
        out = OM.trn_forward(x, sd, T, st)
    assert torch.equal(st['features'], feats) and torch.equal(out, logits), "oracle restatement differs from the reference TRN"
    torch.save(dict(kind="trn_mobilenetv2", consensus="TRN", arch="mobilenetv2", segments=T, kwargs=kw, input_shape=(B, T, 3, hw, hw),
                    seeds=dict(init=SEED_INIT, bn=SEED_BN, input=SEED_INPUT), bn_factors=factors, features=feats.clone(),
                    logits=logits.clone(), weight_digest=OF.state_digest(sd), n_state=len(sd)), os.path.join(GOLDEN_DIR, name + ".pt"))
    print("%-28s logits %s absmax %.4f" % (name, tuple(logits.shape), logits.abs().max()))


def main(argv=None):
    argv = list(sys.argv[1:] if argv is None else argv)
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    for name, (nc, shape) in CASES.items():
        if not argv or name in argv:
            run_case(name, nc, shape)
    if not argv or "trn" in argv:
        run_trn_case()


if __name__ == "__main__":
    main()
