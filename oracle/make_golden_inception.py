"""Generate the Inception-v4 / Inception-ResNet-v2 fixtures tests/golden/{inceptionv4,inceptionresnetv2}_b2_299.pt and
trn_{inceptionv4,inceptionresnetv2}_MSTRN.pt from the UNMODIFIED reference (build container only):

    python -m oracle.make_golden_inception

Same recipe as oracle/make_golden_bninception.py: the reference model is built under a fixed seed, its BatchNorms get random
statistics (oracle.functional.randomize_bn_), its own CPU fp32 forward runs; oracle/inception.py must reproduce its features and
logits bit for bit; logits, a strided sample of the features, the state_dict keys / shapes, a digest of the seeded init and the
reference's registry rows are stored (so the CPU tests run where the reference is absent).
"""
import contextlib
import io
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import pretorched_x_b200 as P                  # noqa: E402  (module geometry for the restatement)
from oracle import functional as OF            # noqa: E402
from oracle import inception as OI             # noqa: E402
from oracle import reference_loader as RL      # noqa: E402
from oracle.make_golden import GOLDEN_DIR, SEED_BN, SEED_INIT, SEED_INPUT, summarize   # noqa: E402

SEED_TUPLES = 3
ARCHS = ('inceptionv4', 'inceptionresnetv2')


def _ref_settings(arch):
    return sys.modules['pretorched.models.%s' % arch].pretrained_settings[arch]


def run_case(arch, shape=(2, 3, 299, 299)):
    RL.load()
    torch.manual_seed(SEED_INIT)
    ref = RL.build(arch, num_classes=1000)
    init_sd = ref.state_dict()
    init_digest = OF.state_digest(init_sd)
    keys = [(k, tuple(v.shape)) for k, v in init_sd.items()]
    OF.randomize_bn_(ref, SEED_BN)
    ref.eval()
    x = OF.seeded_input(shape, SEED_INPUT)
    with torch.no_grad():
        feats = ref.features(x)
        logits = ref.logits(feats)
    sd = {k: v.detach().clone() for k, v in ref.state_dict().items()}
    geom = P.__dict__[arch](pretrained=None)
    with torch.no_grad():
        f2 = OI.features(x, sd, geom)
        out = OI.logits(f2, sd)
    assert torch.equal(f2, feats) and torch.equal(out, logits), "oracle restatement differs from the reference (%s)" % arch
    name = "%s_b2_299" % arch
    torch.save(dict(kind="inception", arch=arch, kwargs=dict(num_classes=1000), input_shape=tuple(shape),
                    seeds=dict(init=SEED_INIT, bn=SEED_BN, input=SEED_INPUT), keys=keys, init_digest=init_digest,
                    settings={arch: _ref_settings(arch)}, logits=logits.clone(), features=summarize(feats),
                    weight_digest=OF.state_digest(sd), n_state=len(sd), torch_version=torch.__version__),
               os.path.join(GOLDEN_DIR, name + ".pt"))
    print("%-28s logits %s absmax %.4f" % (name, tuple(logits.shape), logits.abs().max()))


def run_trn_case(arch, T=4, B=1, hw=299, kw=dict(frame_bottleneck_dim=128, video_feature_dim=64)):
    """TRN(arch, consensus='MSTRN') through the reference's own TRN.  The only patch is to the backbone lookup: the reference's
    factory with ``pretrained=None`` and the preprocessing attributes its ``pretrained='imagenet'`` path would attach."""
    trn = RL.load_trn()
    pt = RL.load()
    orig = pt.__dict__[arch]

    def offline(num_classes=1000, pretrained=None):
        m = orig(num_classes=num_classes, pretrained=None)
        for k, v in _ref_settings(arch)['imagenet'].items():
            if k in ('input_space', 'input_size', 'input_range', 'mean', 'std'):
                setattr(m, k, v)
        return m
    pt.__dict__[arch] = offline
    try:
        torch.manual_seed(SEED_INIT)
        with contextlib.redirect_stdout(io.StringIO()):
            ref = trn.TRN(10, num_segments=T, arch=arch, consensus="MSTRN", pretrained=None, **kw)
    finally:
        pt.__dict__[arch] = orig
    OF.randomize_bn_(ref, SEED_BN)
    ref.eval()
    x = OF.seeded_input((B, T, 3, hw, hw), SEED_INPUT)
    with torch.no_grad():
        np.random.seed(SEED_TUPLES)
        feats = ref.features(x)
        logits = ref.logits(feats)
    sd = {k: v.detach().clone() for k, v in ref.state_dict().items()}
    name = "trn_%s_MSTRN" % arch
    torch.save(dict(kind="trn_inception", consensus="MSTRN", arch=arch, segments=T, kwargs=kw, input_shape=(B, T, 3, hw, hw),
                    seeds=dict(init=SEED_INIT, bn=SEED_BN, input=SEED_INPUT, tuples=SEED_TUPLES), features=feats.clone(),
                    logits=logits.clone(), weight_digest=OF.state_digest(sd), n_state=len(sd)), os.path.join(GOLDEN_DIR, name + ".pt"))
    print("%-28s logits %s absmax %.4f" % (name, tuple(logits.shape), logits.abs().max()))


def main(argv=None):
    argv = list(sys.argv[1:] if argv is None else argv)
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    for arch in ARCHS:
        if not argv or "model" in argv:
            run_case(arch)
        if not argv or "trn" in argv:
            run_trn_case(arch)


if __name__ == "__main__":
    main()
