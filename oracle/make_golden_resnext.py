"""Generate the ResNeXt-101 fixtures tests/golden/resnext101_32x4d_b2_224.pt, resnext101_64x4d_b2_224.pt and
trn_resnext101_32x4d_MSTRN.pt from the UNMODIFIED reference (build container only):

    python -m oracle.make_golden_resnext

Same recipe as oracle/make_golden_senet.py, with one step first: the reference's trunk is a module-level ``nn.Sequential`` shared
by every instance and initialised at import, so under the fixed seed it is re-initialised (oracle.resnext.reseed_modules_, every
convolution / BatchNorm initialiser in module order) before the model is built; the package's constructor draws the same numbers
under the same seed.  Then the BatchNorms get random statistics, the reference's CPU fp32 forward runs with hooks on the max-pool
and the four stages, oracle/resnext.py must reproduce every hooked stage and the logits bit for bit, and the logits, strided stage
samples, the state_dict keys / shapes, a digest of the seeded init and the reference's registry rows are stored.
"""
import contextlib
import io
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import functional as OF            # noqa: E402
from oracle import resnext as OX               # noqa: E402
from oracle import reference_loader as RL      # noqa: E402
from oracle.make_golden import GOLDEN_DIR, SEED_BN, SEED_INIT, SEED_INPUT, summarize   # noqa: E402

CASES = {"resnext101_32x4d_b2_224": "resnext101_32x4d", "resnext101_64x4d_b2_224": "resnext101_64x4d"}
SEED_TUPLES = 3


def seeded_reference(pt, arch, num_classes):
    """The reference model built after its shared trunk was re-initialised: call under ``torch.manual_seed``."""
    OX.reseed_modules_(getattr(pt.models.resnext, arch + '_features'))
    return getattr(pt.models.resnext, arch)(num_classes=num_classes, pretrained=None)


def run_case(name, arch, shape=(2, 3, 224, 224)):
    pt = RL.load()
    torch.manual_seed(SEED_INIT)
    ref = seeded_reference(pt, arch, 1000)
    init_sd = ref.state_dict()
    init_digest = OF.state_digest(init_sd)
    keys = [(k, tuple(v.shape)) for k, v in init_sd.items()]
    OF.randomize_bn_(ref, SEED_BN)
    ref.eval()
    x = OF.seeded_input(shape, SEED_INPUT)
    hooked, handles = {}, []
    for st, i in zip(OX.STAGES, range(3, 8)):
        handles.append(ref.features[i].register_forward_hook(lambda m, inp, o, st=st: hooked.__setitem__(st, o.detach().clone())))
    with torch.no_grad():
        logits = ref(x)
    for h in handles:
        h.remove()
    sd = {k: v.detach().clone() for k, v in ref.state_dict().items()}
    stages = {}
    with torch.no_grad():
        out = OX.forward(x, sd, arch, stages)
    for k, v in hooked.items():
        assert torch.equal(stages[k], v), "oracle restatement differs from the reference at %s/%s" % (name, k)
    assert torch.equal(out, logits)
    settings = {n: pt.models.settings.pretrained_settings[n] for n in OX.ARCHS}
    torch.save(dict(kind="resnext101", arch=arch, kwargs=dict(num_classes=1000), input_shape=tuple(shape),
                    seeds=dict(init=SEED_INIT, bn=SEED_BN, input=SEED_INPUT), keys=keys, init_digest=init_digest,
                    settings=settings, logits=logits.clone(), stages={k: summarize(v) for k, v in hooked.items()},
                    weight_digest=OF.state_digest(sd), n_state=len(sd), torch_version=torch.__version__),
               os.path.join(GOLDEN_DIR, name + ".pt"))
    print("%-28s logits %s absmax %.4f, stage absmax %s" % (name, tuple(logits.shape), logits.abs().max(),
                                                             ["%.1f" % v.abs().max() for v in hooked.values()]))


def _policy_names(ref, groups):
    """The optimizer-policy groups as lists of the reference's parameter names."""
    names = {id(p): n for n, p in ref.named_parameters()}
    return [dict(name=g['name'], lr_mult=g['lr_mult'], decay_mult=g['decay_mult'], params=[names[id(p)] for p in g['params']])
            for g in groups]


def run_trn_case(name="trn_resnext101_32x4d_MSTRN", arch="resnext101_32x4d", T=4, B=1, hw=224,
                 kw=dict(frame_bottleneck_dim=128, video_feature_dim=64)):
    """TRN(arch='resnext101_32x4d', consensus='MSTRN') through the reference's own TRN.  The only patch is to the backbone lookup:
    the reference factory with ``pretrained=None`` after the shared-trunk re-initialisation, with the preprocessing attributes
    loading a checkpoint would attach (resnext.py:90-94)."""
    trn = RL.load_trn()
    pt = RL.load()
    orig = pt.__dict__[arch]

    def offline(num_classes=1000, pretrained=None):
        m = seeded_reference(pt, arch, num_classes)
        for k, v in pt.models.resnext.pretrained_settings[arch]['imagenet'].items():
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
    policies = _policy_names(ref, ref.get_optim_policies())
    x = OF.seeded_input((B, T, 3, hw, hw), SEED_INPUT)
    with torch.no_grad():
        np.random.seed(SEED_TUPLES)
        feats = ref.features(x)
        logits = ref.logits(feats)
        sd = {k: v.detach().clone() for k, v in ref.state_dict().items()}
        st = {}
        np.random.seed(SEED_TUPLES)
        out = OX.trn_forward(x, sd, arch, T, st)
    assert torch.equal(st['features'], feats) and torch.equal(out, logits), "oracle restatement differs from the reference TRN"
    torch.save(dict(kind="trn_resnext101", consensus="MSTRN", arch=arch, segments=T, kwargs=kw, input_shape=(B, T, 3, hw, hw),
                    seeds=dict(init=SEED_INIT, bn=SEED_BN, input=SEED_INPUT, tuples=SEED_TUPLES), features=feats.clone(),
                    logits=logits.clone(), policies=policies, weight_digest=OF.state_digest(sd), n_state=len(sd)),
               os.path.join(GOLDEN_DIR, name + ".pt"))
    print("%-28s logits %s absmax %.4f" % (name, tuple(logits.shape), logits.abs().max()))


def main(argv=None):
    argv = list(sys.argv[1:] if argv is None else argv)
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    for name, arch in CASES.items():
        if not argv or name in argv:
            run_case(name, arch)
    if not argv or "trn" in argv:
        run_trn_case()


if __name__ == "__main__":
    main()
