"""Generate the BNInception fixtures tests/golden/bninception_b2_224.pt and trn_bninception_MSTRN.pt from the UNMODIFIED reference
(build container only):

    python -m oracle.make_golden_bninception

Same recipe as oracle/make_golden_senet.py: the reference model is built under a fixed seed, its BatchNorms get random statistics
(oracle.functional.randomize_bn_), its own CPU fp32 forward runs; oracle/bninception.py must reproduce every captured stage and the
logits bit for bit; logits, strided stage samples, the state_dict keys / shapes, a digest of the seeded init and the reference's
registry row are stored (so the CPU tests run where the reference is absent).  The reference's blocks are not modules, so a stage
output is captured by a forward-pre-hook on its next consumer: the first 1x1 convolution of the following block (3c and 4e have
no 1x1 head: their 3x3 reduce) and ``global_pool`` for 5b.
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
from oracle import bninception as OB           # noqa: E402
from oracle import reference_loader as RL      # noqa: E402
from oracle.make_golden import GOLDEN_DIR, SEED_BN, SEED_INIT, SEED_INPUT, summarize   # noqa: E402

SEED_TUPLES = 3


def _consumers():
    """stage -> the module whose input is that stage's output."""
    firsts = ['inception_%s_%s' % (b[0], '1x1' if b[2] is not None else '3x3_reduce') for b in OB.BLOCKS]
    return dict(zip(OB.STAGES, firsts + ['global_pool']))


def run_case(name="bninception_b2_224", shape=(2, 3, 224, 224)):
    pt = RL.load()
    torch.manual_seed(SEED_INIT)
    ref = RL.build("bninception", num_classes=1000)
    init_sd = ref.state_dict()
    init_digest = OF.state_digest(init_sd)
    keys = [(k, tuple(v.shape)) for k, v in init_sd.items()]
    OF.randomize_bn_(ref, SEED_BN)
    ref.eval()
    x = OF.seeded_input(shape, SEED_INPUT)
    hooked, handles = {}, []
    for st, mod in _consumers().items():
        handles.append(getattr(ref, mod).register_forward_pre_hook(lambda m, i, st=st: hooked.__setitem__(st, i[0].detach().clone())))
    with torch.no_grad():
        logits = ref(x)
    for h in handles:
        h.remove()
    sd = {k: v.detach().clone() for k, v in ref.state_dict().items()}
    stages = {}
    with torch.no_grad():
        out = OB.forward(x, sd, stages)
    for k, v in hooked.items():
        assert torch.equal(stages[k], v), "oracle restatement differs from the reference at %s/%s" % (name, k)
    assert torch.equal(out, logits)
    settings = {'bninception': sys.modules['pretorched.models.bninception'].pretrained_settings['bninception']}
    torch.save(dict(kind="bninception", arch="bninception", kwargs=dict(num_classes=1000), input_shape=tuple(shape),
                    seeds=dict(init=SEED_INIT, bn=SEED_BN, input=SEED_INPUT), keys=keys, init_digest=init_digest,
                    settings=settings, logits=logits.clone(), stages={k: summarize(v) for k, v in hooked.items()},
                    weight_digest=OF.state_digest(sd), n_state=len(sd), torch_version=torch.__version__),
               os.path.join(GOLDEN_DIR, name + ".pt"))
    print("%-28s logits %s absmax %.4f" % (name, tuple(logits.shape), logits.abs().max()))


def run_trn_case(name="trn_bninception_MSTRN", T=4, B=1, hw=224, kw=dict(frame_bottleneck_dim=128, video_feature_dim=64)):
    """TRN(arch='bninception', consensus='MSTRN') through the reference's own TRN.  The only patch is to the backbone lookup: the
    reference's factory with ``pretrained=None`` and the preprocessing attributes its ``pretrained='imagenet'`` path would attach
    (bninception.py:506-510)."""
    trn = RL.load_trn()
    pt = RL.load()
    arch = "bninception"
    orig = pt.__dict__[arch]

    def offline(num_classes=1000, pretrained=None):
        m = orig(num_classes=num_classes, pretrained=None)
        for k, v in sys.modules['pretorched.models.bninception'].pretrained_settings[arch]['imagenet'].items():
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
        st = {}
        np.random.seed(SEED_TUPLES)
        out = OB.trn_forward(x, sd, T, st)
    assert torch.equal(st['features'], feats) and torch.equal(out, logits), "oracle restatement differs from the reference TRN"
    torch.save(dict(kind="trn_bninception", consensus="MSTRN", arch=arch, segments=T, kwargs=kw, input_shape=(B, T, 3, hw, hw),
                    seeds=dict(init=SEED_INIT, bn=SEED_BN, input=SEED_INPUT, tuples=SEED_TUPLES), features=feats.clone(),
                    logits=logits.clone(), weight_digest=OF.state_digest(sd), n_state=len(sd)), os.path.join(GOLDEN_DIR, name + ".pt"))
    print("%-28s logits %s absmax %.4f" % (name, tuple(logits.shape), logits.abs().max()))


def main(argv=None):
    argv = list(sys.argv[1:] if argv is None else argv)
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    if not argv or "model" in argv:
        run_case()
    if not argv or "trn" in argv:
        run_trn_case()


if __name__ == "__main__":
    main()
