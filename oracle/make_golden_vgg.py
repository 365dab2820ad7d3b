"""Generate the VGG / AlexNet fixtures tests/golden/{vgg16,vgg16_bn,vgg11,alexnet}_b2_224.pt and trn_{vgg16,alexnet}_MSTRN.pt (with the
reference TRN's ``get_optim_policies()`` groups, partial BN on and off) from the
UNMODIFIED reference (build container only):

    python -m oracle.make_golden_vgg

Same recipe as oracle/make_golden_densenet.py: the reference model is built under a fixed seed, its BatchNorms get random statistics
(oracle.functional.randomize_bn_), its own CPU fp32 forward runs, and oracle/vgg.py must reproduce its features and logits bit for
bit.  Stored: the input seed, logits, features, a summary of every pool's output (its largest activation included), the state_dict
keys / shapes in order, a digest of the seeded init and the reference's registry rows.  Measured at the seeded init, the largest
activation of every stage stays within fp16's range and away from its subnormals (printed below), so no rescaling is applied.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import functional as OF            # noqa: E402
from oracle import reference_loader as RL      # noqa: E402
from oracle import vgg as OV                   # noqa: E402
from oracle.make_golden import GOLDEN_DIR, SEED_BN, SEED_INIT, SEED_INPUT, summarize   # noqa: E402
from oracle.make_golden_trn_policies import named_policies, reference_trn   # noqa: E402

SEED_TUPLES = 3
ARCHS = ('vgg16', 'vgg16_bn', 'vgg11', 'alexnet')
TRN_KW = dict(frame_bottleneck_dim=128, video_feature_dim=64)


def run_case(arch, shape=(2, 3, 224, 224)):
    pt = RL.load()
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
        logits = ref.logits(feats.clone())
    sd = {k: v.detach().clone() for k, v in ref.state_dict().items()}
    stages = {}
    with torch.no_grad():
        f2 = OV.features(x, sd, arch, stages)
        out = OV.logits(f2, sd)
    assert torch.equal(f2, feats) and torch.equal(out, logits), "oracle restatement differs from the reference (%s)" % arch
    name = "%s_b2_224" % arch
    torch.save(dict(kind="vgg", arch=arch, kwargs=dict(num_classes=1000), input_shape=tuple(shape),
                    seeds=dict(init=SEED_INIT, bn=SEED_BN, input=SEED_INPUT), keys=keys, init_digest=init_digest,
                    settings={arch: pt.pretrained_settings[arch]}, logits=logits.clone(), features=feats.clone(),
                    stages={k: summarize(v) for k, v in stages.items()},
                    weight_digest=OF.state_digest(sd), n_state=len(sd), torch_version=torch.__version__),
               os.path.join(GOLDEN_DIR, name + ".pt"))
    print("%-28s logits %s absmax %.4f | stage absmax %s" % (name, tuple(logits.shape), logits.abs().max(),
                                                            ["%.3g" % v.abs().max() for v in stages.values()]))


def run_trn_case(arch, T=4, B=1, hw=224):
    ref = reference_trn("MSTRN", arch, T, TRN_KW)
    OF.randomize_bn_(ref, SEED_BN)
    ref.eval()
    x = OF.seeded_input((B, T, 3, hw, hw), SEED_INPUT)
    with torch.no_grad():
        np.random.seed(SEED_TUPLES)
        feats = ref.features(x)
        logits = ref.logits(feats)
    sd = {k: v.detach().clone() for k, v in ref.state_dict().items()}
    pol = {}
    for pbn in (True, False):
        ref.partialBN(pbn)
        pol[pbn] = named_policies(ref)
    name = "trn_%s_MSTRN" % arch
    torch.save(dict(kind="trn_vgg", consensus="MSTRN", arch=arch, segments=T, kwargs=TRN_KW, input_shape=(B, T, 3, hw, hw),
                    seeds=dict(init=SEED_INIT, bn=SEED_BN, input=SEED_INPUT, tuples=SEED_TUPLES), features=feats.clone(),
                    logits=logits.clone(), weight_digest=OF.state_digest(sd), n_state=len(sd), policies=pol),
               os.path.join(GOLDEN_DIR, name + ".pt"))
    print("%-28s logits %s absmax %.4f" % (name, tuple(logits.shape), logits.abs().max()))


def main(argv=None):
    """Each case runs in a process of its own: the reference's ``modify_vggs`` / ``modify_alexnet`` patch ``features`` onto
    torchvision's class, so a second model of that class built in the same process finds the method where its ``features``
    Sequential was and recurses."""
    argv = list(sys.argv[1:] if argv is None else argv)
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    if len(argv) == 2 and argv[0] in ("model", "trn"):
        (run_case if argv[0] == "model" else run_trn_case)(argv[1])
        return
    import subprocess
    cases = ([("model", a) for a in ARCHS] if not argv or "model" in argv else []) + \
        ([("trn", a) for a in ('vgg16', 'alexnet')] if not argv or "trn" in argv else [])
    for kind, arch in cases:
        subprocess.run([sys.executable, "-m", "oracle.make_golden_vgg", kind, arch], cwd=ROOT, check=True)


if __name__ == "__main__":
    main()
