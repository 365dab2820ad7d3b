"""Generate the DenseNet fixtures tests/golden/densenet{121,161}_b2_224.pt, trn_densenet121_MSTRN.pt and
trn_densenet_optim_policies.pt from the UNMODIFIED reference (build container only):

    python -m oracle.make_golden_densenet

Same recipe as oracle/make_golden_inception.py: the reference model is built under a fixed seed, its BatchNorms get random
statistics (oracle.functional.randomize_bn_: with the default init norm1 is the identity and a padding or affine bug in the
pre-activated operand would stay hidden), its own CPU fp32 forward runs; oracle/densenet.py must reproduce its features and logits
bit for bit; logits, a summary of every block's and transition's output and of the features, the state_dict keys / shapes, a
digest of the seeded init and the reference's registry rows are stored (so the CPU tests run where the reference is absent).  The
policy fixture holds the reference TRN's ``get_optim_policies()`` groups on densenet121, partial BN on and off.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import densenet as OD              # noqa: E402
from oracle import functional as OF            # noqa: E402
from oracle import reference_loader as RL      # noqa: E402
from oracle.make_golden import GOLDEN_DIR, SEED_BN, SEED_INIT, SEED_INPUT, summarize   # noqa: E402
from oracle.make_golden_trn_policies import named_policies, reference_trn   # noqa: E402

SEED_TUPLES = 3
ARCHS = ('densenet121', 'densenet161')
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
        logits = ref.logits(feats.clone())     # the reference's logits applies F.relu in place
    sd = {k: v.detach().clone() for k, v in ref.state_dict().items()}
    stages = {}
    with torch.no_grad():
        f2 = OD.features(x, sd, stages)
        out = OD.logits(f2, sd)
    assert torch.equal(f2, feats) and torch.equal(out, logits), "oracle restatement differs from the reference (%s)" % arch
    name = "%s_b2_224" % arch
    torch.save(dict(kind="densenet", arch=arch, kwargs=dict(num_classes=1000), input_shape=tuple(shape),
                    seeds=dict(init=SEED_INIT, bn=SEED_BN, input=SEED_INPUT), keys=keys, init_digest=init_digest,
                    settings={arch: pt.pretrained_settings[arch]}, logits=logits.clone(), features=summarize(feats),
                    stages={k: summarize(v) for k, v in stages.items()},
                    weight_digest=OF.state_digest(sd), n_state=len(sd), torch_version=torch.__version__),
               os.path.join(GOLDEN_DIR, name + ".pt"))
    print("%-28s logits %s absmax %.4f" % (name, tuple(logits.shape), logits.abs().max()))


def run_trn_case(arch='densenet121', T=4, B=1, hw=224):
    ref = reference_trn("MSTRN", arch, T, TRN_KW)
    OF.randomize_bn_(ref, SEED_BN)
    ref.eval()
    x = OF.seeded_input((B, T, 3, hw, hw), SEED_INPUT)
    with torch.no_grad():
        np.random.seed(SEED_TUPLES)
        feats = ref.features(x)
        logits = ref.logits(feats)
    sd = {k: v.detach().clone() for k, v in ref.state_dict().items()}
    name = "trn_%s_MSTRN" % arch
    torch.save(dict(kind="trn_densenet", consensus="MSTRN", arch=arch, segments=T, kwargs=TRN_KW, input_shape=(B, T, 3, hw, hw),
                    seeds=dict(init=SEED_INIT, bn=SEED_BN, input=SEED_INPUT, tuples=SEED_TUPLES), features=feats.clone(),
                    logits=logits.clone(), weight_digest=OF.state_digest(sd), n_state=len(sd)), os.path.join(GOLDEN_DIR, name + ".pt"))
    print("%-28s logits %s absmax %.4f" % (name, tuple(logits.shape), logits.abs().max()))


def run_policies(arch='densenet121', T=4):
    ref = reference_trn("MSTRN", arch, T, TRN_KW)
    pol = {}
    for pbn in (True, False):
        ref.partialBN(pbn)
        pol[pbn] = named_policies(ref)
    torch.save(dict(kind="trn_optim_policies", cases={"densenet121_MSTRN": dict(consensus="MSTRN", arch=arch, segments=T, kwargs=TRN_KW,
                                                                                policies=pol)}),
               os.path.join(GOLDEN_DIR, "trn_densenet_optim_policies.pt"))
    print("trn_densenet_optim_policies  groups (partial BN on) %s" % [len(g['params']) for g in pol[True]])


def main(argv=None):
    argv = list(sys.argv[1:] if argv is None else argv)
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    if not argv or "model" in argv:
        for arch in ARCHS:
            run_case(arch)
    if not argv or "trn" in argv:
        run_trn_case()
        run_policies()


if __name__ == "__main__":
    main()
