"""Generate the Inception-v3 fixtures tests/golden/inceptionv3_b2_299.pt and trn_inceptionv3_MSTRN.pt from the UNMODIFIED
reference (build container only):

    python -m oracle.make_golden_inceptionv3

Same recipe as oracle/make_golden_inception.py: the reference model (torchvision's Inception3 behind the reference's
``inceptionv3``) is built under a fixed seed, its convolution weights are rescaled to their fan-in
(oracle.inceptionv3.fan_in_scale_: torchvision's init would take the activations past fp16's range) and its BatchNorms get random
statistics (oracle.functional.randomize_bn_), its own CPU fp32 forward runs; oracle/inceptionv3.py must reproduce its features and
logits bit for bit; logits, a strided sample of the features and of every stem unit's and block's output, the state_dict keys /
shapes, a digest of the seeded init, the reference's registry row and the keys of a ``pretrained=None`` model built with another
``num_classes`` (which the reference ignores) are stored.  The TRN
fixture holds the reference TRN-MSTRN's features and logits on Inception-v3 and its ``get_optim_policies()`` groups, partial BN on
and off.  Writes only these two files.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import pretorched_x_b200 as P                  # noqa: E402  (module geometry for the restatement)
from oracle import functional as OF            # noqa: E402
from oracle import inceptionv3 as OV3          # noqa: E402
from oracle import reference_loader as RL      # noqa: E402
from oracle.make_golden import GOLDEN_DIR, SEED_BN, SEED_INIT, SEED_INPUT, summarize   # noqa: E402
from oracle.make_golden_trn_policies import named_policies, reference_trn   # noqa: E402

ARCH = 'inceptionv3'
SEED_TUPLES = 3
TRN_KW = dict(frame_bottleneck_dim=128, video_feature_dim=64)


def run_case(shape=(2, 3, 299, 299)):
    pt = RL.load()
    torch.manual_seed(SEED_INIT)
    ref = RL.build(ARCH, num_classes=1000)
    init_sd = ref.state_dict()
    init_digest = OF.state_digest(init_sd)
    keys = [(k, tuple(v.shape)) for k, v in init_sd.items()]
    other = RL.build(ARCH, num_classes=10)         # torchvision_models.py:383: num_classes is not passed on
    other_keys = [(k, tuple(v.shape)) for k, v in other.state_dict().items()]
    OV3.fan_in_scale_(ref)
    OF.randomize_bn_(ref, SEED_BN)
    ref.eval()
    x = OF.seeded_input(shape, SEED_INPUT)
    with torch.no_grad():
        feats = ref.features(x)
        logits = ref.logits(feats)
    sd = {k: v.detach().clone() for k, v in ref.state_dict().items()}
    geom = P.inceptionv3(pretrained=None)
    stages = {}
    with torch.no_grad():
        f2 = OV3.features(x, sd, geom, stages)
        out = OV3.logits(f2, sd)
    assert torch.equal(f2, feats) and torch.equal(out, logits), "oracle restatement differs from the reference"
    name = "%s_b2_299" % ARCH
    torch.save(dict(kind="inceptionv3", arch=ARCH, kwargs=dict(num_classes=1000), input_shape=tuple(shape),
                    seeds=dict(init=SEED_INIT, bn=SEED_BN, input=SEED_INPUT), keys=keys, init_digest=init_digest,
                    keys_num_classes_10=other_keys, settings={ARCH: pt.pretrained_settings[ARCH]}, logits=logits.clone(),
                    features=summarize(feats), stages={k: summarize(v) for k, v in stages.items()},
                    weight_digest=OF.state_digest(sd), n_state=len(sd), torch_version=torch.__version__),
               os.path.join(GOLDEN_DIR, name + ".pt"))
    print("%-28s logits %s absmax %.4f" % (name, tuple(logits.shape), logits.abs().max()))


def run_trn_case(T=4, B=1, hw=299):
    ref = reference_trn("MSTRN", ARCH, T, TRN_KW)
    pol = {}
    for pbn in (True, False):
        ref.partialBN(pbn)
        pol[pbn] = named_policies(ref)
    ref.partialBN(True)
    OV3.fan_in_scale_(ref)
    OF.randomize_bn_(ref, SEED_BN)
    ref.eval()
    x = OF.seeded_input((B, T, 3, hw, hw), SEED_INPUT)
    with torch.no_grad():
        np.random.seed(SEED_TUPLES)
        feats = ref.features(x)
        logits = ref.logits(feats)
    sd = {k: v.detach().clone() for k, v in ref.state_dict().items()}
    name = "trn_%s_MSTRN" % ARCH
    torch.save(dict(kind="trn_inception", consensus="MSTRN", arch=ARCH, segments=T, kwargs=TRN_KW, input_shape=(B, T, 3, hw, hw),
                    seeds=dict(init=SEED_INIT, bn=SEED_BN, input=SEED_INPUT, tuples=SEED_TUPLES), features=feats.clone(),
                    logits=logits.clone(), frame_feature_dim=ref.frame_feature_dim, input_size=list(ref.input_size), policies=pol,
                    weight_digest=OF.state_digest(sd), n_state=len(sd)), os.path.join(GOLDEN_DIR, name + ".pt"))
    print("%-28s logits %s absmax %.4f, groups (partial BN on) %s" % (name, tuple(logits.shape), logits.abs().max(),
                                                                       [len(g['params']) for g in pol[True]]))


def main(argv=None):
    argv = list(sys.argv[1:] if argv is None else argv)
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    if not argv or "model" in argv:
        run_case()
    if not argv or "trn" in argv:
        run_trn_case()


if __name__ == "__main__":
    main()
