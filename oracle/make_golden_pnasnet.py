"""Generate the PNASNet-5-Large fixtures tests/golden/pnasnet5large_b2_331.pt and trn_pnasnet5large_MSTRN.pt (with the reference
TRN's ``get_optim_policies()`` groups, partial BN on and off) from the UNMODIFIED reference (build container only):

    python -m oracle.make_golden_pnasnet

Same recipe as oracle/make_golden_vgg.py: the reference model is built under a fixed seed (PyTorch's default initialisers, in the
reference's construction order), its BatchNorms get random statistics (oracle.functional.randomize_bn_), its own CPU fp32 forward
runs with hooks on conv_0 and every cell, and oracle/pnasnet.py must reproduce every hooked stage, the features and the logits bit
for bit.  Stored: the input seed, logits, a summary of the features and of every stage, the
state_dict keys / shapes in order, a digest of the seeded init and the reference's registry row.
Rescaling rule: the init digest is recorded at the seeded default init; then every Conv2d weight is multiplied by 1.7
(oracle.pnasnet.rescale_), because at the default init the activations shrink cell by cell (conv_0 std 0.58, cell_11 about 1e-4,
at the edge of fp16's normal range), and at He's std they grow about 4x per cell.  The generator asserts that every stage's std stays within 10x of conv_0's and
prints them.  oracle.pnasnet.build_package_model applies the same rule to the package's model.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import functional as OF            # noqa: E402
from oracle import reference_loader as RL      # noqa: E402
from oracle import pnasnet as OPn              # noqa: E402
from oracle.make_golden import GOLDEN_DIR, SEED_BN, SEED_INIT, SEED_INPUT, summarize   # noqa: E402
from oracle.make_golden_trn_policies import named_policies, reference_trn   # noqa: E402

ARCH = 'pnasnet5large'
SEED_TUPLES = 3
TRN_KW = dict(frame_bottleneck_dim=128, video_feature_dim=64)


def run_case(hw, B=2):
    pt = RL.load()
    torch.manual_seed(SEED_INIT)
    ref = RL.build(ARCH, num_classes=1000)
    init_sd = ref.state_dict()
    init_digest = OF.state_digest(init_sd)
    keys = [(k, tuple(v.shape)) for k, v in init_sd.items()]
    OPn.rescale_(ref)
    OF.randomize_bn_(ref, SEED_BN)
    ref.eval()
    x = OF.seeded_input((B, 3, hw, hw), SEED_INPUT)
    hooked = {}
    handles = [getattr(ref, b).register_forward_hook(lambda m, inp, o, b=b: hooked.__setitem__(b, o.detach().clone()))
               for b in OPn.STAGES]
    with torch.no_grad():
        feats = ref.features(x)
        logits = ref.logits(feats.clone())
    for h in handles:
        h.remove()
    sd = {k: v.detach().clone() for k, v in ref.state_dict().items()}
    stages = {}
    with torch.no_grad():
        f2 = OPn.features(x, sd, stages)
        out = OPn.logits(f2, sd)
    assert list(stages) == list(hooked) == OPn.STAGES
    for k, v in hooked.items():
        assert torch.equal(stages[k], v), "oracle restatement differs from the reference at %s" % k
    assert torch.equal(f2, feats) and torch.equal(out, logits), "oracle restatement differs from the reference"
    s0 = hooked['conv_0'].std()
    stds = [float(v.std()) for v in hooked.values()]
    assert all(s0 / 10 <= v <= s0 * 10 for v in stds), "stage stds %s are not within 10x of conv_0's" % stds
    print("stage std", ["%.3g" % v for v in stds])
    name = "%s_b%d_%d" % (ARCH, B, hw)
    torch.save(dict(kind="pnasnet", arch=ARCH, kwargs=dict(num_classes=1000), input_shape=(B, 3, hw, hw),
                    seeds=dict(init=SEED_INIT, bn=SEED_BN, input=SEED_INPUT), keys=keys, init_digest=init_digest,
                    settings={ARCH: pt.pretrained_settings[ARCH]}, logits=logits.clone(), features=summarize(feats),
                    stages={k: summarize(v) for k, v in hooked.items()}, weight_digest=OF.state_digest(sd), n_state=len(sd),
                    torch_version=torch.__version__),
               os.path.join(GOLDEN_DIR, name + ".pt"))
    print("%-28s logits %s absmax %.4f | features absmax %.3g | stage absmax %s" % (
        name, tuple(logits.shape), logits.abs().max(), feats.abs().max(), ["%.3g" % v.abs().max() for v in hooked.values()]))


def run_trn_case(T=4, B=1, hw=331):
    ref = reference_trn("MSTRN", ARCH, T, TRN_KW)
    pol = {}
    for pbn in (True, False):
        ref.partialBN(pbn)
        pol[pbn] = named_policies(ref)
    ref.partialBN(True)
    OPn.rescale_(ref)
    OF.randomize_bn_(ref, SEED_BN)
    ref.eval()
    x = OF.seeded_input((B, T, 3, hw, hw), SEED_INPUT)
    with torch.no_grad():
        np.random.seed(SEED_TUPLES)
        feats = ref.features(x)
        logits = ref.logits(feats)
    sd = {k: v.detach().clone() for k, v in ref.state_dict().items()}
    name = "trn_%s_MSTRN" % ARCH
    torch.save(dict(kind="trn_pnasnet", consensus="MSTRN", arch=ARCH, segments=T, kwargs=TRN_KW, input_shape=(B, T, 3, hw, hw),
                    seeds=dict(init=SEED_INIT, bn=SEED_BN, input=SEED_INPUT, tuples=SEED_TUPLES), features=feats.clone(),
                    logits=logits.clone(), frame_feature_dim=ref.frame_feature_dim, input_size=list(ref.input_size), policies=pol,
                    weight_digest=OF.state_digest(sd), n_state=len(sd)), os.path.join(GOLDEN_DIR, name + ".pt"))
    print("%-28s logits %s absmax %.4f, groups (partial BN on) %s" % (name, tuple(logits.shape), logits.abs().max(),
                                                                       [len(g['params']) for g in pol[True]]))


def main(argv=None):
    argv = list(sys.argv[1:] if argv is None else argv)
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    if not argv or "model" in argv:
        run_case(331)
    if not argv or "trn" in argv:
        run_trn_case()


if __name__ == "__main__":
    main()
