"""Generate the PolyNet fixtures tests/golden/polynet_b2_331.pt and trn_polynet_MSTRN.pt from the UNMODIFIED reference (build
container only):

    python -m oracle.make_golden_polynet

Same recipe as oracle/make_golden_inceptionv3.py: the reference model is built under a fixed seed and the digest of that init
is recorded; then its weights are rescaled (oracle.polynet.rescale_: at the default init the residual branches barely move the
trunk, so a fixture could not tell a wrong branch from a right one), its BatchNorms get random statistics
(oracle.functional.randomize_bn_) and its own CPU fp32 forward runs.  Before anything is written, oracle.polynet.module_report
must show every residual module's scaled branch sum at >= MIN_RATIO of its input and every activation well inside fp16's range,
and oracle/polynet.py must reproduce the reference's features and logits bit for bit.  Stored: logits, a strided sample of the
features and of every module's output, the state_dict keys / shapes, the init digest, the registry row and the module report.
The TRN fixture holds the reference TRN-MSTRN's features and logits on PolyNet and its ``get_optim_policies()`` groups, partial
BN on and off.  Writes only these two files.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import pretorched_x_b200 as P                  # noqa: E402  (module geometry for the restatement)
from oracle import functional as OF            # noqa: E402
from oracle import polynet as OP               # noqa: E402
from oracle import reference_loader as RL      # noqa: E402
from oracle.make_golden import GOLDEN_DIR, SEED_BN, SEED_INIT, SEED_INPUT, summarize   # noqa: E402
from oracle.make_golden_trn_policies import named_policies, reference_trn   # noqa: E402

ARCH = 'polynet'
CLOSE = 0.15              # oracle.polynet.rescale_'s factor on the residual branches' closing 1x1 convolutions
MIN_RATIO, MAX_ACT = 0.1, 2048.0
SEED_TUPLES = 3
STAGE_SAMPLE = 512        # elements kept per module output (43 of them: the file stays well under 1 MB)
TRN_KW = dict(frame_bottleneck_dim=128, video_feature_dim=64)


def small_summary(t):
    flat = t.detach().reshape(-1)
    step = max(1, flat.numel() // STAGE_SAMPLE)
    return dict(shape=tuple(t.shape), absmax=float(t.abs().max()), sample=flat[::step][:STAGE_SAMPLE].clone(), step=step)


def run_case(shape=(2, 3, 331, 331)):
    pt = RL.load()
    torch.manual_seed(SEED_INIT)
    ref = RL.build(ARCH, num_classes=1000)
    init_sd = ref.state_dict()
    init_digest = OF.state_digest(init_sd)
    keys = [(k, tuple(v.shape)) for k, v in init_sd.items()]
    n_params = sum(p.numel() for p in ref.parameters())
    OP.rescale_(ref, CLOSE)
    OF.randomize_bn_(ref, SEED_BN)
    ref.eval()
    x = OF.seeded_input(shape, SEED_INPUT)
    sd = {k: v.detach().clone() for k, v in ref.state_dict().items()}
    geom = P.polynet(pretrained=None)
    with torch.no_grad():
        report, peak = OP.module_report(x[:1], sd, geom)
    worst = min(r[1] for r in report)
    assert worst >= MIN_RATIO and peak <= MAX_ACT, "rescaled init out of range: min ratio %.3f, peak %.1f" % (worst, peak)
    with torch.no_grad():
        feats = ref.features(x)
        logits = ref.logits(feats)
    stages = {}
    with torch.no_grad():
        f2 = OP.features(x, sd, geom, stages)
        out = OP.logits(f2, sd)
    assert torch.equal(f2, feats) and torch.equal(out, logits), "oracle restatement differs from the reference"
    name = "%s_b2_331" % ARCH
    torch.save(dict(kind="polynet", arch=ARCH, kwargs=dict(num_classes=1000), input_shape=tuple(shape), close=CLOSE,
                    seeds=dict(init=SEED_INIT, bn=SEED_BN, input=SEED_INPUT), keys=keys, n_params=n_params, init_digest=init_digest,
                    settings={ARCH: pt.pretrained_settings[ARCH]}, logits=logits.clone(), features=summarize(feats),
                    stages={k: small_summary(v) for k, v in stages.items()}, report=report, peak=peak,
                    weight_digest=OF.state_digest(sd), n_state=len(sd), torch_version=torch.__version__),
               os.path.join(GOLDEN_DIR, name + ".pt"))
    print("%-28s logits %s absmax %.4f; branch / input %.3f .. %.3f, peak activation %.1f"
          % (name, tuple(logits.shape), logits.abs().max(), worst, max(r[1] for r in report), peak))


def run_trn_case(T=4, B=1, hw=331):
    ref = reference_trn("MSTRN", ARCH, T, TRN_KW)
    pol = {}
    for pbn in (True, False):
        ref.partialBN(pbn)
        pol[pbn] = named_policies(ref)
    ref.partialBN(True)
    OP.rescale_(ref, CLOSE)
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
                    close=CLOSE, seeds=dict(init=SEED_INIT, bn=SEED_BN, input=SEED_INPUT, tuples=SEED_TUPLES), features=feats.clone(),
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
