"""Generate tests/golden/trn_optim_policies.pt from the UNMODIFIED reference (build container only):

    python -m oracle.make_golden_trn_policies

For the TRN configurations of oracle/make_golden.py (TRN_CASES) the reference's own ``TRN`` is built the way ``run_trn_cases``
builds it (the only patch: the backbone factory runs with ``pretrained=None`` and gets the registry's preprocessing attributes),
and its ``get_optim_policies()`` (trn.py:287-330) is called with partial BN on and off.  The fixture stores, per configuration
and setting, the five groups in order: name, lr_mult, decay_mult and the ``named_parameters`` names of the group's parameters in
order.  The tests compare ``pretorched_x_b200.TRN.get_optim_policies()`` against it without the reference.
"""
import contextlib
import io
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import reference_loader as RL      # noqa: E402
from oracle.make_golden import GOLDEN_DIR, SEED_INIT, TRN_CASES   # noqa: E402


def reference_trn(consensus, arch, T, kw):
    trn = RL.load_trn()
    pt = RL.load()
    orig = pt.__dict__[arch]

    def offline(num_classes=1000, pretrained=None):
        m = orig(num_classes=num_classes, pretrained=None)
        for k, v in pt.pretrained_settings[arch]['imagenet'].items():
            if k in ('input_space', 'input_size', 'input_range', 'mean', 'std'):
                setattr(m, k, v)
        return m
    pt.__dict__[arch] = offline
    try:
        torch.manual_seed(SEED_INIT)
        with contextlib.redirect_stdout(io.StringIO()):
            return trn.TRN(10, num_segments=T, arch=arch, consensus=consensus, pretrained=None, **kw)
    finally:
        pt.__dict__[arch] = orig


def named_policies(model):
    names = {id(p): n for n, p in model.named_parameters()}
    return [dict(name=g['name'], lr_mult=g['lr_mult'], decay_mult=g['decay_mult'], params=[names[id(p)] for p in g['params']])
            for g in model.get_optim_policies()]


def main():
    cases = {}
    for name, (consensus, arch, T, _B, _hw, kw, _np_seed) in TRN_CASES.items():
        ref = reference_trn(consensus, arch, T, kw)
        pol = {}
        for pbn in (True, False):
            ref.partialBN(pbn)
            pol[pbn] = named_policies(ref)
        cases[name] = dict(consensus=consensus, arch=arch, segments=T, kwargs=kw, policies=pol)
        print("%-24s groups (partial BN on) %s" % (name, [len(g['params']) for g in pol[True]]))
    torch.save(dict(kind="trn_optim_policies", cases=cases), os.path.join(GOLDEN_DIR, "trn_optim_policies.pt"))


if __name__ == "__main__":
    main()
