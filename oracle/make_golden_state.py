"""Write tests/golden/reference_state_sha256.json: for a few architectures, the number of tensors and ONE SHA-256 over the
key order, shapes, dtypes and bytes of every tensor of the seeded state_dict the UNMODIFIED reference builds (needs the
reference tree; see reference_loader).  tests/test_oracle_golden.py requires the package's seeded init to hash the same.

Usage:  python -m oracle.make_golden_state
"""
import hashlib
import json
import os
import warnings

import torch

from oracle import reference_loader as RL

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "..", "tests", "golden", "reference_state_sha256.json")

# (arch, factory kwargs, torch seed); R(2+1)D first: reference_loader.load_r2plus1d documents why
CASES = [
    ("r2plus1d18", dict(num_classes=400), 3),
    ("resnet3d50", dict(num_classes=400), 3),
    ("nonlocalresnet3d50", dict(), 3),
    ("resnext3d50", dict(num_classes=400), 5),
    ("resnext3d18", dict(num_classes=10, shortcut_type="A"), 5),
    ("resnext3d101", dict(), 5),
]


def state_sha256(sd):
    h = hashlib.sha256()
    for k, t in sd.items():
        t = t.detach().cpu().contiguous()
        h.update(k.encode() + str(t.dtype).encode() + str(tuple(t.shape)).encode() + t.numpy().tobytes())
    return h.hexdigest()


def main():
    RL.load(); RL.load_r2plus1d()
    out = []
    for arch, kw, seed in CASES:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            torch.manual_seed(seed)
            sd = RL.build(arch, **kw).state_dict()
        out.append({"arch": arch, "kwargs": kw, "seed": seed, "n_state": len(sd), "sha256": state_sha256(sd)})
    with open(OUT, "w") as fh:
        json.dump(out, fh, indent=1)
        fh.write("\n")
    print("wrote", os.path.normpath(OUT))


if __name__ == "__main__":
    main()
