#!/usr/bin/env python
"""One small forward of every model family (every kernel of the library on a real call path), meant to run under
compute-sanitizer (tools/sanitize.sh): memcheck for out-of-bounds / misaligned accesses, synccheck for barrier misuse.
Prints one line per case; a sanitizer error makes compute-sanitizer exit non-zero (--error-exitcode)."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import pretorched_x_b200 as P  # noqa: E402
from pretorched_x_b200 import _lib, engine  # noqa: E402
from oracle import functional as OF  # noqa: E402  (seeded BN statistics only)
from oracle import inceptionv3 as OV3  # noqa: E402  (Inception-v3's weights rescaled to stay in fp16 range)

dev = torch.device("cuda:0")
only = set(sys.argv[1:])


def case(name, build, shape, **kw):
    if only and name not in only:
        return
    torch.manual_seed(0)
    m = OF.randomize_bn_(build(), 1).eval().to(dev)
    x = torch.randn(shape, generator=torch.Generator().manual_seed(1)).to(dev)
    c0 = _lib.launch_count()
    with torch.no_grad():
        y = m(x, **kw)
    torch.cuda.synchronize()
    assert torch.isfinite(y.float()).all(), name
    print("%-28s in %-22s out %-14s launches %d" % (name, tuple(shape), tuple(y.shape), _lib.launch_count() - c0), flush=True)


case("resnet3d50", lambda: P.resnet3d50(num_classes=400, pretrained=None), (2, 3, 8, 64, 64))
case("resnet3d18", lambda: P.resnet3d18(num_classes=400, pretrained=None), (1, 3, 8, 64, 64))
case("resnet3d50_224", lambda: P.resnet3d50(num_classes=400, pretrained=None), (1, 3, 16, 224, 224))
case("r2plus1d34", lambda: P.r2plus1d34(num_classes=400), (1, 3, 8, 64, 64))
case("r2plus1d34_112", lambda: P.r2plus1d34(num_classes=400), (2, 3, 16, 112, 112))
case("resnet18", lambda: P.resnet18(num_classes=1000, pretrained=None), (3, 3, 64, 64))
case("resnet18_224", lambda: P.resnet18(num_classes=1000, pretrained=None), (40, 3, 224, 224))
case("resnet50", lambda: P.resnet50(num_classes=1000, pretrained=None), (2, 3, 64, 64))
case("resnext3d50", lambda: P.resnext3d50(num_classes=400), (1, 3, 8, 64, 64))
case("preact_resnet3d50", lambda: P.preact_resnet3d50(num_classes=400), (2, 3, 8, 64, 64))


if not only or "resnet3d50_t128" in only:
    # the slab kernel's 128-wide transposed form, forced (the rule takes it only at large batches), at stride 1 and 2
    lib = _lib.load()
    lib.b2_debug_set_densem(0, 0)
    lib.b2_debug_set_slab_t128(1)
    case("resnet3d50_t128", lambda: P.resnet3d50(num_classes=400, pretrained=None), (2, 3, 8, 64, 64))
    lib.b2_debug_set_slab_t128(-1)
    lib.b2_debug_set_densem(-1, 0)
case("nonlocalresnet3d50", lambda: P.nonlocalresnet3d50(pretrained=None), (1, 3, 16, 96, 96))
case("mobilenetv2", lambda: P.mobilenetv2(num_classes=1000, pretrained=None), (2, 3, 96, 64))
case("se_resnet50", lambda: P.se_resnet50(pretrained=None), (2, 3, 224, 224))
case("se_resnext50_32x4d", lambda: P.se_resnext50_32x4d(pretrained=None), (2, 3, 224, 224))
case("slowfast18", lambda: P.slowfast.resnet18(mode="sf", num_classes=12), (1, 3, 32, 64, 64))
case("densenet121", lambda: P.densenet121(pretrained=None), (2, 3, 224, 224))
case("densenet161", lambda: P.densenet161(pretrained=None), (1, 3, 224, 224))
case("inceptionv3", lambda: OV3.fan_in_scale_(P.inceptionv3(pretrained=None)), (1, 3, 299, 299))

if not only or "trn" in only:
    torch.manual_seed(0)
    m = OF.randomize_bn_(P.TRN(num_classes=339, num_segments=8, arch="resnet18", pretrained=None, consensus="MSTRN"), 1).eval().to(dev)
    x = torch.randn((2, 8, 3, 64, 64), generator=torch.Generator().manual_seed(3)).to(dev)
    with torch.no_grad():
        y = m(x)
    torch.cuda.synchronize()
    print("%-28s in %-22s out %-14s" % ("TRN(resnet18, MSTRN)", tuple(x.shape), tuple(y.shape)), flush=True)

if not only or "biggan" in only:
    from oracle import biggan as OB
    for res, B in ((128, 3), (256, 2)):
        model, _, z, lab = OB.build_case(P.biggan_deep, res, 16, 10, B, init="N02")
        with torch.no_grad():
            img = model.to(dev)(z.to(dev), lab.to(dev), out_dtype=torch.float16)
        torch.cuda.synchronize()
        assert torch.isfinite(img.float()).all()
        print("%-28s B %d -> %s" % ("biggan_deep%d (ch 16)" % res, B, tuple(img.shape)), flush=True)

if not only or "dfs" in only:
    # the chunked walk (out= row ranges, ragged chunk) on the kernels
    torch.manual_seed(0)
    m = OF.randomize_bn_(P.resnet3d50(num_classes=400, pretrained=None), 1).eval().to(dev)
    x = torch.randn((5, 3, 8, 64, 64), generator=torch.Generator().manual_seed(4)).to(dev)
    engine.set_dfs("5:2,4:3")
    with torch.no_grad():
        y = m(x)
    engine.set_dfs("off")
    torch.cuda.synchronize()
    print("%-28s %s" % ("resnet3d50 depth-first", tuple(y.shape)), flush=True)
if not only or "finetune" in only:
    # one fine-tuning step through layer3..layer4 (weight-gradient, zero-insert, mask, column-sum, loss-scale, pool backward)
    for arch in ("resnet3d50", "resnet3d18"):
        torch.manual_seed(0)
        m = OF.randomize_bn_(getattr(P, arch)(num_classes=10, pretrained=None), 1).eval().to(dev)
        groups = P.models.resnet3d.get_fine_tuning_parameters(m, 3)
        x = torch.randn((2, 3, 8, 64, 64), generator=torch.Generator().manual_seed(5)).to(dev)
        loss = torch.nn.functional.cross_entropy(m(x), torch.tensor([1, 2], device=dev))
        loss.backward()
        torch.optim.SGD(groups, lr=1e-5).step()
        torch.cuda.synchronize()
        assert all(torch.isfinite(p.grad).all() for p in m.parameters() if p.grad is not None)
        print("%-28s loss %.4f" % ("%s fine-tune step" % arch, loss.item()), flush=True)
if not only or "finetune2d" in only:
    # the 2-D / TRN fine-tuning step: (1, 3, 3) and (1, 1, 1) weight gradients, stride-2 zero insertion at T = 1, the relation's
    # differentiable path into the backbone
    torch.manual_seed(0)
    m = OF.randomize_bn_(P.resnet50(num_classes=10, pretrained=None), 1).eval().to(dev)
    groups = P.models.resnet3d.get_fine_tuning_parameters(m, 3)
    x = torch.randn((2, 3, 64, 64), generator=torch.Generator().manual_seed(6)).to(dev)
    loss = torch.nn.functional.cross_entropy(m(x), torch.tensor([1, 2], device=dev))
    loss.backward()
    torch.optim.SGD(groups, lr=1e-5).step()
    torch.manual_seed(0)
    t = OF.randomize_bn_(P.TRN(num_classes=10, num_segments=8, arch="resnet18", pretrained=None, consensus="MSTRN"), 1).eval().to(dev)
    t.fine_tune(3)
    x = torch.randn((2, 8, 3, 64, 64), generator=torch.Generator().manual_seed(7)).to(dev)
    tloss = torch.nn.functional.cross_entropy(t(x), torch.tensor([1, 2], device=dev))
    tloss.backward()
    torch.cuda.synchronize()
    for mod in (m, t):
        assert all(torch.isfinite(p.grad).all() for p in mod.parameters() if p.grad is not None)
    print("%-28s loss %.4f, TRN(resnet18, MSTRN) k=3 loss %.4f" % ("resnet50 2-D fine-tune step", loss.item(), tloss.item()), flush=True)
print("sanitize_run: done")
