"""GPU: a fine-tuning step captured in one CUDA graph (graph.GraphedFineTuneStep) against the same step run eagerly.

Every kernel on the fine-tuning path is deterministic (fixed-order weight-gradient and column-sum reductions), and a replay
runs the same kernels on the same values as the eager step, so replayed and eager training agree bit for bit: losses,
parameters and optimizer state."""
import copy

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import pretorched_x_b200 as P
from pretorched_x_b200 import ops
from pretorched_x_b200.graph import GraphedFineTuneStep
from oracle import functional as OF
from tests.conftest import has_h100

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_h100(), reason="needs an H100")]

dev = torch.device("cuda:0")


def _resnet3d(arch, k):
    def make():
        torch.manual_seed(0)
        m = OF.randomize_bn_(getattr(P, arch)(num_classes=10, pretrained=None), 1).eval()
        return m.fine_tune(k) if k else m
    return make


def _resnet18(k):
    def make():
        torch.manual_seed(0)
        return OF.randomize_bn_(P.resnet18(num_classes=10, pretrained=None), 1).eval().fine_tune(k)
    return make


def _trn(k):
    def make():
        torch.manual_seed(0)
        m = P.TRN(10, num_segments=8, arch="resnet18", consensus="MSTRN", pretrained=None)
        return OF.randomize_bn_(m, 1).eval().fine_tune(k)
    return make


def _head_only():
    """Frozen resnet3d18 trunk, trainable last_linear (functions.LinearFunction)."""
    m = _resnet3d("resnet3d18", 0)()
    for n, p in m.named_parameters():
        p.requires_grad_(n.startswith("last_linear."))
    return m


def _bn_only(k):
    """fine_tune(k), then the convolutions of the trained stages frozen: BatchNorm gamma / beta and the head are trained, and
    the frozen convolutions' packs fold trainable BatchNorm affines."""
    def make():
        m = _resnet3d("resnet3d18", k)()
        for n, p in m.named_parameters():
            if p.requires_grad and p.dim() == 5:
                p.requires_grad_(False)
        return m
    return make


def _sgd(m):
    return torch.optim.SGD([p for p in m.parameters() if p.requires_grad], lr=1e-3, momentum=0.9)


def _adam(m):
    return torch.optim.Adam([p for p in m.parameters() if p.requires_grad], lr=1e-4, capturable=True)


def _twins(make, opt_fn):
    base = make()
    a, b = copy.deepcopy(base).to(dev), copy.deepcopy(base).to(dev)
    return a, opt_fn(a), b, opt_fn(b)


def _eager_step(model, opt, x, target):
    opt.zero_grad(set_to_none=True)
    loss = F.cross_entropy(model(x), target)
    loss.backward()
    opt.step()
    return loss.detach().clone()


def _inputs(shape, n, seed=10):
    xs = [OF.seeded_input(shape, seed + i).to(dev) for i in range(n)]
    ts = [(torch.arange(shape[0], device=dev) * (3 + i)) % 10 for i in range(n)]
    return xs, ts


def _assert_same_training(a, oa, b, ob, state=True):
    for (n, p), (_, q) in zip(a.named_parameters(), b.named_parameters()):
        assert torch.equal(p, q), n
        if not state:
            continue
        sa, sb = oa.state.get(p, {}), ob.state.get(q, {})
        assert sa.keys() == sb.keys(), n
        for key in sa:
            assert torch.equal(torch.as_tensor(sa[key]), torch.as_tensor(sb[key])), (n, key)


CASES = [
    # id, model factory, optimizer, input shape
    ("resnet3d18_k3_sgd", _resnet3d("resnet3d18", 3), _sgd, (2, 3, 8, 64, 64)),
    ("resnet3d50_k4_sgd", _resnet3d("resnet3d50", 4), _sgd, (2, 3, 8, 64, 64)),
    ("resnet18_k3_sgd", _resnet18(3), _sgd, (4, 3, 64, 64)),
    ("trn_mstrn_resnet18_k4_sgd", _trn(4), _sgd, (2, 8, 3, 64, 64)),
    ("resnet3d18_k4_adam", _resnet3d("resnet3d18", 4), _adam, (2, 3, 8, 64, 64)),
    ("resnet3d18_head_only_sgd", _head_only, _sgd, (2, 3, 8, 64, 64)),
    ("resnet3d18_k3_bn_only_sgd", _bn_only(3), _sgd, (2, 3, 8, 64, 64)),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_replay_equals_eager_bitwise(case):
    _, make, opt_fn, shape = case
    eager, e_opt, graphed, g_opt = _twins(make, opt_fn)
    xs, ts = _inputs(shape, 4)
    step = GraphedFineTuneStep(graphed, g_opt, F.cross_entropy, xs[0], ts[0])
    _assert_same_training(eager, e_opt, graphed, g_opt, state=False)     # construction trains nothing
    assert all(torch.count_nonzero(v) == 0 for st in g_opt.state.values() for v in st.values())
    losses = []
    for i, (x, t) in enumerate(zip(xs, ts)):
        np.random.seed(100 + i)
        want = _eager_step(eager, e_opt, x, t)
        np.random.seed(100 + i)
        got = step(x, t).clone()
        assert got.dtype == torch.float32
        assert torch.equal(got, want), (i, got.item(), want.item())
        losses.append(got.item())
    _assert_same_training(eager, e_opt, graphed, g_opt)
    assert all(np.isfinite(losses)), losses


STALE_CASES = [
    # id, model factory, parameters edited in place after the capture
    ("resnet3d18_k3", _resnet3d("resnet3d18", 3), ("layer4.0.conv1.weight", "layer3.1.bn2.weight")),
    ("resnet3d18_k3_bn_only", _bn_only(3), ("layer4.0.bn1.weight", "layer3.1.bn2.bias")),
]


@pytest.mark.parametrize("case", STALE_CASES, ids=[c[0] for c in STALE_CASES])
def test_parameters_reach_the_graph_and_no_pack_is_stale(case):
    _, make, edited = case
    eager, e_opt, graphed, g_opt = _twins(make, _sgd)
    (x,), (t,) = _inputs((2, 3, 8, 64, 64), 1)
    step = GraphedFineTuneStep(graphed, g_opt, F.cross_entropy, x, t)
    stem = graphed.conv1.__dict__["_b2_cache"]["pc"][1]
    frozen_conv = graphed.layer1[0].conv1.__dict__["_b2_cache"]["pc"][1]
    frozen = {n: p.detach().clone() for n, p in graphed.named_parameters() if not p.requires_grad}
    with torch.no_grad():
        graphed(x)                                   # caches packs of the trainable layers as they are now
    losses = []
    for _ in range(3):
        want = _eager_step(eager, e_opt, x, t)
        got = step().clone()
        assert torch.equal(got, want)
        losses.append(got.item())
    assert len(set(losses)) == 3, losses             # the same batch, a lower loss: the updates reach the forward
    # in-place edits after capture reach the next replay: a packed filter and a folded BatchNorm affine
    for m in (eager, graphed):
        params = dict(m.named_parameters())
        with torch.no_grad():
            for name in edited:
                params[name].mul_(0.5)
    assert torch.equal(step().clone(), _eager_step(eager, e_opt, x, t))
    _assert_same_training(eager, e_opt, graphed, g_opt)
    # after the replays the eager forward uses packs of the trained parameters
    fresh = make().to(dev)
    fresh.load_state_dict(graphed.state_dict())
    with torch.no_grad():
        assert torch.equal(graphed(x), fresh(x))
    # frozen parts: parameters unchanged, packs the very same tensors as before the replays
    for n, p in graphed.named_parameters():
        if n in frozen:
            assert torch.equal(p, frozen[n]), n
    assert graphed.conv1.__dict__["_b2_cache"]["pc"][1] is stem
    assert graphed.layer1[0].conv1.__dict__["_b2_cache"]["pc"][1] is frozen_conv


def test_trn_replays_use_the_tuples_drawn_for_each_step():
    """With lr = 0 the parameters stay put, so two replays differ only by their frame tuples."""
    def zero_lr(m):
        return torch.optim.SGD([p for p in m.parameters() if p.requires_grad], lr=0.0, momentum=0.9)
    eager, e_opt, graphed, g_opt = _twins(_trn(4), zero_lr)
    (x,), (t,) = _inputs((2, 8, 3, 64, 64), 1)
    step = GraphedFineTuneStep(graphed, g_opt, F.cross_entropy, x, t)
    rel = graphed.temporal_relation
    picks = []
    for seed in (1, 2):
        np.random.seed(seed)
        picks.append(rel.sample_tuples())
    assert picks[0] != picks[1]
    got = []
    for seed in (1, 2):
        np.random.seed(seed)
        want = _eager_step(eager, e_opt, x, t)
        np.random.seed(seed)
        got.append(step(x, t).clone())
        assert torch.equal(got[-1], want), seed
    assert not torch.equal(got[0], got[1])


def test_refusals():
    make = _resnet3d("resnet3d18", 4)
    (x,), (t,) = _inputs((2, 3, 8, 64, 64), 1)
    m = make().to(dev)
    with pytest.raises(RuntimeError, match="eval"):
        GraphedFineTuneStep(m.train(), _sgd(m), F.cross_entropy, x, t)
    m.eval()
    with pytest.raises(RuntimeError, match="profile"):
        with ops.profile():
            GraphedFineTuneStep(m, _sgd(m), F.cross_entropy, x, t)
    with pytest.raises(ValueError, match="capturable"):
        GraphedFineTuneStep(m, torch.optim.Adam([p for p in m.parameters() if p.requires_grad]), F.cross_entropy, x, t)
    step = GraphedFineTuneStep(m, _sgd(m), F.cross_entropy, x, t)
    m.layer4[0].conv1.weight.requires_grad_(False)
    with pytest.raises(RuntimeError, match="requires_grad"):
        step(x, t)
    m.layer4[0].conv1.weight.requires_grad_(True)
    with pytest.raises(ValueError, match="captured for"):
        step(x[:1], t[:1])
    with pytest.raises(ValueError, match="captured for"):
        step(x, t.float())
    assert torch.isfinite(step(x, t)).item()


def test_trn_two_forwards_before_one_backward():
    """Gradient accumulation over two forwards, with an evaluation forward in between, before one backward: each forward's
    backward reads its own frame tuples, and the gradients are those of two separate backwards."""
    make = _trn(4)
    a, b = make().to(dev), make().to(dev)
    xs, ts = _inputs((2, 8, 3, 64, 64), 2)
    np.random.seed(5)
    la = F.cross_entropy(a(xs[0]), ts[0])
    with torch.no_grad():
        np.random.seed(9)
        a(xs[1])
    np.random.seed(6)
    (la + F.cross_entropy(a(xs[1]), ts[1])).backward()
    for seed, x, t in ((5, xs[0], ts[0]), (6, xs[1], ts[1])):
        np.random.seed(seed)
        F.cross_entropy(b(x), t).backward()
    n_grads = 0
    for (n, p), (_, q) in zip(a.named_parameters(), b.named_parameters()):
        assert (p.grad is None) == (q.grad is None), n
        if p.grad is not None:
            n_grads += 1
            torch.testing.assert_close(p.grad, q.grad, rtol=1e-5, atol=1e-7, msg=n)
    assert n_grads > 0
