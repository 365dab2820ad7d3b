"""CPU: the packed-parameter cache switch behind graph-captured fine-tuning (engine.repack_trainable), the optimizer checks and
state restore of graph.GraphedFineTuneStep, and the tuple-table layout the relation's differentiable path indexes."""
import numpy as np
import pytest
import torch
import torch.nn as nn

import pretorched_x_b200 as P
from pretorched_x_b200 import engine
from pretorched_x_b200 import graph as G


def _net():
    """A frozen and a trainable owner under one root."""
    root = nn.Sequential(nn.Linear(4, 4), nn.Sequential(nn.Linear(4, 4)))
    for p in root[0].parameters():
        p.requires_grad_(False)
    return root, root[0], root[1][0]


class _Builds:
    def __init__(self):
        self.n = 0

    def __call__(self):
        self.n += 1
        return object()


def _get(owner, builds):
    return engine._cached(owner, "slot", engine._sig(owner.weight, owner.bias), builds)


def test_trainable_packs_rebuild_on_every_call_while_switch_is_on():
    root, frozen, trained = _net()
    bf, bt = _Builds(), _Builds()
    with engine.repack_trainable():
        assert engine.repacking_trainable()
        vals_t = [_get(trained, bt) for _ in range(3)]
        vals_f = [_get(frozen, bf) for _ in range(3)]
    assert not engine.repacking_trainable()
    assert bt.n == 3 and len({id(v) for v in vals_t}) == 3
    assert bf.n == 1 and all(v is vals_f[0] for v in vals_f)
    # a rebuilt pack is not stored: after the switch the trainable owner builds afresh, the frozen one hits
    assert "slot" not in trained.__dict__.get("_b2_cache", {})
    _get(trained, bt)
    assert bt.n == 4
    assert _get(frozen, bf) is vals_f[0] and bf.n == 1


def test_switch_nests_and_is_off_by_default():
    assert not engine.repacking_trainable()
    with engine.repack_trainable():
        with engine.repack_trainable():
            pass
        assert engine.repacking_trainable()
    assert not engine.repacking_trainable()


def test_pack_follows_the_tensors_it_reads():
    """A pack is trainable when its owner (or a child) has a trainable parameter, or when a tensor it folds does: a frozen
    convolution whose BatchNorm is trained."""
    root, frozen, trained = _net()
    assert engine._reads_trainable(root, ()) and engine._reads_trainable(root[1], ()) and engine._reads_trainable(trained, ())
    assert not engine._reads_trainable(frozen, ()) and not engine._reads_trainable(object(), (None,))
    conv, bn = nn.Conv2d(4, 4, 1, bias=False), nn.BatchNorm2d(4)
    conv.weight.requires_grad_(False)
    assert engine._reads_trainable(conv, engine._bn_tensors(bn))
    bn.requires_grad_(False)
    assert not engine._reads_trainable(conv, engine._bn_tensors(bn))


def test_frozen_conv_with_trainable_bn_is_rebuilt_and_follows_the_epoch():
    conv, bn = nn.Conv2d(4, 4, 1, bias=False), nn.BatchNorm2d(4)
    conv.weight.requires_grad_(False)
    builds = _Builds()
    get = lambda: engine._cached(conv, "pc", engine._sig(conv.weight, *engine._bn_tensors(bn)), builds,
                                 reads=engine._bn_tensors(bn))
    with engine.repack_trainable():
        get(), get()
    assert builds.n == 2 and "pc" not in conv.__dict__.get("_b2_cache", {})
    first = get()
    assert get() is first and builds.n == 3
    engine.parameters_changed()
    assert get() is not first and builds.n == 4


def test_new_epoch_rebuilds_only_packs_of_trainable_tensors():
    """After a replay (engine.parameters_changed) a pack made before it is not reused unless it reads only frozen tensors."""
    root, frozen, trained = _net()
    bf, bt, br = _Builds(), _Builds(), _Builds()
    pf, pt = _get(frozen, bf), _get(trained, bt)
    ph = engine._cached(root, "head", (), br)                # an owner whose trainable parameter sits in a child
    assert _get(trained, bt) is pt and bt.n == 1             # same epoch, same key: a hit
    engine.parameters_changed()
    assert _get(frozen, bf) is pf and bf.n == 1
    assert _get(trained, bt) is not pt and bt.n == 2
    assert engine._cached(root, "head", (), br) is not ph and br.n == 2
    engine.invalidate(root)                                   # the full invalidation still drops everything
    assert "_b2_cache" not in frozen.__dict__


def test_optimizer_checks():
    p = [nn.Parameter(torch.zeros(3))]
    G._check_optimizer(torch.optim.SGD(p, lr=0.1, momentum=0.9))
    G._check_optimizer(torch.optim.Adam(p, lr=0.1, capturable=True))
    G._check_optimizer(torch.optim.AdamW(p, lr=0.1, capturable=True))
    with pytest.raises(ValueError, match="capturable"):
        G._check_optimizer(torch.optim.Adam(p, lr=0.1))
    with pytest.raises(TypeError, match="SGD"):
        G._check_optimizer(torch.optim.RMSprop(p, lr=0.1))


def _sgd_steps(opt, params, n):
    for i in range(n):
        for q in params:
            q.grad = torch.full_like(q, 0.5 + i)
        opt.step()


@pytest.mark.parametrize("kind", ["sgd", "adam"])
def test_restore_returns_parameters_and_optimizer_state(kind):
    torch.manual_seed(0)
    params = [nn.Parameter(torch.randn(5)), nn.Parameter(torch.randn(2, 3))]
    opt = (torch.optim.SGD(params, lr=0.1, momentum=0.9) if kind == "sgd" else torch.optim.Adam(params, lr=0.1))
    _sgd_steps(opt, params, 1)                                # existing state comes back with its values
    want_p = [q.detach().clone() for q in params]
    want_s = {k: v.clone() for k, v in opt.state[params[0]].items()}
    saved = G._snapshot(params, opt)
    _sgd_steps(opt, params, 3)
    G._restore(params, opt, saved)
    assert all(torch.equal(q, w) for q, w in zip(params, want_p))
    assert opt.state[params[0]].keys() == want_s.keys()
    for k, v in want_s.items():
        assert torch.equal(torch.as_tensor(opt.state[params[0]][k]), torch.as_tensor(v)), k


def test_restore_zeroes_state_created_by_the_warmup():
    params = [nn.Parameter(torch.ones(4))]
    opt = torch.optim.SGD(params, lr=0.1, momentum=0.9)
    saved = G._snapshot(params, opt)
    _sgd_steps(opt, params, 2)
    buf_before = opt.state[params[0]]["momentum_buffer"]
    G._restore(params, opt, saved)
    assert opt.state[params[0]]["momentum_buffer"] is buf_before and torch.equal(buf_before, torch.zeros(4))
    assert torch.equal(params[0].detach(), torch.ones(4))
    damp = torch.optim.SGD(params, lr=0.1, momentum=0.9, dampening=0.1)
    saved = G._snapshot(params, damp)
    _sgd_steps(damp, params, 1)
    with pytest.raises(ValueError, match="dampening"):
        G._restore(params, damp, saved)


def test_zero_momentum_buffer_gives_torchs_first_step():
    """The captured SGD step always takes the 'buffer exists' branch: from a zero buffer it equals torch's first step."""
    torch.manual_seed(1)
    w0 = torch.randn(64)
    g = torch.randn(64)
    for foreach in (False, True):
        a, b = nn.Parameter(w0.clone()), nn.Parameter(w0.clone())
        oa = torch.optim.SGD([a], lr=0.37, momentum=0.9, weight_decay=1e-4, foreach=foreach)
        ob = torch.optim.SGD([b], lr=0.37, momentum=0.9, weight_decay=1e-4, foreach=foreach)
        ob.state[b]["momentum_buffer"] = torch.zeros(64)
        a.grad, b.grad = g.clone(), g.clone()
        oa.step()
        ob.step()
        assert torch.equal(a, b) and torch.equal(oa.state[a]["momentum_buffer"], ob.state[b]["momentum_buffer"])


def test_refuses_a_model_in_train_mode():
    model = nn.Linear(4, 2).train()
    with pytest.raises(RuntimeError, match="eval"):
        G.GraphedFineTuneStep(model, torch.optim.SGD(model.parameters(), lr=0.1), nn.functional.mse_loss,
                              torch.zeros(1, 4), torch.zeros(1, 2))


def test_relation_tuple_table_slices_are_the_drawn_tuples():
    """The differentiable relation path indexes frames with slices of the tuple table: slice j of scale si holds picks[si][j]."""
    r = P.MultiScaleRelation(8, 16, 4, bottleneck_dim=8)
    np.random.seed(3)
    picks = r.sample_tuples()
    table = r.upload_tuples(picks, torch.device("cpu"))
    for si, s in enumerate(r.scales):
        assert len(picks[si]) == r.subsample_scales[si]
        for j, tup in enumerate(picks[si]):
            o = r._offsets[si] + j * s
            assert table[o:o + s].tolist() == list(tup)
    feats = torch.randn(2, 8, 16)
    tup = picks[1][2]
    o = r._offsets[1] + 2 * r.scales[1]
    assert torch.equal(feats.index_select(1, table[o:o + r.scales[1]]), feats[:, list(tup), :])
