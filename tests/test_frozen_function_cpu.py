"""CPU: the frozen-block autograd boundary (functions.frozen / FrozenFunction) with plain-torch bodies on CPU tensors -- what it
returns, that its outputs are constants to autograd next to trainable tensors, and that an ``out=`` row range is written in place."""
import torch

from pretorched_x_b200 import functions as Fn
from pretorched_x_b200.ops import Act


def _act(N=2, T=1, H=3, W=4, C=6, ld=8, requires_grad=False):
    data = torch.randn(N * T * H * W, ld, generator=torch.Generator().manual_seed(0)).requires_grad_(requires_grad)
    return Act(data, N, T, H, W, C)


def _pool_w(x, out=None):
    """A body that changes the geometry: the mean of each pair of columns (W halves), written into ``out`` when given."""
    y = x.data.view(-1, 2, x.ld).mean(1)
    if out is not None:
        out.copy_(y)
        y = out
    return Act(y, x.N, x.T, x.H, x.W // 2, x.C)


def _geom(a):
    return (a.N, a.T, a.H, a.W, a.C, a.ld)


def test_single_output_keeps_its_geometry():
    a = _act()
    y = Fn.frozen(_pool_w, a)
    assert isinstance(y, Act)
    assert _geom(y) == (2, 1, 3, 2, 6, 8)
    assert torch.equal(y.data, _pool_w(a).data)


def test_pair_output_keeps_both_geometries():
    a = _act()
    y, h = Fn.frozen(lambda x, o: (_pool_w(x, o), Act(x.data[:, :4] * 2, x.N, x.T, x.H, x.W, 4)), a)
    assert _geom(y) == (2, 1, 3, 2, 6, 8)
    assert _geom(h) == (2, 1, 3, 4, 4, 4)
    assert torch.equal(h.data, a.data[:, :4] * 2)


def test_pair_with_none_comes_back_as_pair_with_none():
    res = Fn.frozen(lambda x, o: (_pool_w(x, o), None), _act())
    assert isinstance(res, tuple) and len(res) == 2
    assert isinstance(res[0], Act) and res[1] is None


def test_outputs_do_not_require_grad_in_grad_mode():
    a = _act(requires_grad=True)
    with torch.enable_grad():
        y = Fn.frozen(_pool_w, a)
        p, q = Fn.frozen(lambda x, o: (_pool_w(x, o), _pool_w(x)), a)
    assert not any(t.data.requires_grad for t in (y, p, q))


def test_trainable_tensor_behind_frozen_output_gets_its_gradient():
    a = _act(requires_grad=True)
    w = torch.full((8,), 3.0, requires_grad=True)
    y = Fn.frozen(_pool_w, a)
    (y.data * w).sum().backward()
    assert torch.equal(w.grad, y.data.sum(0))
    assert a.data.grad is None


def test_out_row_view_is_written_in_place_and_returned():
    a = _act()
    buf = torch.zeros(3 * 12, 8)
    out = buf[12:24]                                   # the middle row range of a larger buffer
    y = Fn.frozen(_pool_w, a, out)
    assert y.data.data_ptr() == out.data_ptr()
    assert torch.equal(buf[12:24], _pool_w(a).data)
    assert not buf[:12].any() and not buf[24:].any()
