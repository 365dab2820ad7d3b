"""CUDA-graph replay of a whole forward pass.

A forward of resnet3d50 is ~75 kernel launches, each preceded by a Python -> ctypes crossing and a host-side
CUtensorMap encode; at H100 speeds that host work is comparable to the device time.  Capturing the launch
sequence once (static shapes, buffers from the graph's private pool) removes it: the timed step is one
``cudaGraphLaunch``.  All C-ABI entry points are capture-safe (no syncs, no allocations).

``GraphedFineTuneStep`` does the same for a whole fine-tuning step: forward, loss, backward and optimizer update.
"""
import numpy as np
import torch

from . import engine, ops


class GraphedForward:
    """``g = GraphedForward(model, example); y = g(x)`` with ``x`` of ``example``'s shape (device or pinned host).
    ``example`` may be a tuple of tensors for models that take several inputs (the BigGAN generator's ``(z, y)``);
    ``**kwargs`` are passed to every ``model(...)`` call."""

    def __init__(self, model, example_input, warmup=2, **kwargs):
        self.multi = isinstance(example_input, (tuple, list))
        examples = tuple(example_input) if self.multi else (example_input,)
        if not all(e.is_cuda for e in examples):
            raise RuntimeError("GraphedForward needs CUDA example inputs: the engine has no CPU path")
        self.model = model
        self.static_ins = tuple(e.detach().clone() for e in examples)
        self.static_in = self.static_ins if self.multi else self.static_ins[0]
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side), torch.no_grad():
            for _ in range(max(1, warmup)):          # packs weights, sets kernel attributes, warms the allocator
                model(*self.static_ins, **kwargs)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph), torch.no_grad():
            self.static_out = model(*self.static_ins, **kwargs)

    def load(self, x):
        """Copy new input(s) into the static buffers (asynchronously on the current stream)."""
        xs = tuple(x) if self.multi else (x,)
        for dst, src in zip(self.static_ins, xs):
            if src.data_ptr() != dst.data_ptr():
                dst.copy_(src, non_blocking=True)

    def __call__(self, x=None):
        if x is not None:
            self.load(x)
        self.graph.replay()
        return self.static_out


class PipelinedForward:
    """Host-fed inference loop: pinned host batches in, logits in pinned host memory out.

    Two ``GraphedForward`` replicas (own static input + activation pool, shared weights) alternate; the H2D copy
    of batch i+1 runs on a copy stream while the graph of batch i replays on the compute stream, and the logits
    of batch i are copied back asynchronously.  Steady-state cost per batch = max(H2D, forward) instead of their
    sum -- with fp32 NCDHW clips (the reference's input format) the PCIe copy is as long as the forward itself.
    """

    def __init__(self, model, example_input, depth=2, **kwargs):
        self.graphs = [GraphedForward(model, example_input, **kwargs) for _ in range(depth)]
        self.copy_stream = torch.cuda.Stream()
        self.compute_stream = torch.cuda.Stream()
        self.copied = [torch.cuda.Event() for _ in range(depth)]
        self.done = [torch.cuda.Event() for _ in range(depth)]
        out = self.graphs[0].static_out
        self.host_out = [torch.empty(out.shape, dtype=out.dtype).pin_memory() for _ in range(depth)]
        self.step = 0
        for ev in self.done:
            ev.record(self.compute_stream)

    def submit(self, host_batch):
        """Enqueue one pinned host batch; returns the index of the result slot (valid after ``wait(slot)``)."""
        d = self.step % len(self.graphs)
        g = self.graphs[d]
        with torch.cuda.stream(self.copy_stream):
            self.copy_stream.wait_event(self.done[d])          # slot's previous forward (and D2H) finished
            g.load(host_batch)
            self.copied[d].record(self.copy_stream)
        with torch.cuda.stream(self.compute_stream):
            self.compute_stream.wait_event(self.copied[d])
            g.graph.replay()
            self.host_out[d].copy_(g.static_out, non_blocking=True)
            self.done[d].record(self.compute_stream)
        self.step += 1
        return d

    def wait(self, slot):
        self.done[slot].synchronize()
        return self.host_out[slot]

    def drain(self):
        self.compute_stream.synchronize()
        self.copy_stream.synchronize()


def _check_optimizer(optimizer):
    """Refuse optimizers whose step keeps host-side state a graph would freeze."""
    if isinstance(optimizer, (torch.optim.Adam, torch.optim.AdamW)):
        if not all(g.get("capturable", False) for g in optimizer.param_groups):
            raise ValueError("GraphedFineTuneStep: %s must be built with capturable=True (its step count then lives on the "
                             "device)" % type(optimizer).__name__)
    elif not isinstance(optimizer, torch.optim.SGD):
        raise TypeError("GraphedFineTuneStep supports torch.optim.SGD and Adam / AdamW(capturable=True), got %s"
                        % type(optimizer).__name__)


def _snapshot(trainable, optimizer):
    return ([p.detach().clone() for p in trainable],
            {p: {k: v.clone() if torch.is_tensor(v) else v for k, v in st.items()} for p, st in optimizer.state.items()})


def _restore(trainable, optimizer, saved):
    """Put the parameters and the optimizer state back as ``_snapshot`` found them, in place (the graph keeps the addresses).
    State the warm-up created is zeroed: zero momentum / moment buffers and a zero step count are the fresh state."""
    params, state = saved
    with torch.no_grad():
        for p, v in zip(trainable, params):
            p.copy_(v)
        for p, st in optimizer.state.items():
            old = state.get(p, {})
            for k, v in st.items():
                if torch.is_tensor(v):
                    v.copy_(old[k]) if k in old else v.zero_()
                elif k in old:
                    st[k] = old[k]
            if isinstance(optimizer, torch.optim.SGD) and "momentum_buffer" in st and "momentum_buffer" not in old:
                group = next(g for g in optimizer.param_groups if any(q is p for q in g["params"]))
                if group["dampening"] != 0:
                    raise ValueError("GraphedFineTuneStep: SGD with dampening starts its momentum buffer from the first gradient, "
                                     "which a graph cannot do: take one eager step before capturing")


class GraphedFineTuneStep:
    """One fine-tuning step -- forward, ``loss_fn``, backward and ``optimizer.step()`` -- captured once and replayed.

    ``s = GraphedFineTuneStep(model, optimizer, loss_fn, example_input, example_target); loss = s(x, target)``: each call
    copies ``x`` / ``target`` (same shapes and dtypes as the examples; device or pinned host) into the static buffers, replays
    the step and returns the static fp32 loss tensor, overwritten by the next call.

    Models: those with ``fine_tune(k)`` (``ResNet3D``, ``ResNet2D``, ``TRN``) and frozen-trunk models with a trainable
    ``nn.Linear`` head.  The model stays in ``eval()`` (frozen BatchNorm); a model in ``train()`` mode is refused.

    Capture follows torch's whole-network recipe: ``warmup`` eager steps on a side stream, then the capture with the gradients
    allocated in the graph's pool -- after construction ``p.grad`` of every trainable parameter is a static tensor the
    replays rewrite.  The warm-up steps do not count: the parameters, the optimizer state and NumPy's global RNG are put
    back as they were, so the first replay is the first step.  While the step is captured every module that owns a trainable
    parameter, and every convolution whose folded BatchNorm is trainable, rebuilds its packed filter / folded affine on each
    call (``engine.repack_trainable``), so each replay packs the live parameters; packs of frozen tensors stay cached.  Every
    replay starts a new parameter epoch (``engine.parameters_changed``), so an eager forward never reuses a pack of trainable
    tensors made before the replay.  In-place edits of a trainable parameter (``with torch.no_grad(): p.mul_(0.5)``) reach
    the next replay; an edit of a frozen one does not (its pack is part of the graph).  The trainable set is fixed at capture:
    a call after ``requires_grad`` of a parameter changed raises.

    Optimizers: ``torch.optim.SGD`` (with or without momentum, Nesterov, weight decay; with dampening only when the momentum
    buffers already exist) and ``Adam`` / ``AdamW`` built with ``capturable=True``; anything else raises.  A Python-float
    learning rate is baked into the graph: changing ``param_groups[i]['lr']`` afterwards has no effect -- capture again, or
    give the optimizer a tensor ``lr``.  Learning-rate schedules are not captured.

    TRN's ``MultiScaleRelation`` draws its frame tuples on the host (``np.random``, as the reference does); each call draws
    them for that step and writes them into the relation's persistent tuple table before the replay, so seeding NumPy the
    same way before an eager step and before a call gives both the same tuples.

    The capture runs eager steps and synchronises: it cannot run inside ``ops.profile()``.
    """

    def __init__(self, model, optimizer, loss_fn, example_input, example_target, warmup=2):
        if model.training:
            raise RuntimeError("GraphedFineTuneStep: the engine trains with frozen BatchNorm -- call model.eval() first")
        if ops._PROFILE is not None:
            raise RuntimeError("GraphedFineTuneStep cannot capture inside ops.profile(): its per-launch events would be "
                               "captured and its exit synchronises")
        if not (example_input.is_cuda and example_target.is_cuda):
            raise RuntimeError("GraphedFineTuneStep needs CUDA example tensors: the engine has no CPU path")
        _check_optimizer(optimizer)
        self.model, self.optimizer = model, optimizer
        self.trainable = [p for p in model.parameters() if p.requires_grad]
        if not self.trainable:
            raise ValueError("GraphedFineTuneStep: the model has no trainable parameter (call fine_tune(k) or unfreeze a head)")
        self._params = list(model.parameters())
        self._trainable_mask = [p.requires_grad for p in self._params]
        self.relations = [m for m in model.modules() if hasattr(m, "sample_tuples") and hasattr(m, "upload_tuples")]
        self.static_input = example_input.detach().clone()
        self.static_target = example_target.detach().clone()

        def step():
            optimizer.zero_grad(set_to_none=True)
            loss = loss_fn(model(self.static_input), self.static_target)
            loss.backward()
            optimizer.step()
            return loss

        np_state = np.random.get_state()
        saved = _snapshot(self.trainable, optimizer)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(max(1, warmup)):      # packs frozen weights, creates the optimizer state, warms the allocator
                step()
        torch.cuda.current_stream().wait_stream(side)
        _restore(self.trainable, optimizer, saved)
        del saved
        optimizer.zero_grad(set_to_none=True)    # the captured backward allocates the gradients in the graph's pool
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with engine.repack_trainable(), torch.cuda.graph(self.graph):
            self.static_loss = step().detach()   # keeps no autograd node of the captured step alive
        engine.parameters_changed()
        np.random.set_state(np_state)

    @staticmethod
    def _load(dst, src, what):
        if tuple(src.shape) != tuple(dst.shape) or src.dtype != dst.dtype:
            raise ValueError("GraphedFineTuneStep was captured for a %s of %s %s, got %s %s" % (what, tuple(dst.shape), dst.dtype,
                                                                                             tuple(src.shape), src.dtype))
        if src.data_ptr() != dst.data_ptr():
            dst.copy_(src, non_blocking=True)

    def __call__(self, x=None, target=None):
        if [p.requires_grad for p in self._params] != self._trainable_mask:
            raise RuntimeError("GraphedFineTuneStep: requires_grad of a parameter changed since the capture; the graph still "
                               "trains the parameters that were trainable then -- build a new GraphedFineTuneStep")
        if x is not None:
            self._load(self.static_input, x, "input")
        if target is not None:
            self._load(self.static_target, target, "target")
        for rel in self.relations:
            rel.upload_tuples(rel.sample_tuples(), self.static_input.device)
        self.graph.replay()
        engine.parameters_changed()
        return self.static_loss
