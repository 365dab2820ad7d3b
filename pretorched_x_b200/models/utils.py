"""Small module helpers kept for API parity (reference: pretorched/models/utils.py:81-87), and the trunk container of the 2-D
zoo models whose ``features`` is an ``nn.Sequential`` in the reference."""
import torch.nn as nn


class Identity(nn.Module):
    """Drop-in replacement for ``last_linear`` when a caller wants pooled features (README.md:520-547)."""

    def forward(self, x):
        return x


class Trunk(nn.Sequential):
    """A model's ``features`` Sequential, kept under the reference's name so that its keys are ``features.<name>.*``.  Calling it
    runs the whole trunk on the engine (``_run``, defined by each model) and returns fp32 NCHW.  A slice (``features[a:b]``) is of
    the same class and refuses to run: the engine runs a trunk whole, never a part of it."""

    _partial = False
    _model = None              # the owning model's class name, for the refusal message

    def __getitem__(self, idx):
        out = super().__getitem__(idx)
        if isinstance(idx, slice):
            out._partial = True
        return out

    def forward(self, input):
        from .. import ops
        return ops.to_ncdhw(self.run_act(input)).squeeze(2)

    def check_runnable(self):
        if self._partial:
            raise NotImplementedError("%s.features[a:b] does not run on the engine: only the whole trunk does" % self._model)
        if self.training:
            raise RuntimeError("the forward engine is inference-only: call model.eval() first")

    def run_act(self, x):
        """The trunk's output on the engine's native layout (fp16 NDHWC ``Act``)."""
        self.check_runnable()
        return self._run(x)

    def _run(self, x):
        raise NotImplementedError
