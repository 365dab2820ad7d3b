"""Temporal Relation Network heads (reference: pretorched/models/trn.py).

``Relation`` (trn.py:20-56) is ReLU -> Linear(T*F, bottleneck) -> ReLU -> Linear(bottleneck, out) over the
concatenated frame features; ``MultiScaleRelation`` (trn.py:59-113) sums such MLPs over sub-sampled frame
tuples of every scale.  Both keep the reference's parameter names (``relate.1.*``, ``relate.3.*``,
``relations.{i}.relate.*``); the bodies run as wgmma GEMMs with the bias / ReLU in the epilogue and the
cross-tuple sum accumulated in fp32 by the second GEMM.

Upstream defects mirrored, not fixed (SURVEY.md section 0.6-0.8): ``HierarchicalRelation`` with depth > 0
and ``MultiScaleHierarchicalRelation`` raise in the reference (torch.stack shape error), and the ``TRN``
wrapper / ``trn()`` factory cannot be built offline upstream (they need the missing ``pretrainedmodels`` package and a
downloaded backbone); here ``TRN`` is built on this package's own 2-D ResNets (see the class docstring).  The degenerate
``HierarchicalRelation`` (depth 0), which is what ``TRN(consensus='HTRN')`` actually instantiates, is provided.
"""
import itertools

import numpy as np
import torch
import torch.nn as nn

from .. import engine, ops
from .. import functions as Fn

__all__ = ['Relation', 'MultiScaleRelation', 'HierarchicalRelation', 'TRN', 'trn']


def _packed(linear):
    return engine._cached(linear, "pl", engine._sig(linear.weight, linear.bias),
                          lambda: ops.PackedLinear(linear.weight, linear.bias))


def _wants_grad(module):
    return torch.is_grad_enabled() and any(p.requires_grad for p in module.parameters())


class Relation(engine.CacheOwner, nn.Module):
    """input[..., num_inputs, in_features] -> output[batch, -1, out_features]"""

    def __init__(self, num_inputs, in_features, out_features, bottleneck_dim=512):
        super().__init__()
        self.num_inputs, self.in_features = num_inputs, in_features
        self.out_features, self.bottleneck_dim = out_features, bottleneck_dim
        self.relate = nn.Sequential(
            nn.ReLU(),
            nn.Linear(num_inputs * in_features, bottleneck_dim),
            nn.ReLU(),
            nn.Linear(bottleneck_dim, out_features),
        )

    def mlp_f16(self, x16, out=None, accumulate=False):
        """x16: fp16 [rows][num_inputs*in_features], already ReLU'd.  Returns fp32 [rows][out_features]."""
        hidden = ops.linear(x16, _packed(self.relate[1]), relu=True)
        return ops.linear(hidden, _packed(self.relate[3]), out_f32=True, out=out, accumulate=accumulate)

    def mlp_grad(self, flat):
        """Differentiable path (training a relation head): the same GEMM kernel through functions.LinearFunction, whose
        backward computes dX / dW on it too."""
        hidden = Fn.linear(flat, self.relate[1].weight, self.relate[1].bias, relu_input=True)
        return Fn.linear(hidden, self.relate[3].weight, self.relate[3].bias, relu_input=True)

    def forward(self, input):
        flat = input.contiguous().view(-1, self.num_inputs * self.in_features)
        if _wants_grad(self):
            return self.mlp_grad(flat.float()).view(input.size(0), -1, self.out_features)
        x16 = ops.cast_rows(flat, relu=True)          # leading nn.ReLU fused into the fp16 cast
        return self.mlp_f16(x16).view(input.size(0), -1, self.out_features)


class MultiScaleRelation(engine.CacheOwner, nn.Module):
    def __init__(self, num_input, in_features, out_features, bottleneck_dim=512, num_relations=3):
        super().__init__()
        self.num_input, self.in_features, self.out_features = num_input, in_features, out_features
        self.num_relations, self.bottleneck_dim = num_relations, bottleneck_dim
        self.scales = list(range(num_input, 1, -1))
        self.relations_scales = [self.return_relationset(num_input, s) for s in self.scales]
        self.subsample_scales = [min(num_relations, len(r)) for r in self.relations_scales]
        self.relations = nn.ModuleList(
            [Relation(s, in_features, out_features, bottleneck_dim) for s in self.scales])
        # one int32 table holds every sampled tuple of a forward: filled on the host (NumPy draws, as upstream), moved with a
        # single pinned -> device copy; scale si occupies [offset[si], offset[si] + n_si * s_i)
        self._offsets = np.cumsum([0] + [n * s for n, s in zip(self.subsample_scales, self.scales)]).tolist()
        self._host_table = None
        self._dev_table = None

    def return_relationset(self, num_input, num_input_relation):
        return list(itertools.combinations(range(num_input), num_input_relation))

    def sample_tuples(self):
        """The frame tuples one forward pass uses: np.random.choice per scale, exactly as trn.py:103-106
        (so seeding NumPy's global RNG reproduces the reference's choice)."""
        picks = []
        for si in range(len(self.scales)):
            idx = np.random.choice(len(self.relations_scales[si]), self.subsample_scales[si], replace=False)
            picks.append([self.relations_scales[si][i] for i in idx])
        return picks

    def upload_tuples(self, picks, device):
        """Writes ``picks`` into the persistent device table with ONE asynchronous copy from pinned host memory.  The table
        keeps its address, so a CUDA graph captured over ``forward_tuples`` is replayable: draw new tuples, call this, replay."""
        flat = [f for tuples in picks for tup in tuples for f in tup]
        if self._host_table is None or self._dev_table is None or self._dev_table.device != device:
            self._host_table = torch.empty(self._offsets[-1], dtype=torch.int32).pin_memory() if device.type == "cuda" \
                else torch.empty(self._offsets[-1], dtype=torch.int32)
            self._dev_table = torch.empty(self._offsets[-1], dtype=torch.int32, device=device)
        self._host_table.copy_(torch.tensor(flat, dtype=torch.int32))
        self._dev_table.copy_(self._host_table, non_blocking=True)
        return self._dev_table

    def _stacked_w2(self, rel, n):
        """Second Linear of a scale's MLP tiled ``n`` times along K, bias scaled by ``n``: sum_t (W2 h_t + b2) in one GEMM."""
        lin = rel.relate[3]

        def build():
            pl = ops.PackedLinear(lin.weight, lin.bias)
            w = pl.w.repeat(1, n).contiguous()            # [out][n * bottleneck_pitch]
            return w, pl.scale, (pl.shift * n).contiguous()
        return engine._cached(lin, "pl_x%d" % n, engine._sig(lin.weight, lin.bias), build)

    def forward_tuples(self, x16, table, total):
        """Launch sequence for tuples already resident in ``table`` (capture-safe: no host work, no allocation of indices).
        Per scale: one gather of all its tuples, one GEMM over (row, tuple) pairs, one GEMM that reduces over the tuples
        (K = n_tuples * bottleneck) and accumulates across scales in fp32 -- 3 launches per scale, 21 for 8 frames."""
        rows = x16.shape[0]
        for si, s in enumerate(self.scales):
            n = self.subsample_scales[si]
            rel = self.relations[si]
            idx = table[self._offsets[si]:self._offsets[si + 1]]
            gathered = ops.gather_frame_tuples(x16, idx, n, s)                    # [rows * n][s * F], tuple fastest
            hidden = ops.linear(gathered, _packed(rel.relate[1]), relu=True)       # [rows * n][bottleneck]
            if hidden.shape[1] != self.bottleneck_dim:
                raise ValueError("bottleneck_dim must be a multiple of 8 for the batched relation GEMM")
            w2, sc2, sh2 = self._stacked_w2(rel, n)
            ops.gemm(hidden.view(rows, n * self.bottleneck_dim), w2, sc2, sh2, rows, self.out_features,
                     n * self.bottleneck_dim, out=total, out_f32=True, accumulate=(si > 0))
        return total

    def forward(self, input):
        feats = input.contiguous().view(-1, self.num_input, self.in_features)
        rows = feats.shape[0]
        picks = self.sample_tuples()
        if _wants_grad(self):
            # differentiable path: per tuple, through LinearFunction (indexing and the sum are torch autograd ops)
            total = None
            for si, tuples in enumerate(picks):
                for tup in tuples:
                    y = self.relations[si].mlp_grad(feats[:, list(tup), :].reshape(rows, -1).float())
                    total = y if total is None else total + y
            return total.view(input.size(0), -1, self.out_features)
        x16 = ops.cast_rows(feats.view(rows, -1), relu=True).view(rows, self.num_input, -1)
        if x16.shape[2] != self.in_features:
            raise ValueError("in_features must be a multiple of 8 for the fp16 frame gather")
        table = self.upload_tuples(picks, input.device)
        total = torch.empty((rows, self.out_features), dtype=torch.float32, device=input.device)
        return self.forward_tuples(x16, table, total).view(input.size(0), -1, self.out_features)


class HierarchicalRelation(engine.CacheOwner, nn.Module):
    """Only the depth-0 configuration works upstream (trn.py:116-159); it reduces to one Relation over all
    inputs averaged with nothing else."""

    def __init__(self, num_inputs, in_features, out_features, relation_size=4, relation_dist=1, bottleneck_dim=1024):
        super().__init__()
        self.num_inputs, self.in_features, self.out_features = num_inputs, in_features, out_features
        self.relation_size, self.relation_dist, self.bottleneck_dim = relation_size, relation_dist, bottleneck_dim
        depth = int(np.ceil((num_inputs - relation_size) / (relation_size - 1)))
        if depth > 0:
            raise NotImplementedError(
                "HierarchicalRelation with depth > 0 raises a torch.stack shape error in the reference "
                "(trn.py:155-158); only the degenerate depth-0 form is reproducible")
        self.relations = nn.ModuleList([])
        self.linears = nn.ModuleList([])
        self.final_linear = nn.Linear(in_features, out_features)
        self.final_relation = Relation(num_inputs, in_features, out_features)

    def forward(self, input):
        x = input.view(-1, self.num_inputs, self.in_features)
        return self.final_relation(x)     # torch.stack([out]).mean(0) == out


class TRN(engine.CacheOwner, nn.Module):
    """Temporal Relation Network (trn.py:192-338): frames -> 2-D backbone -> temporal relation -> Linear.

    ``features`` (trn.py:246-255) folds the T frames of every clip into the batch of the 2-D backbone (``base_model``: one of
    this package's 2-D ResNets, whose ``last_linear`` is replaced by Dropout exactly as upstream, :211-212), regroups the
    pooled frame features as [B, 1, T, F] and applies the consensus module; ``logits`` (:257-258) is the final Linear.

    Upstream quirks kept (SURVEY.md section 0.6): the relation class receives ``frame_bottleneck_dim`` as its 4th POSITIONAL
    argument (trn.py:230-233), which for the default ``consensus='HTRN'`` is ``relation_size`` -- the module degenerates to
    one 8-frame ``Relation`` with a 512-wide bottleneck; 'MSHTRN' and HTRN with depth > 0 raise upstream and raise here.
    Upstream defect NOT kept (section 0.8): ``TRN(pretrained=None)`` crashes on ``base_model.std`` because preprocessing
    attributes are only attached by ``load_pretrained``; here they fall back to the backbone's ImageNet registry row."""

    def __init__(self, num_classes, num_segments=8, arch='resnet50', frame_bottleneck_dim=1024, video_feature_dim=1024,
                 consensus='HTRN', pretrained='moments', dropout=0.5, partial_bn=True):
        super().__init__()
        import pretorched_x_b200 as pkg
        self.arch, self.reshape, self.dropout = arch, True, dropout
        self._enable_pbn = True
        self.consensus, self.num_classes, self.num_segments = consensus, num_classes, num_segments
        self.video_feature_dim, self.frame_bottleneck_dim = video_feature_dim, frame_bottleneck_dim
        num_pc = 1000 if pretrained == 'imagenet' else 339
        self.base_model = pkg.__dict__[arch](num_pc, pretrained)
        self.frame_feature_dim = self.base_model.last_linear.in_features
        self.base_model.last_linear = nn.Dropout(self.dropout)
        settings = pkg.pretrained_settings[arch]['imagenet']
        self.std = getattr(self.base_model, 'std', settings['std'])
        self.mean = getattr(self.base_model, 'mean', settings['mean'])
        self.input_size = getattr(self.base_model, 'input_size', settings['input_size'])[1:]
        self.input_space = getattr(self.base_model, 'input_space', settings['input_space'])
        mods = {'TRN': Relation, 'HTRN': HierarchicalRelation, 'MSTRN': MultiScaleRelation}
        if consensus == 'MSHTRN':
            raise NotImplementedError("MultiScaleHierarchicalRelation raises a shape error upstream (trn.py:162-189)")
        if consensus not in mods:
            raise ValueError('Unrecognized temporal consensus.')
        self.temporal_relation = mods[consensus](self.num_segments, self.frame_feature_dim, self.video_feature_dim,
                                                 self.frame_bottleneck_dim)
        self.last_linear = nn.Linear(self.video_feature_dim, self.num_classes)

    def features(self, input):
        batch_size = input.size(0)
        base_rep = self.base_model(input.view((-1, 3) + input.size()[-2:]))
        base_rep = base_rep.view(batch_size, -1, self.num_segments, base_rep.size(-1))
        num_inputs = base_rep.size(1)
        t_in = base_rep.view(-1, num_inputs, self.num_segments, base_rep.size(-1))
        return self.temporal_relation(t_in).squeeze()

    def logits(self, features):
        feats = features.reshape(-1, self.video_feature_dim)
        head = self.last_linear
        if not isinstance(head, nn.Linear):
            return head(features)
        if _wants_grad(head):
            out = Fn.linear(feats.float(), head.weight, head.bias)
        else:
            out = ops.linear(ops.cast_rows(feats), _packed(head), out_f32=True)
        return out.view(features.shape[:-1] + (head.out_features,))

    def forward(self, input):
        return self.logits(self.features(input))

    def partialBN(self, enable):
        self._enable_pbn = enable

    @property
    def crop_size(self):
        return self.input_size

    @property
    def scale_size(self):
        return self.input_size[0] * 256 // 224


def trn(num_classes=339, num_segments=8, consensus='MSTRN', arch='resnet50', pretrained='moments',
        frame_bottleneck_dim=1024, video_feature_dim=1024):
    """trn.py:345-355.  Upstream ignores ``consensus`` / ``frame_bottleneck_dim`` / ``video_feature_dim`` here (the TRN is
    built with its class defaults); kept.  ``pretrained`` checkpoints need network access (model_zoo)."""
    if pretrained:
        raise RuntimeError("trn(pretrained=%r) downloads a checkpoint (trn.py:349-352); build with pretrained=None and "
                           "load_state_dict a local file" % (pretrained,))
    return TRN(num_classes=num_classes, num_segments=num_segments, arch=arch, pretrained=None)
