"""CPU restatement of the reference's PNASNet-5-Large forward (pretorched/models/pnasnet.py:33-369) -- TEST INFRASTRUCTURE.

Plain functional torch over a ``state_dict`` in the reference's layout, in the reference's order of operations: ZeroPad2d and crop
included where the reference pads, BatchNorm eps 1e-3.  The cell table is ``pretorched_x_b200.models.pnasnet.CELLS``.  Pinned bit
for bit against the unmodified reference by oracle/make_golden_pnasnet.py.  Works in the dtype of its inputs.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

BN_EPS = 1e-3
STAGES = ['conv_0', 'cell_stem_0', 'cell_stem_1'] + ['cell_%d' % i for i in range(12)]
REDUCTION = {'cell_stem_1', 'cell_4', 'cell_8'}
ZERO_PAD = {'cell_4'}
FACTORIZED = {'cell_stem_1', 'cell_0', 'cell_5', 'cell_9'}


def rescale_(model, factor=1.7):
    """The fixture's init, applied after the seeded init (whose digest the fixture records first) and before
    ``oracle.functional.randomize_bn_``: every Conv2d weight times ``factor``.  At PyTorch's default init the activations shrink
    cell by cell (cell_11's std near 1e-4, at the edge of fp16's normal range), so the parity would measure fp16 rounding rather than
    the kernels; at He's std (times sqrt(6)) they grow about 4x per cell, since every combination adds two branches.  Measured on
    the reference at seed 0 with a unit-normal 331^2 input, times 1.7 keeps every stage's std between 0.7 and 1.4 (conv_0: 1.1);
    oracle/make_golden_pnasnet.py asserts each stage within 10x of conv_0's and prints them."""
    with torch.no_grad():
        for m in model.modules():
            if isinstance(m, nn.Conv2d):
                m.weight.mul_(factor)
    return model


def _bn(x, sd, p):
    return F.batch_norm(x, sd[p + 'running_mean'], sd[p + 'running_var'], sd[p + 'weight'], sd[p + 'bias'], False, 0.0, BN_EPS)


def _pool(x, stride, zero_pad):
    if zero_pad:
        return F.max_pool2d(F.pad(x, (1, 0, 1, 0)), 3, stride, 1)[:, :, 1:, 1:]
    return F.max_pool2d(x, 3, stride, 1)


def branch(x, sd, p, stride, zero_pad):
    """BranchSeparables ``p`` (with the trailing dot)."""
    w1 = sd[p + 'separable_1.depthwise_conv2d.weight']
    k = w1.shape[-1]
    x = F.relu(x)
    if zero_pad:
        x = F.pad(x, (1, 0, 1, 0))
    x = F.conv2d(x, w1, None, stride, k // 2, 1, x.shape[1])
    x = F.conv2d(x, sd[p + 'separable_1.pointwise_conv2d.weight'])
    if zero_pad:
        x = x[:, :, 1:, 1:].contiguous()
    x = F.relu(_bn(x, sd, p + 'bn_sep_1.'))
    x = F.conv2d(x, sd[p + 'separable_2.depthwise_conv2d.weight'], None, 1, k // 2, 1, x.shape[1])
    x = F.conv2d(x, sd[p + 'separable_2.pointwise_conv2d.weight'])
    return _bn(x, sd, p + 'bn_sep_2.')


def relu_conv_bn(x, sd, p, stride=1):
    return _bn(F.conv2d(F.relu(x), sd[p + 'conv.weight'], stride=stride), sd, p + 'bn.')


def factorized_reduction(x, sd, p):
    x = F.relu(x)
    x1 = F.conv2d(F.avg_pool2d(x, 1, 2, count_include_pad=False), sd[p + 'path_1.conv.weight'])
    x2 = F.pad(x, (0, 1, 0, 1))[:, :, 1:, 1:]
    x2 = F.conv2d(F.avg_pool2d(x2, 1, 2, count_include_pad=False), sd[p + 'path_2.conv.weight'])
    return _bn(torch.cat([x1, x2], 1), sd, p + 'final_path_bn.')


def cell(name, x_left, x_right, sd):
    """One cell; ``x_right`` is None for cell_stem_0 (its right input is conv_1x1 of the left)."""
    p = name + '.'
    stem0 = name == 'cell_stem_0'
    s = 2 if stem0 or name in REDUCTION else 1
    zp = name in ZERO_PAD
    if stem0:
        x_right = relu_conv_bn(x_left, sd, p + 'conv_1x1.')
    else:
        x_left = (factorized_reduction(x_left, sd, p + 'conv_prev_1x1.') if name in FACTORIZED
                  else relu_conv_bn(x_left, sd, p + 'conv_prev_1x1.'))
        x_right = relu_conv_bn(x_right, sd, p + 'conv_1x1.')
    c0l = branch(x_left, sd, p + 'comb_iter_0_left.', s, zp)
    if stem0:
        c0r = _bn(F.conv2d(_pool(x_left, 2, False), sd[p + 'comb_iter_0_right.conv.weight']), sd, p + 'comb_iter_0_right.bn.')
    else:
        c0r = _pool(x_left, s, zp)
    c0 = c0l + c0r
    c1 = branch(x_right, sd, p + 'comb_iter_1_left.', s, zp) + _pool(x_right, s, zp)
    c2 = branch(x_right, sd, p + 'comb_iter_2_left.', s, zp) + branch(x_right, sd, p + 'comb_iter_2_right.', s, zp)
    c3 = branch(c2, sd, p + 'comb_iter_3_left.', 1, False) + _pool(x_right, s, zp)
    c4l = branch(x_left, sd, p + 'comb_iter_4_left.', s, zp)
    c4r = relu_conv_bn(x_right, sd, p + 'comb_iter_4_right.', 2) if (p + 'comb_iter_4_right.conv.weight') in sd else x_right
    return torch.cat([c0, c1, c2, c3, c4l + c4r], 1)


def features(x, sd, stages=None):
    """conv_0 .. cell_11: cell_11's output.  ``stages``: optional dict that receives every stage's output."""
    x0 = _bn(F.conv2d(x, sd['conv_0.conv.weight'], stride=2), sd, 'conv_0.bn.')
    outs = [x0, cell('cell_stem_0', x0, None, sd)]
    for name in STAGES[2:]:
        outs.append(cell(name, outs[-2], outs[-1], sd))
    if stages is not None:
        stages.update(zip(STAGES, outs))
    return outs[-1]


def logits(f, sd):
    x = F.avg_pool2d(F.relu(f), 11, 1, 0).view(f.size(0), -1)
    return F.linear(x, sd['last_linear.weight'], sd['last_linear.bias'])


def forward(x, sd):
    return logits(features(x, sd), sd)


def build_package_model(pkg, fx):
    """The package-under-test's model for a ``kind == 'pnasnet'`` / ``'trn_pnasnet'`` fixture: same constructor call, seeds and
    rescaling as oracle/make_golden_pnasnet.py applied to the reference."""
    from oracle import functional as OF
    torch.manual_seed(fx["seeds"]["init"])
    if fx["kind"] == "trn_pnasnet":
        m = pkg.TRN(10, num_segments=fx["segments"], arch="pnasnet5large", consensus="MSTRN", pretrained=None, **fx["kwargs"])
    else:
        m = pkg.pnasnet5large(pretrained=None, **fx["kwargs"])
    rescale_(m)
    OF.randomize_bn_(m, fx["seeds"]["bn"])
    return m.eval()
