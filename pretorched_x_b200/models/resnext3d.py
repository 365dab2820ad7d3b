"""ResNeXt-3D family behind the reference's factory API (reference: pretorched/models/resnext3D.py, exported by
pretorched/__init__.py:66-72).

``ResNeXtBottleneck`` (resnext3D.py:78-122) is a 3-D bottleneck whose middle 3x3x3 convolution is *grouped*
(``groups = cardinality = 32``), with widths 128 / 256 / 512 / 1024, expansion 2 and an ``fc`` head (the reference never
runs ``modify_resnets`` on this family, so there is no ``last_linear`` in its ``state_dict``).  The containers below create
the reference's tensors in the reference's order (seeded init is bit-identical, checkpoints such as
``resnext3d101_kinetics-8e57b772.pth`` load unchanged); the block body is ``engine.run_bottleneck``.

Grouped convolution on the tensor cores: a group is 4..32 channels wide -- far below one MMA tile -- but a 64-channel slice
holds whole groups and reads only its own 64 input channels.  ``conv2`` runs the slab convolution per slice with the filter
packed as its diagonal 16 x 16 (32 x 32) blocks, each K step of a tap accumulating into its own 16 (32) output columns
(``ops.PackedGroupedConv``, csrc/b2_groupconv.cuh): 4x / 2x / 1x / 1x the grouped multiply-accumulates for 4 / 8 / 16 / 32
channels per group, and ``C * 16 * 27`` (``C * 32 * 27``) filter elements.  A grouped convolution outside that kernel's
contract is packed as the block-diagonal DENSE filter (``ops.dense_from_grouped``): same result at ``groups`` times the work.
Like R(2+1)D the class additionally offers ``features / logits / last_linear`` (alias of ``fc``).  Upstream quirk kept: ``fc``
is sized ``cardinality * 32 * expansion`` (resnext3D.py:139) while the trunk always ends with 2048 channels, so only the
default ``cardinality=32`` yields a network whose forward works -- here as there.
"""
from collections import defaultdict

import torch.nn as nn

from . import resnet3d
from .resnet3d import EngineModule, ResNet3D, ShortcutA
from .. import engine

__all__ = ['ResNeXt3D', 'resnext3d10', 'resnext3d18', 'resnext3d34', 'resnext3d50', 'resnext3d101', 'resnext3d152',
           'resnext3d200']

# registry rows in the reference's schema (resnext3D.py:16-50): only resnext3d101 has a published checkpoint
pretrained_settings = resnet3d._make_settings(
    [n for n in __all__ if n != 'ResNeXt3D'],
    {'kinetics-400': defaultdict(lambda: None, {'resnext3d101': 'resnext3d101_kinetics-8e57b772.pth'})})


class ResNeXtBottleneck(EngineModule):
    expansion = 2

    def __init__(self, inplanes, planes, cardinality, stride=1, downsample=None):
        super().__init__()
        mid_planes = cardinality * int(planes / 32)
        self.conv1 = nn.Conv3d(inplanes, mid_planes, kernel_size=1, bias=False)
        self.bn1 = nn.BatchNorm3d(mid_planes)
        self.conv2 = nn.Conv3d(mid_planes, mid_planes, kernel_size=3, stride=stride, padding=1, groups=cardinality, bias=False)
        self.bn2 = nn.BatchNorm3d(mid_planes)
        self.conv3 = nn.Conv3d(mid_planes, planes * self.expansion, kernel_size=1, bias=False)
        self.bn3 = nn.BatchNorm3d(planes * self.expansion)
        self.relu = nn.ReLU(inplace=True)
        self.downsample = downsample
        self.stride = stride

    def _run(self, a):
        return engine.run_bottleneck(self, a)


class ResNeXt3D(ResNet3D):
    head_name = 'fc'

    def __init__(self, block, layers, shortcut_type='B', cardinality=32, num_classes=400):
        nn.Module.__init__(self)
        self.inplanes = 64
        self.conv1 = nn.Conv3d(3, 64, kernel_size=7, stride=(1, 2, 2), padding=(3, 3, 3), bias=False)
        self.bn1 = nn.BatchNorm3d(64)
        self.relu = nn.ReLU(inplace=True)
        self.maxpool = nn.MaxPool3d(kernel_size=(3, 3, 3), stride=2, padding=1)
        self.layer1 = self._make_layer(block, 128, layers[0], shortcut_type, cardinality)
        self.layer2 = self._make_layer(block, 256, layers[1], shortcut_type, cardinality, stride=2)
        self.layer3 = self._make_layer(block, 512, layers[2], shortcut_type, cardinality, stride=2)
        self.layer4 = self._make_layer(block, 1024, layers[3], shortcut_type, cardinality, stride=2)
        self.avgpool = nn.AdaptiveAvgPool3d(1)
        self.fc = nn.Linear(cardinality * 32 * block.expansion, num_classes)
        self.init_weights()
        self._register_load_state_dict_pre_hook(self._accept_zoo_head_keys)

    def _make_layer(self, block, planes, blocks, shortcut_type, cardinality, stride=1):
        out_planes = planes * block.expansion
        downsample = None
        if stride != 1 or self.inplanes != out_planes:
            if shortcut_type == 'A':
                downsample = ShortcutA(out_planes, stride)
            else:
                downsample = nn.Sequential(nn.Conv3d(self.inplanes, out_planes, kernel_size=1, stride=stride, bias=False),
                                           nn.BatchNorm3d(out_planes))
        seq = [block(self.inplanes, planes, cardinality, stride, downsample)]
        self.inplanes = out_planes
        seq += [block(self.inplanes, planes, cardinality) for _ in range(1, blocks)]
        return nn.Sequential(*seq)

    @property
    def last_linear(self):
        return self.fc

    def __setattr__(self, name, value):
        # nn.Module.__setattr__ would register a second module called `last_linear`; keep one head: `fc`
        super().__setattr__('fc' if name == 'last_linear' else name, value)


def resnext3d10(**kwargs):
    return ResNeXt3D(ResNeXtBottleneck, [1, 1, 1, 1], **kwargs)


def resnext3d18(**kwargs):
    return ResNeXt3D(ResNeXtBottleneck, [2, 2, 2, 2], **kwargs)


def resnext3d34(**kwargs):
    return ResNeXt3D(ResNeXtBottleneck, [3, 4, 6, 3], **kwargs)


def resnext3d50(**kwargs):
    return ResNeXt3D(ResNeXtBottleneck, [3, 4, 6, 3], **kwargs)


def resnext3d101(**kwargs):
    return ResNeXt3D(ResNeXtBottleneck, [3, 4, 23, 3], **kwargs)


def resnext3d152(**kwargs):
    return ResNeXt3D(ResNeXtBottleneck, [3, 8, 36, 3], **kwargs)


def resnext3d200(**kwargs):
    return ResNeXt3D(ResNeXtBottleneck, [3, 24, 36, 3], **kwargs)
