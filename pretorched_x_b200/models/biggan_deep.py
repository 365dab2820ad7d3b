"""BigGAN-deep generator on the H100 engine (BASELINE.json configs[4]; SURVEY.md section 8a row a14 / 8f row n1).

The reference tree has **no GAN code** (nothing to be a drop-in for), so the boundary kept here is the one the public
BigGAN-deep implementation established and that published checkpoints use: a ``Generator`` whose ``state_dict`` has

    shared.weight [n_classes, 128]
    linear.{weight [16ch*16, 256], bias, u0, sv0}
    blocks.{i}.{0,1}.conv{1..4}.{weight, bias, u0, sv0}           GBlock: 1x1 (in -> in/4), 3x3, 3x3, 1x1 (in/4 -> out)
    blocks.{i}.{0,1}.bn{1..4}.{gain,bias}.{weight [C, 256], u0, sv0}, bn{1..4}.{stored_mean, stored_var}
    blocks.{i}.2.{theta,phi,g,o}.{weight, u0, sv0}, blocks.{i}.2.gamma     (self-attention after the 64x64 stage)
    output_layer.0.{gain, bias, stored_mean, stored_var}, output_layer.2.{weight [3, ch, 3, 3], bias, u0, sv0}

and whose ``forward(z, y)`` takes z fp32 ``[B, dim_z]`` and either class indices (int64 ``[B]``) or an already embedded
``[B, shared_dim]`` tensor.  The modules below are *parameter containers* only (like every other model in this
package); the arithmetic is ``pretorched_x_b200/biggan_engine.py`` on hand-written sm_90a kernels.  Evaluation mode
only: BatchNorm uses ``stored_mean/var`` (standing statistics), spectral norm divides by the sigma obtained from one
power-iteration step off the stored ``u0`` (no update).
"""
import torch
import torch.nn as nn

from .. import engine as _engine

__all__ = ['Generator', 'biggan_deep', 'biggan_deep128', 'biggan_deep256', 'biggan_deep512', 'G_ARCH']

# resolution -> (in multipliers, out multipliers, resolutions with attention); channels = multiplier * ch
G_ARCH = {
    512: ([16, 16, 8, 8, 4, 2, 1], [16, 8, 8, 4, 2, 1, 1], (64,)),
    256: ([16, 16, 8, 8, 4, 2], [16, 8, 8, 4, 2, 1], (64,)),
    128: ([16, 16, 8, 4, 2], [16, 8, 4, 2, 1], (64,)),
    64: ([16, 16, 8, 4], [16, 8, 4, 2], (64,)),
    32: ([4, 4, 4], [4, 4, 4], ()),
}


class _SNMixin:
    """Registers the spectral-norm buffers (left singular vector estimate u0 [1, out], its sigma sv0 [1])."""

    def _sn_init(self, num_outputs):
        self.register_buffer('u0', torch.randn(1, num_outputs))
        self.register_buffer('sv0', torch.ones(1))


class SNConv2d(nn.Conv2d, _SNMixin):
    def __init__(self, in_channels, out_channels, kernel_size=3, padding=1, bias=True):
        nn.Conv2d.__init__(self, in_channels, out_channels, kernel_size, 1, padding, bias=bias)
        self._sn_init(out_channels)

    def forward(self, x):
        raise RuntimeError("parameter container: the convolution runs inside biggan_engine (no torch fallback)")


class SNLinear(nn.Linear, _SNMixin):
    def __init__(self, in_features, out_features, bias=True):
        nn.Linear.__init__(self, in_features, out_features, bias)
        self._sn_init(out_features)

    def forward(self, x):
        raise RuntimeError("parameter container: the layer runs inside biggan_engine (no torch fallback)")


class ccbn(nn.Module):
    """Class-conditional BatchNorm: BN(x; stored stats) * (1 + gain(y)) + bias(y)."""

    def __init__(self, output_size, input_size, eps=1e-5):
        super().__init__()
        self.output_size, self.input_size, self.eps = output_size, input_size, eps
        self.gain = SNLinear(input_size, output_size, bias=False)
        self.bias = SNLinear(input_size, output_size, bias=False)
        self.register_buffer('stored_mean', torch.zeros(output_size))
        self.register_buffer('stored_var', torch.ones(output_size))


class bn(nn.Module):
    """Plain BatchNorm with learned gain / bias and stored statistics (output layer)."""

    def __init__(self, output_size, eps=1e-5):
        super().__init__()
        self.output_size, self.eps = output_size, eps
        self.gain = nn.Parameter(torch.ones(output_size))
        self.bias = nn.Parameter(torch.zeros(output_size))
        self.register_buffer('stored_mean', torch.zeros(output_size))
        self.register_buffer('stored_var', torch.ones(output_size))


class GBlock(nn.Module):
    def __init__(self, in_channels, out_channels, cond_dim, upsample, channel_ratio=4, eps=1e-5):
        super().__init__()
        self.in_channels, self.out_channels = in_channels, out_channels
        self.hidden_channels = in_channels // channel_ratio
        self.upsample = bool(upsample)
        h = self.hidden_channels
        self.conv1 = SNConv2d(in_channels, h, kernel_size=1, padding=0)
        self.conv2 = SNConv2d(h, h)
        self.conv3 = SNConv2d(h, h)
        self.conv4 = SNConv2d(h, out_channels, kernel_size=1, padding=0)
        self.bn1 = ccbn(in_channels, cond_dim, eps)
        self.bn2 = ccbn(h, cond_dim, eps)
        self.bn3 = ccbn(h, cond_dim, eps)
        self.bn4 = ccbn(h, cond_dim, eps)


class Attention(nn.Module):
    def __init__(self, ch):
        super().__init__()
        self.ch = ch
        self.theta = SNConv2d(ch, ch // 8, kernel_size=1, padding=0, bias=False)
        self.phi = SNConv2d(ch, ch // 8, kernel_size=1, padding=0, bias=False)
        self.g = SNConv2d(ch, ch // 2, kernel_size=1, padding=0, bias=False)
        self.o = SNConv2d(ch // 2, ch, kernel_size=1, padding=0, bias=False)
        self.gamma = nn.Parameter(torch.tensor(0.))


class Generator(_engine.CacheOwner, nn.Module):
    def __init__(self, G_ch=128, dim_z=128, bottom_width=4, resolution=256, n_classes=1000, shared_dim=128,
                 G_attn='64', BN_eps=1e-5, SN_eps=1e-12, G_init='ortho', hier=True, **unused):
        super().__init__()
        if not hier:
            raise NotImplementedError("BigGAN-deep feeds [embedding | z] to every block (hier=True)")
        self.ch, self.dim_z, self.bottom_width, self.resolution = G_ch, dim_z, bottom_width, resolution
        self.n_classes, self.shared_dim, self.BN_eps, self.SN_eps, self.init = n_classes, shared_dim, BN_eps, SN_eps, G_init
        ins, outs, _ = G_ARCH[resolution]
        att_res = tuple(int(r) for r in G_attn.split('_')) if G_attn and G_attn != '0' else ()
        self.arch = {'in_channels': [G_ch * i for i in ins], 'out_channels': [G_ch * o for o in outs],
                     'resolution': [8 << k for k in range(len(ins))],
                     'attention': {8 << k: (8 << k) in att_res for k in range(len(ins))}}
        cond = dim_z + shared_dim
        self.shared = nn.Embedding(n_classes, shared_dim)
        self.linear = SNLinear(cond, self.arch['in_channels'][0] * bottom_width ** 2)
        blocks = []
        for i, (cin, cout) in enumerate(zip(self.arch['in_channels'], self.arch['out_channels'])):
            stage = [GBlock(cin, cin, cond, False, eps=BN_eps), GBlock(cin, cout, cond, True, eps=BN_eps)]
            if self.arch['attention'][self.arch['resolution'][i]]:
                stage.append(Attention(cout))
            blocks.append(nn.ModuleList(stage))
        self.blocks = nn.ModuleList(blocks)
        self.output_layer = nn.Sequential(bn(self.arch['out_channels'][-1], BN_eps), nn.ReLU(),
                                          SNConv2d(self.arch['out_channels'][-1], 3))
        self.input_space, self.input_range = 'RGB', [-1, 1]
        self.init_weights()

    def init_weights(self):
        for m in self.modules():
            if isinstance(m, (nn.Conv2d, nn.Linear, nn.Embedding)):
                if self.init == 'ortho':
                    nn.init.orthogonal_(m.weight)
                elif self.init == 'N02':
                    nn.init.normal_(m.weight, 0, 0.02)
                elif self.init in ('glorot', 'xavier'):
                    nn.init.xavier_uniform_(m.weight)
                else:
                    raise ValueError("unknown init %r" % (self.init,))

    def forward(self, z, y, out_dtype=torch.float32):
        """z: fp32 [B, dim_z]; y: int64 class indices [B] (or an embedded [B, shared_dim] tensor).
        Returns images [B, 3, R, R] in (-1, 1), NCHW, ``out_dtype`` (fp32 like the public model, or fp16)."""
        from .. import biggan_engine
        return biggan_engine.generator_forward(self, z, y, out_dtype=out_dtype)


def biggan_deep(resolution=256, pretrained=None, **kwargs):
    if pretrained is not None:
        raise RuntimeError("no network in this environment: load a checkpoint with load_state_dict() instead")
    return Generator(resolution=resolution, **kwargs).eval()


def biggan_deep128(**kw):
    return biggan_deep(128, **kw)


def biggan_deep256(**kw):
    return biggan_deep(256, **kw)


def biggan_deep512(**kw):
    return biggan_deep(512, **kw)
