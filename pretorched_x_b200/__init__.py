"""pretorched_x_b200 -- H100-native forward engine for pretorched-x's video-ConvNet hot path.

Drop-in for the reference's factory API: ``pretorched_x_b200.__dict__[name](num_classes=..., pretrained=...)``
returns a module with ``features / logits / forward / last_linear`` and the reference's ``state_dict`` layout
(reference: pretorched/__init__.py:11-83).  The block bodies are hand-written sm_90a kernels reached through
the C ABI in ``include/b2_pretorched.h``; there is no CPU or library fallback.
"""
from .__version__ import __version__  # noqa: F401

from . import models  # noqa: F401
from .models.settings import pretrained_settings, model_names  # noqa: F401

from .models.resnet2d import resnet18, resnet34, resnet50, resnet101, resnet152  # noqa: F401
from .models.resnet3d import (resnet3d10, resnet3d18, resnet3d34, resnet3d50, resnet3d101,  # noqa: F401
                              resnet3d152, resnet3d200, resneti3d50)
from .models.nonlocalnet import (nonlocalresnet3d18, nonlocalresnet3d34, nonlocalresnet3d50,  # noqa: F401
                                 nonlocalresnet3d101)
# not exported by the reference's __init__ (r2plus1d.py / trn.py are import-broken upstream); offered here
from .models.r2plus1d import (r2plus1d10, r2plus1d18, r2plus1d34, r2plus1d50, r2plus1d101,  # noqa: F401
                              r2plus1d152, r2plus1d200)
from .models.pre_act_resnet3d import (preact_resnet3d10, preact_resnet3d18, preact_resnet3d34, preact_resnet3d50,  # noqa: F401
                                      preact_resnet3d101, preact_resnet3d152, preact_resnet3d200)   # pre_act_resnet3D.py:100-139
from .models.resnext3d import (resnext3d10, resnext3d18, resnext3d34, resnext3d50, resnext3d101,  # noqa: F401
                               resnext3d152, resnext3d200)          # pretorched/__init__.py:66-72
from .models.trn import Relation, MultiScaleRelation, HierarchicalRelation, TRN, trn  # noqa: F401
from .models.utils import Identity  # noqa: F401
# BigGAN-deep generator (BASELINE.json configs[4]; not in the reference tree -- see models/biggan_deep.py)
from .models.biggan_deep import biggan_deep, biggan_deep128, biggan_deep256, biggan_deep512  # noqa: F401
from .models import slowfast  # noqa: F401  (module, as in pretorched/__init__.py:83)
