"""Registry of per-model preprocessing / checkpoint settings (reference: pretorched/models/settings.py:20-44),
restricted to the model families this engine implements."""
from .resnet3d import pretrained_settings as resnet3d_settings
from .nonlocalnet import pretrained_settings as nonlocal_settings
from .resnet2d import pretrained_settings as resnet2d_settings
from .resnext3d import pretrained_settings as resnext3d_settings      # settings.py:18,36 of the reference
from .mobilenet import pretrained_settings as mobilenet_settings      # mobilenet.py:7-19 (not in the reference's registry)
from .senet import pretrained_settings as senet_settings              # senet.py:15-82 (not in the reference's registry)
from .bninception import pretrained_settings as bninception_settings  # bninception.py:10-25 (settings.py:3 of the reference)
from .inception import pretrained_settings as inception_settings      # inceptionv4.py:10-31, inceptionresnetv2.py:10-31
from .densenet import pretrained_settings as densenet_settings        # torchvision_models.py:80-130
from .inceptionv3 import pretrained_settings as inceptionv3_settings  # torchvision_models.py:39, 74-92
from .polynet import pretrained_settings as polynet_settings          # polynet.py:8-21 (settings.py:15 of the reference)
from .vgg import pretrained_settings as vgg_settings                  # torchvision_models.py:64-119
from .resnext import pretrained_settings as resnext_settings          # resnext.py:12-35 (settings.py:4,23 of the reference)
from .xception import pretrained_settings as xception_settings      # xception.py:33-47
from .pnasnet import pretrained_settings as pnasnet_settings        # pnasnet.py:9-30

all_settings = [resnet2d_settings, resnet3d_settings, resnext3d_settings, nonlocal_settings, mobilenet_settings, senet_settings,
                bninception_settings, inception_settings, densenet_settings, inceptionv3_settings, polynet_settings,
                vgg_settings, resnext_settings, xception_settings, pnasnet_settings]

model_names = []
pretrained_settings = {}
for _settings in all_settings:
    for _name, _rows in _settings.items():
        pretrained_settings[_name] = _rows
        model_names.append(_name)
