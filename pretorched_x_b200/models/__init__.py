from . import (resnet3d, r2plus1d, nonlocalnet, resnet2d, resnext3d, trn, slowfast, mobilenet, senet, bninception,  # noqa: F401
               inception, densenet, inceptionv3, polynet, vgg, resnext, xception, pnasnet,
               utils, settings)

# the reference spells the module `resnet3D` (capital D); keep that import path working
resnet3D = resnet3d
resnext3D = resnext3d
