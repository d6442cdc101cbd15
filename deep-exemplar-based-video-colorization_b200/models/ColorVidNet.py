"""H100-native drop-in for `models.ColorVidNet.ColorVidNet` (the reference's models/ColorVidNet.py:6-144).

Same constructor / forward signature and the same 65 state_dict keys; forward() runs the 34-conv
encoder-decoder (InstanceNorm x9, dilated middle, three skip adds, tanh*128) in libdvc.so.
"""
import torch.nn as nn

import dvc
from models._params import ConvParams, indexed


class ColorVidNet(nn.Module):
    def __init__(self, ic):
        super().__init__()
        if ic != 7:
            raise NotImplementedError("the inference path feeds 7 channels (FrameColor.py:64)")
        self.conv1_1 = indexed({0: ConvParams(ic, 32), 2: ConvParams(32, 64)})
        self.conv1_2 = ConvParams(64, 64)
        self.conv1_2norm_ss = ConvParams(64, 64, k=1, bias=False, groups=64)
        self.conv2_1 = ConvParams(64, 128)
        self.conv2_2 = ConvParams(128, 128)
        self.conv2_2norm_ss = ConvParams(128, 128, k=1, bias=False, groups=128)
        self.conv3_1 = ConvParams(128, 256)
        self.conv3_2 = ConvParams(256, 256)
        self.conv3_3 = ConvParams(256, 256)
        self.conv3_3norm_ss = ConvParams(256, 256, k=1, bias=False, groups=256)
        self.conv4_1 = ConvParams(256, 512)
        for n in ("conv4_2", "conv4_3", "conv5_1", "conv5_2", "conv5_3", "conv6_1", "conv6_2", "conv6_3", "conv7_1",
                  "conv7_2", "conv7_3"):
            setattr(self, n, ConvParams(512, 512))
        self.conv8_1 = indexed({1: ConvParams(512, 256)})
        self.conv3_3_short = ConvParams(256, 256)
        self.conv8_2 = ConvParams(256, 256)
        self.conv8_3 = ConvParams(256, 256)
        self.conv9_1 = indexed({1: ConvParams(256, 128)})
        self.conv2_2_short = ConvParams(128, 128)
        self.conv9_2 = ConvParams(128, 128)
        self.conv10_1 = indexed({1: ConvParams(128, 128)})
        self.conv1_2_short = ConvParams(64, 128)
        self.conv10_2 = ConvParams(128, 128)
        self.conv10_ab = ConvParams(128, 2, k=1)
        print("replace all deconv with [nearest + conv]")      # ColorVidNet.py:80
        print("replace all batchnorm with instancenorm")       # ColorVidNet.py:85

    def forward(self, x):
        if not x.is_cuda:
            raise dvc.DvcError("the H100 drop-in modules run on CUDA tensors only (no CPU fallback)")
        ctx = dvc.get_context(x.device.index)
        ctx.sync_module_weights(dvc.NET_COLOR, self)
        return ctx.colorvidnet_forward(x)
