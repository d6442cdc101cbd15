"""H100-native drop-ins for `models.NonlocalNet.VGG19_pytorch` and `models.NonlocalNet.WarpNet`.

Same constructor / forward signatures and state_dict keys as the reference
(the reference's models/NonlocalNet.py:192-256 and 355-502) so that the reference's test.py and
models/FrameColor.py run unchanged with this directory ahead of the reference on sys.path.  The
forward passes call hand-written sm_90a kernels in libdvc.so through ctypes (dvc/__init__.py);
there is no torch fallback and no CPU path.
"""
import torch
import torch.nn as nn

import dvc
from models._params import ConvParams, SlopeParam, indexed

_VGG_CFG = [("conv1_1", 3, 64), ("conv1_2", 64, 64), ("conv2_1", 64, 128), ("conv2_2", 128, 128),
            ("conv3_1", 128, 256), ("conv3_2", 256, 256), ("conv3_3", 256, 256), ("conv3_4", 256, 256),
            ("conv4_1", 256, 512), ("conv4_2", 512, 512), ("conv4_3", 512, 512), ("conv4_4", 512, 512),
            ("conv5_1", 512, 512), ("conv5_2", 512, 512), ("conv5_3", 512, 512), ("conv5_4", 512, 512)]


_COMPARE = __import__("os").environ.get("DVC_DROPIN_COMPARE", "1") != "0"


def _ctx_for(t):
    if not t.is_cuda:
        raise dvc.DvcError("the H100 drop-in modules run on CUDA tensors only (no CPU fallback); call .cuda() like test.py:164-166")
    return dvc.get_context(t.device.index)


class VGG19_pytorch(nn.Module):
    """NonlocalNet.py:192-256.  Input RGB in [0,1]; returns the requested ReLU / pool maps (NCHW fp32)."""

    def __init__(self, pool="max"):
        super().__init__()
        if pool != "max":
            raise NotImplementedError("pool='avg' is not used by the inference path (NonlocalNet.py:221-226)")
        for name, cin, cout in _VGG_CFG:
            setattr(self, name, ConvParams(cin, cout))

    def forward(self, x, out_keys, preprocess=True):
        ctx = _ctx_for(x)
        ctx.sync_module_weights(dvc.NET_VGG, self)
        return ctx.vgg19_forward(x, list(out_keys), preprocess)


def _head(c_in, c_mid, second):
    # indices follow the reference's nn.Sequential numbering (pad, conv, norm, prelu, [up], pad, conv, norm, prelu)
    return indexed({1: ConvParams(c_in, c_mid), 3: SlopeParam(), second: ConvParams(c_mid, 64), second + 2: SlopeParam()})


class _ResidualParams(nn.Module):
    def __init__(self):
        super().__init__()
        self.conv1 = ConvParams(256, 256)
        self.prelu = SlopeParam()
        self.conv2 = ConvParams(256, 256)


class WarpNet(nn.Module):
    """NonlocalNet.py:355-502: feature heads, residual blocks, theta/phi, dense correlation, softmax, warp."""

    def __init__(self, batch_size):
        super().__init__()
        self.feature_channel = 64
        self.in_channels = 256
        self.inter_channels = 256
        self.layer2_1 = _head(128, 128, 5)
        self.layer3_1 = _head(256, 128, 5)
        self.layer4_1 = _head(512, 256, 5)
        self.layer5_1 = _head(512, 256, 6)
        self.layer = indexed({i: _ResidualParams() for i in range(3)})
        self.theta = ConvParams(256, 256, k=1)
        self.phi = ConvParams(256, 256, k=1)
        self._b_cache = None

    def forward(self, B_lab_map, A_relu2_1, A_relu3_1, A_relu4_1, A_relu5_1, B_relu2_1, B_relu3_1, B_relu4_1,
                B_relu5_1, temperature=0.001 * 5, detach_flag=False, WTA_scale_weight=1, feature_noise=0):
        ctx = _ctx_for(B_lab_map)
        before = ctx._weight_sig.get(dvc.NET_WARP)
        ctx.sync_module_weights(dvc.NET_WARP, self)
        weights_changed = before != ctx._weight_sig.get(dvc.NET_WARP)
        b_inputs = [B_lab_map, B_relu2_1, B_relu3_1, B_relu4_1, B_relu5_1]
        # The reference recomputes the exemplar side every frame (FrameColor.py:20-36).  Every B-side op is
        # per-sample, so when the B tensors are the tensors of the previous call the cached phi / pooled Lab operands
        # give the identical result.  Two checks, cheapest first:
        #  (1) identity: same storage, same version counter, same shape -- no device work, no sync.  The previous
        #      call's tensors are kept referenced, so a NEW tensor can never alias their (recycled) address;
        #  (2) content: FrameColor.py:33-36 re-normalises the exemplar features every frame into fresh tensors, so
        #      (1) misses there; one fused device comparison + one host sync per call decides (DVC_DROPIN_COMPARE=0
        #      turns it off: the B side is then simply recomputed like the reference does).
        reuse = False
        if self._b_cache is not None and not weights_changed and not torch.is_grad_enabled():
            prev_keys, prev = self._b_cache
            keys = [(t.data_ptr(), t._version, tuple(t.shape), t.device) for t in b_inputs]
            if keys == prev_keys:
                reuse = True
            elif (_COMPARE and all(p.shape == t.shape and p.device == t.device for p, t in zip(prev, b_inputs))
                  and all(p._version == k[1] for p, k in zip(prev, prev_keys))):  # the kept tensors are still what was cached
                diff = torch.stack([(p != t).any() for p, t in zip(prev, b_inputs)]).any()
                reuse = not bool(diff.item())
        y, sim = ctx.warpnet_forward(B_lab_map, [A_relu2_1, A_relu3_1, A_relu4_1, A_relu5_1],
                                     [B_relu2_1, B_relu3_1, B_relu4_1, B_relu5_1], temperature, WTA_scale_weight, reuse)
        # keep the caller's tensors referenced (identity check) -- no clone: an in-place edit bumps _version
        self._b_cache = ([(t.data_ptr(), t._version, tuple(t.shape), t.device) for t in b_inputs], [t.detach() for t in b_inputs])
        return y, sim
