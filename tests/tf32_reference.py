"""The reference as it runs on a GPU, emulated on the fp64 CPU oracle: PyTorch lets cuDNN run fp32 convolutions on TF32
operands (torch.backends.cudnn.allow_tf32 defaults to True) while matmuls, and so the correlation, stay fp32.

    with tf32_conv_operands():
        ab, ... = O.frame_colorization(sds64, ...)   # every convolution's input and weight rounded to 11 bits

The oracle itself is left as it is: inside the block its module-level `F` is replaced by a view of
torch.nn.functional whose conv2d rounds both operands (not the bias) before the exact convolution.
"""
import contextlib

import torch
import torch.nn.functional as F

from oracle import dvc_oracle as O


def round_tf32(t):
    """t rounded to 11 significant bits (TF32's 10 explicit mantissa bits), nearest, ties to even; any float dtype."""
    m, e = torch.frexp(t)  # t = m * 2^e, 0.5 <= |m| < 1
    return torch.ldexp(torch.round(torch.ldexp(m, torch.full_like(e, 11))), e - 11).to(t.dtype)


class _RoundedConvFunctional:
    """torch.nn.functional, except that conv2d sees TF32-rounded operands."""

    def __getattr__(self, name):
        return getattr(F, name)

    @staticmethod
    def conv2d(x, w, bias=None, *args, **kw):
        return F.conv2d(round_tf32(x), round_tf32(w), bias, *args, **kw)


@contextlib.contextmanager
def tf32_conv_operands():
    saved = O.F
    O.F = _RoundedConvFunctional()
    try:
        yield
    finally:
        O.F = saved
