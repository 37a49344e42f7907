"""Conv1d / Conv2d / Conv3d / Deconv3d + BN + ReLU containers (reference nn/conv.py:7-81, 176-216, and its
Deconv3d).  Parameter names
(``conv.weight``, ``bn.*``) match the reference so its checkpoints load unchanged; inside
PointFlow the arithmetic is done by the fused sm_90a kernels, this forward is the
stock-library path for stand-alone use."""
import torch.nn.functional as F
from torch import nn

from .init import init_bn, init_uniform


class Conv1d(nn.Module):
    """1-D convolution, then (optionally) train-mode-aware BatchNorm1d and ReLU.

    With ``bn=True`` the convolution has no bias (the BN shift replaces it), as in the reference."""

    def __init__(self, in_channels, out_channels, kernel_size, relu=True, bn=True, bn_momentum=0.1, **kwargs):
        super().__init__()
        self.relu = bool(relu)
        self.conv = nn.Conv1d(in_channels, out_channels, kernel_size, bias=not bn, **kwargs)
        init_uniform(self.conv)
        self.bn = None
        if bn:
            self.bn = nn.BatchNorm1d(out_channels, momentum=bn_momentum)
            init_bn(self.bn)

    def init_weights(self):
        """Re-draw the parameters (Xavier-uniform weights, BN affine = (1, 0))."""
        for module, init in ((self.conv, init_uniform), (self.bn, init_bn)):
            if module is not None:
                init(module)

    def forward(self, x):
        y = self.conv(x)
        if self.bn is not None:
            y = self.bn(y)
        return F.relu(y) if self.relu else y


class Conv2d(nn.Module):
    """2-D convolution + BatchNorm2d + ReLU with the reference's submodule names (nn/conv.py:43-81).  Only the
    pyramid producer (``networks.ImageConv``, SURVEY.md 8 row f1) uses it; the arithmetic is the stock library's,
    run in whatever memory format the input arrives in (channels-last in, channels-last out)."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, relu=True, bn=True, bn_momentum=0.1, **kwargs):
        super().__init__()
        self.kernel_size, self.stride, self.relu = kernel_size, stride, bool(relu)
        self.conv = nn.Conv2d(in_channels, out_channels, kernel_size, stride=stride, bias=not bn, **kwargs)
        self.bn = nn.BatchNorm2d(out_channels, momentum=bn_momentum) if bn else None
        self.init_weights()

    def init_weights(self):
        init_uniform(self.conv)
        if self.bn is not None:
            init_bn(self.bn)

    def forward(self, x):
        y = self.conv(x)
        if self.bn is not None:
            y = self.bn(y)
        return F.relu(y, inplace=True) if self.relu else y


class Conv3d(nn.Module):
    """3-D convolution + BatchNorm3d + ReLU with the reference's submodule names (nn/conv.py:176-216).  The layers of
    ``networks.VolumeConv`` are these containers, so its checkpoints load unchanged; ``VolumeConv.forward`` runs them
    through the fused sm_90a kernels, and this forward is the stock-library path for stand-alone use."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, relu=True, bn=True, bn_momentum=0.1, **kwargs):
        super().__init__()
        if stride not in (1, 2):
            raise ValueError("Conv3d: stride must be 1 or 2, got %r" % (stride,))
        self.out_channels, self.kernel_size, self.stride, self.relu = out_channels, kernel_size, stride, bool(relu)
        self.conv = nn.Conv3d(in_channels, out_channels, kernel_size, stride=stride, bias=not bn, **kwargs)
        self.bn = nn.BatchNorm3d(out_channels, momentum=bn_momentum) if bn else None
        self.init_weights()

    def init_weights(self):
        init_uniform(self.conv)
        if self.bn is not None:
            init_bn(self.bn)

    def forward(self, x):
        y = self.conv(x)
        if self.bn is not None:
            y = self.bn(y)
        return F.relu(y, inplace=True) if self.relu else y


class Deconv3d(nn.Module):
    """3-D transposed convolution + BatchNorm3d + ReLU with the reference's submodule names (its nn/conv.py
    Deconv3d).  With kernel 3, stride 2, padding 1 and output_padding 1, as VolumeConv uses it, the output is
    exactly twice the input on every axis."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, relu=True, bn=True, bn_momentum=0.1, **kwargs):
        super().__init__()
        if stride not in (1, 2):
            raise ValueError("Deconv3d: stride must be 1 or 2, got %r" % (stride,))
        self.out_channels, self.stride, self.relu = out_channels, stride, bool(relu)
        self.conv = nn.ConvTranspose3d(in_channels, out_channels, kernel_size, stride=stride, bias=not bn, **kwargs)
        self.bn = nn.BatchNorm3d(out_channels, momentum=bn_momentum) if bn else None
        self.init_weights()

    def init_weights(self):
        init_uniform(self.conv)
        if self.bn is not None:
            init_bn(self.bn)

    def forward(self, x):
        y = self.conv(x)
        if self.bn is not None:
            y = self.bn(y)
        return F.relu(y, inplace=True) if self.relu else y
