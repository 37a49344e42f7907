"""Conv1d / Conv2d + BN + ReLU containers (reference nn/conv.py:7-41, 43-81).  Parameter names
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
