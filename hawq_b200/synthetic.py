"""Synthetic float ResNets with the attribute layout the quantized graphs read.

The reference builds its quantized ResNets from pytorchcv float models
(reference ``quant_train.py:227``, attribute reads at ``utils/models/q_resnet.py:22-51,
84-112,206-229,270-289``).  pytorchcv and its pretrained weights cannot be fetched
here, so this module provides float networks of the same *shape*
(``features.init_block.conv.{conv,bn}``, ``features.stageN.unitM.body.convK.{conv,bn}``,
``identity_conv``, ``resize_identity``, ``output``) with seeded random weights.
They exist to drive benchmarks and parity tests with synthetic data
(SURVEY.md §8d: Kaiming conv init, randomised BN statistics).

ResNet-50/101 use the v1 stride placement (stride on the first 1x1 conv), which is
what pytorchcv's ``resnet50`` does and what the reference's tuned shapes show.
"""
import torch
import torch.nn as nn


class _ConvBn(nn.Module):
    def __init__(self, cin, cout, k, stride, pad):
        super().__init__()
        self.conv = nn.Conv2d(cin, cout, k, stride, pad, bias=False)
        self.bn = nn.BatchNorm2d(cout)


class _Body(nn.Module):
    pass


class _Unit(nn.Module):
    def __init__(self, cin, cout, stride, bottleneck):
        super().__init__()
        self.resize_identity = (cin != cout) or (stride != 1)
        self.body = _Body()
        if bottleneck:
            mid = cout // 4
            self.body.conv1 = _ConvBn(cin, mid, 1, stride, 0)
            self.body.conv2 = _ConvBn(mid, mid, 3, 1, 1)
            self.body.conv3 = _ConvBn(mid, cout, 1, 1, 0)
        else:
            self.body.conv1 = _ConvBn(cin, cout, 3, stride, 1)
            self.body.conv2 = _ConvBn(cout, cout, 3, 1, 1)
        if self.resize_identity:
            self.identity_conv = _ConvBn(cin, cout, 1, stride, 0)


class _InitBlock(nn.Module):
    def __init__(self):
        super().__init__()
        self.conv = _ConvBn(3, 64, 7, 2, 3)


class SyntheticResNet(nn.Module):
    """Float skeleton; not meant to be run, only to be wrapped by the quantized graph."""

    def __init__(self, layers, bottleneck, num_classes=1000):
        super().__init__()
        self.features = nn.Module()
        self.features.init_block = _InitBlock()
        cin = 64
        widths = [64, 128, 256, 512]
        for si, (n, w) in enumerate(zip(layers, widths)):
            stage = nn.Module()
            cout = w * 4 if bottleneck else w
            for ui in range(n):
                stride = 2 if (ui == 0 and si > 0) else 1
                setattr(stage, "unit%d" % (ui + 1), _Unit(cin, cout, stride, bottleneck))
                cin = cout
            setattr(self.features, "stage%d" % (si + 1), stage)
        self.output = nn.Linear(cin, num_classes)


_ARCHS = {
    "resnet18": ([2, 2, 2, 2], False),
    "resnet50": ([3, 4, 6, 3], True),
    "resnet101": ([3, 4, 23, 3], True),
}


def randomize_bn_(model, generator):
    """BN statistics away from identity so the fold (weight * gamma / sqrt(var+eps)) is exercised."""
    for m in model.modules():
        if isinstance(m, nn.BatchNorm2d):
            c = m.num_features
            m.running_var.copy_(torch.rand(c, generator=generator) + 0.5)
            m.running_mean.copy_(torch.randn(c, generator=generator) * 0.1)
            m.weight.data.copy_(torch.rand(c, generator=generator) + 0.5)
            m.bias.data.copy_(torch.randn(c, generator=generator) * 0.1)


def synthetic_float_resnet(arch, seed=0):
    """Seeded float skeleton: default (Kaiming-uniform) conv/linear init + randomised BN."""
    layers, bottleneck = _ARCHS[arch]
    prev = torch.random.get_rng_state()
    try:
        torch.manual_seed(seed)
        net = SyntheticResNet(layers, bottleneck)
        g = torch.Generator().manual_seed(seed + 1000)
        with torch.no_grad():
            randomize_bn_(net, g)
    finally:
        torch.random.set_rng_state(prev)
    net.eval()
    return net


def synthetic_batch(batch, seed, hw=224):
    """Seeded N(0,1) image batch, NCHW fp32 on CPU (the calibration / parity input).  hw: side of a square image, or (H, W)."""
    h, w = (hw, hw) if isinstance(hw, int) else tuple(hw)
    g = torch.Generator().manual_seed(seed)
    return torch.randn(batch, 3, h, w, generator=g)


# ----------------------------------------------------------------------------- MobileNetV2 (pytorchcv `mobilenetv2_w1` layout)
MOBILENETV2_CHANNELS = [[16], [24, 24], [32, 32, 32], [64, 64, 64, 64, 96, 96, 96], [160, 160, 160, 320]]


class _DwConvBn(nn.Module):
    def __init__(self, c, stride):
        super().__init__()
        self.conv = nn.Conv2d(c, c, 3, stride, 1, groups=c, bias=False)
        self.bn = nn.BatchNorm2d(c)


class _LinearBottleneck(nn.Module):
    def __init__(self, cin, cout, stride, expansion):
        super().__init__()
        mid = cin * 6 if expansion else cin
        self.conv1 = _ConvBn(cin, mid, 1, 1, 0)
        self.conv2 = _DwConvBn(mid, stride)
        self.conv3 = _ConvBn(mid, cout, 1, 1, 0)


class SyntheticMobileNetV2(nn.Module):
    """Float skeleton with the attributes the quantized graph reads (reference ``utils/models/q_mobilenetv2.py:45-55,142-180``):
    ``features.init_block.{conv,bn}``, ``features.stageN.unitM.convK.{conv,bn}``, ``features.final_block.{conv,bn}``,
    ``features.final_pool``, ``output`` (a bias-free 1x1 convolution, as in pytorchcv)."""

    def __init__(self, num_classes=1000):
        super().__init__()
        self.features = nn.Module()
        self.features.init_block = _ConvBn(3, 32, 3, 2, 1)
        cin = 32
        for si, stage_channels in enumerate(MOBILENETV2_CHANNELS):
            stage = nn.Module()
            for ui, cout in enumerate(stage_channels):
                stride = 2 if (ui == 0 and si != 0) else 1
                setattr(stage, "unit%d" % (ui + 1), _LinearBottleneck(cin, cout, stride, expansion=(si != 0 or ui != 0)))
                cin = cout
            setattr(self.features, "stage%d" % (si + 1), stage)
        self.features.final_block = _ConvBn(cin, 1280, 1, 1, 0)
        self.features.final_pool = nn.AvgPool2d(kernel_size=7, stride=1)
        self.output = nn.Conv2d(1280, num_classes, 1, bias=False)


def synthetic_float_mobilenetv2(seed=0):
    """Seeded float skeleton of MobileNetV2-1.0: default conv init + randomised BN (same recipe as the ResNets)."""
    prev = torch.random.get_rng_state()
    try:
        torch.manual_seed(seed)
        net = SyntheticMobileNetV2()
        g = torch.Generator().manual_seed(seed + 1000)
        with torch.no_grad():
            randomize_bn_(net, g)
    finally:
        torch.random.set_rng_state(prev)
    net.eval()
    return net
