"""Quantized MobileNetV2 graph on the hawq_b200 modules (module API of reference ``utils/models/q_mobilenetv2.py:12-262``).

Same module names, constructor reads and forward wiring as the reference's ``Q_LinearBottleneck`` / ``Q_MobileNetV2`` (so its
bit configs, ``bit_config.py:3602-4202``, and checkpoints key identically):

  unit:  quant_act (16 -> low bit, from the previous unit's scale) -> conv1 1x1 + ReLU6 -> quant_act1 -> conv2 depthwise 3x3 +
         ReLU6 -> quant_act2 -> conv3 1x1 (linear) -> quant_act_int32 (case 0, or case 1 with the unit input as identity: no ReLU)
  net:   quant_input -> init_block 3x3/2 + ReLU6 -> quant_act_int32 -> units -> quant_act_before_final_block -> final_block 1x1 +
         ReLU6 -> quant_act_int32_final -> final_pool -> quant_act_output -> output (QuantConv2d 1x1) -> logits

Un-frozen, the graph runs the reference's fake-quant arithmetic (calibration; tests/test_mobilenetv2_cpu.py).  Frozen, it runs on
the integer engine (qtensor.py, DESIGN.md section 2 row f3): the stem and the depthwise layers on their own kernels
(hawq_stem3x3_i8, hawq_dwconv3x3), every 1x1 layer on the convolution kernel with channels zero-padded to multiples of 64, ReLU6
as a per-channel output clamp of the consuming QuantAct, the signed 16-bit stream stored as int32, and the 1x1 classifier as
fp32 logits; ``compile_model`` captures it in one CUDA graph like the ResNets.
"""
import torch.nn as nn

from .modules import QuantAct, QuantAveragePool2d, QuantBnConv2d, QuantConv2d
from .synthetic import MOBILENETV2_CHANNELS


def _folded(block):
    """QuantBnConv2d over one float conv + BN pair of the wrapped model."""
    q = QuantBnConv2d()
    q.set_param(block.conv, block.bn)
    return q


class Q_LinearBottleneck(nn.Module):
    """Inverted-residual unit: [expand 1x1 + ReLU6] -> depthwise 3x3 + ReLU6 -> linear 1x1 projection, every edge behind a QuantAct;
    module names as in the reference (``quant_act``, ``conv1``, ``quant_act1``, ``conv2``, ``quant_act2``, ``conv3``, ``quant_act_int32``)."""

    def __init__(self, model, in_channels, out_channels, stride, expansion, remove_exp_conv=False):
        super().__init__()
        self.residual = stride == 1 and in_channels == out_channels
        self.use_exp_conv = expansion or not remove_exp_conv
        self.activatition_func = nn.ReLU6()          # (attribute name as in the reference)
        self.quant_act = QuantAct()
        stages = (1, 2) if self.use_exp_conv else (2,)
        for k in stages:                             # expand (optional) and depthwise, each followed by ReLU6 + QuantAct
            self.add_module("conv%d" % k, _folded(getattr(model, "conv%d" % k)))
            self.add_module("quant_act%d" % k, QuantAct())
        self._relu6_stages = stages
        self.conv3 = _folded(model.conv3)
        self.quant_act_int32 = QuantAct()

    def forward(self, x, scaling_factor_int32=None):
        unit_input = x
        x, a_sf = self.quant_act(x, scaling_factor_int32, None, None, None, None)       # 16-bit stream -> low bit
        for k in self._relu6_stages:
            x, w_sf = getattr(self, "conv%d" % k)(x, a_sf)
            x, a_sf = getattr(self, "quant_act%d" % k)(self.activatition_func(x), a_sf, w_sf, None, None)
        x, w_sf = self.conv3(x, a_sf)                # linear bottleneck: nothing between the projection and the sum
        if not self.residual:
            return self.quant_act_int32(x, a_sf, w_sf, None, None, None)
        # case 1 with the unit's own input (scale of the previous quant_act_int32) as identity; no ReLU follows
        return self.quant_act_int32(x + unit_input, a_sf, w_sf, unit_input, scaling_factor_int32, None)


class Q_MobileNetV2(nn.Module):
    """quant_input -> init_block -> units -> final_block -> pool -> 1x1 classifier; ``channels`` lists the output width of every unit
    per stage (a new stage starts where the float model downsamples)."""

    def __init__(self, model, channels=None, remove_exp_conv=False):
        super().__init__()
        f = model.features
        self.channels = [list(c) for c in (channels or MOBILENETV2_CHANNELS)]
        self.activatition_func = nn.ReLU6()
        self.quant_input = QuantAct()
        self.init_block = _folded(f.init_block)
        self.quant_act_int32 = QuantAct()
        self.features = nn.Sequential()
        width = f.init_block.conv.out_channels
        for si, widths in enumerate(self.channels, 1):
            src, stage = getattr(f, "stage%d" % si), nn.Sequential()
            for ui, cout in enumerate(widths, 1):
                first_of_net = si == 1 and ui == 1
                stage.add_module("unit%d" % ui, Q_LinearBottleneck(getattr(src, "unit%d" % ui), width, cout,
                                                                    stride=2 if (ui == 1 and si > 1) else 1,
                                                                    expansion=not first_of_net, remove_exp_conv=remove_exp_conv))
                width = cout
            self.features.add_module("stage%d" % si, stage)
        self.quant_act_before_final_block = QuantAct()
        self.features.add_module("final_block", _folded(f.final_block))
        self.quant_act_int32_final = QuantAct()
        pool = QuantAveragePool2d()
        pool.set_param(f.final_pool)
        self.features.add_module("final_pool", pool)
        self.quant_act_output = QuantAct()
        self.output = QuantConv2d()
        self.output.set_param(model.output)

    def units(self):
        for si, widths in enumerate(self.channels, 1):
            stage = getattr(self.features, "stage%d" % si)
            for ui in range(1, len(widths) + 1):
                yield getattr(stage, "unit%d" % ui)

    def forward(self, x):
        relu6 = self.activatition_func
        x, a_sf = self.quant_input(x)
        x, w_sf = self.init_block(x, a_sf)
        x, a_sf = self.quant_act_int32(relu6(x), a_sf, w_sf, None, None)
        for unit in self.units():
            x, a_sf = unit(x, a_sf)
        x, a_sf = self.quant_act_before_final_block(x, a_sf, None, None, None, None)
        x, w_sf = self.features.final_block(x, a_sf)
        x, a_sf = self.quant_act_int32_final(relu6(x), a_sf, w_sf, None, None, None)
        x = self.features.final_pool(x, a_sf)
        x, a_sf = self.quant_act_output(x, a_sf, None, None, None, None)
        logits, _ = self.output(x, a_sf)
        return logits.view(logits.size(0), -1)


def q_mobilenetv2_w1(model):
    """Quantized MobileNetV2-1.0 from a float model with the pytorchcv attribute layout (reference ``q_mobilenetv2_w1``)."""
    return Q_MobileNetV2(model)
