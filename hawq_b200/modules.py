"""Drop-in counterparts of the reference's quantization modules (same class names, constructor keywords,
``set_param`` / ``fix`` / ``unfix``, registered buffer names and (tensor, scale) calling convention as
reference ``utils/quantization_utils/quant_modules.py``), so that HAWQ graphs, bit configs (attributes written with
plain ``setattr``, reference ``quant_train.py:264-299``) and checkpoints load unchanged.

Two regimes, chosen exactly like the reference does (``fix_flag`` / ``running_stat``):

* un-frozen: float "fake-quant" arithmetic in torch (``quant_math``) — this is the calibration / QAT-side behaviour
  (range statistics are updated); it is not the product's hot path.
* frozen (after ``freeze_model``): integer-only execution on the H100 kernels behind the C ABI.  A frozen module
  accepts an ``IntActivation`` payload from the previous engine module (no fp32 round trip) or a CUDA fp32
  tensor at a graph edge; there is no CPU or PyTorch fallback — a frozen forward without CUDA raises.
  ``hawq_b200.compile_model`` turns a whole frozen graph into a fused plan replayed as one CUDA graph.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.nn import Module, Parameter

from . import quant_math as qmath


def _split(x, sf):
    """(tensor, scale[, channel_num]) tuple-or-positional convention (quant_modules.py:83-85,219-223,395-397)."""
    if type(x) is tuple:
        return x[0], x[1]
    return x, sf


def _check_mode(mode):
    if mode not in ("symmetric", "asymmetric"):
        raise ValueError("unknown quant mode: {}".format(mode))


_generation = [0]


def _next_generation():
    """Monotonic counter for cache keys of installed overrides (never reused, unlike id())."""
    _generation[0] += 1
    return _generation[0]


def _drop_plan(module):
    """unfix(): the device-resident integer plan is rebuilt on the next frozen forward (SURVEY.md 8(b) lifecycle)."""
    module.__dict__.pop("_hawq_cache", None)


def _frozen_dispatch(module, name, *args, **kw):
    from . import qtensor
    return getattr(qtensor, name)(module, *args, **kw)


class QuantAct(Module):
    """Activation (re)quantisation — reference quant_modules.py:133-305."""

    def __init__(self, activation_bit=4, act_range_momentum=0.95, full_precision_flag=False, running_stat=True,
                 quant_mode="symmetric", fix_flag=False, act_percentile=0, fixed_point_quantization=False):
        super().__init__()
        self.activation_bit = activation_bit
        self.act_range_momentum = act_range_momentum
        self.full_precision_flag = full_precision_flag
        self.running_stat = running_stat
        self.quant_mode = quant_mode
        self.fix_flag = fix_flag
        self.act_percentile = act_percentile
        self.fixed_point_quantization = fixed_point_quantization
        self.register_buffer('x_min', torch.zeros(1))
        self.register_buffer('x_max', torch.zeros(1))
        self.register_buffer('act_scaling_factor', torch.zeros(1))
        self.register_buffer('pre_weight_scaling_factor', torch.ones(1))
        self.register_buffer('identity_weight_scaling_factor', torch.ones(1))

    def extra_repr(self):
        return "activation_bit={}, quant_mode={}, Act_min: {:.2f}, Act_max: {:.2f}".format(
            self.activation_bit, self.quant_mode, self.x_min.item(), self.x_max.item())

    def fix(self):
        self.running_stat = False
        self.fix_flag = True

    def unfix(self):
        self.running_stat = True
        self.fix_flag = False
        self.load_frozen_scale(None)      # a stored scale belongs to the frozen plan: ranges calibrated from here on take over

    def load_frozen_scale(self, scale):
        """Use a stored ``act_scaling_factor`` (quantized_checkpoint.pth.tar) instead of the scale implied by x_min / x_max;
        ``None`` returns to the range buffers."""
        self.__dict__["_override_gen"] = _next_generation()
        if scale is None:
            self.__dict__.pop("_scale_override", None)
            return
        sf = scale.detach().to(self.x_min.device, torch.float32).reshape(-1)[:1].clone()
        self.__dict__["_scale_override"] = sf
        self.act_scaling_factor = sf.clone()

    def current_scale(self):
        """Scale implied by the range buffers (quant_modules.py:262-270), or the one loaded by ``load_frozen_scale``."""
        _check_mode(self.quant_mode)
        ov = self.__dict__.get("_scale_override")
        if ov is not None:
            return ov
        if self.quant_mode == "symmetric":
            return qmath.symmetric_scale(self.activation_bit, self.x_min, self.x_max, False)
        return qmath.asymmetric_scale(self.activation_bit, self.x_min, self.x_max)

    def _observe(self, x):
        """Running range update (quant_modules.py:233-258)."""
        if self.act_percentile == 0:
            lo, hi = x.data.min(), x.data.max()
        else:
            flat = x.detach().view(-1)
            k_hi = round(flat.shape[0] * self.act_percentile * 0.01)
            hi = torch.kthvalue(flat, k=k_hi).values
            if self.quant_mode == 'asymmetric':
                lo = hi * 0
            else:
                k_lo = round(flat.shape[0] * (1 - (100 - self.act_percentile) * 0.01))
                lo = -torch.kthvalue(-flat, k=k_lo).values
        if self.x_min == self.x_max:
            self.x_min += lo
            self.x_max += hi
        elif self.act_range_momentum == -1:
            self.x_min = min(self.x_min, lo)
            self.x_max = max(self.x_max, hi)
        else:
            mom = self.act_range_momentum
            self.x_min = self.x_min * mom + lo * (1 - mom)
            self.x_max = self.x_max * mom + hi * (1 - mom)

    def forward(self, x, pre_act_scaling_factor=None, pre_weight_scaling_factor=None, identity=None,
                identity_scaling_factor=None, identity_weight_scaling_factor=None):
        channel_num = x[2] if type(x) is tuple and len(x) == 3 else None     # multi-branch input (quant_modules.py:219-223)
        x, pre_act_scaling_factor = _split(x, pre_act_scaling_factor)
        _check_mode(self.quant_mode)
        if self.full_precision_flag:
            return x
        if not self.running_stat:
            if type(pre_act_scaling_factor) is list:
                raise NotImplementedError("frozen multi-branch QuantAct (Inception concat) has no integer kernel yet")
            return _frozen_dispatch(self, "act_forward", x, pre_act_scaling_factor, pre_weight_scaling_factor,
                                    identity, identity_scaling_factor, identity_weight_scaling_factor)
        # ---- un-frozen: observe + float emulation (calibration) ----
        self._observe(x)
        self.act_scaling_factor = self.current_scale()
        sf = self.act_scaling_factor
        if pre_act_scaling_factor is None or self.fixed_point_quantization:
            q = qmath.quantize(x, self.activation_bit, sf, signed=(self.quant_mode == "symmetric"))
        elif type(pre_act_scaling_factor) is list:
            # concatenated branches, each with its own input scale (quant_modules.py:275-286): case 0 per channel slice with
            # weight scale s_i / s_i = 1
            if channel_num is None or len(channel_num) != len(pre_act_scaling_factor):
                raise ValueError("multi-branch QuantAct needs (x, [scales], [channels per branch])")
            q = x.clone()
            start = 0
            for s_i, n_i in zip(pre_act_scaling_factor, channel_num):
                q[:, start:start + n_i] = qmath.float_case0(x[:, start:start + n_i], self.activation_bit, self.quant_mode, sf, s_i, s_i / s_i)
                start += n_i
        elif identity is None:
            if pre_weight_scaling_factor is None:
                pre_weight_scaling_factor = self.pre_weight_scaling_factor
            q = qmath.float_case0(x, self.activation_bit, self.quant_mode, sf, pre_act_scaling_factor,
                                  pre_weight_scaling_factor)
        else:
            if identity_weight_scaling_factor is None:
                identity_weight_scaling_factor = self.identity_weight_scaling_factor
            q = qmath.float_case1(x, sf, pre_act_scaling_factor, pre_weight_scaling_factor, identity,
                                  identity_scaling_factor, identity_weight_scaling_factor)
        return (q * sf.view(-1), sf)


class _WeightQuantMixin:
    def load_frozen_integers(self, w_sf, w_int=None, b_int=None):
        """Use stored integers (``weight_integer`` in the float weights' layout, per-channel scale, optional 32-bit
        ``bias_integer``) instead of deriving them from the float parameters; ``w_sf=None`` returns to the float parameters."""
        self.__dict__["_override_gen"] = _next_generation()
        if w_sf is None:
            self.__dict__.pop("_frozen_integers", None)
            return
        ref = self.conv.weight if hasattr(self, "conv") else self.weight
        w_int = w_int.detach().to(ref.device, torch.float32).reshape(ref.shape).clone()
        w_sf = w_sf.detach().to(ref.device, torch.float32).reshape(-1).clone()
        if w_sf.numel() not in (1, ref.shape[0]):
            raise ValueError("scale has %d entries for %d output channels" % (w_sf.numel(), ref.shape[0]))
        lim = 2 ** (self.weight_bit - 1)
        if float(w_int.min()) < -lim or float(w_int.max()) > lim - 1:
            raise ValueError("weight_integer does not fit %d bits" % self.weight_bit)
        if b_int is not None:
            b_int = b_int.detach().to(ref.device, torch.float32).reshape(-1).clone()
        self.__dict__["_frozen_integers"] = (w_sf, w_int, b_int)

    def _weight_params(self, w, bias, pre_act_sf, percentile):
        """Per-channel (or per-tensor) symmetric integer weights + 32-bit integer bias
        (quant_modules.py:451-484 / 97-118 / 689-722)."""
        if self.quant_mode != "symmetric":
            _check_mode(self.quant_mode)
            raise Exception('For weight, we only support symmetric quantization.')
        ov = self.__dict__.get("_frozen_integers")
        if ov is not None:                       # integers loaded from a quantized checkpoint: they are the plan
            w_sf, w_int, b_int = ov
            return w_sf, w_int, b_int, w_sf.view(1, -1) * pre_act_sf.view(1, -1)
        w2 = w.data.contiguous().view(w.shape[0], -1)
        if self.per_channel:
            lo, hi = qmath.per_channel_minmax(w2, percentile)
        elif percentile == 0:
            lo, hi = w.data.min().expand(1), w.data.max().expand(1)
        else:                                    # per-tensor percentile range: get_percentile_min_max (quant_utils.py:40-70)
            lo, hi = qmath.percentile_minmax(w.data.reshape(-1), 100 - percentile, percentile)
            lo, hi = lo.expand(1), hi.expand(1)
        w_sf = qmath.symmetric_scale(self.weight_bit, lo, hi, self.per_channel)
        w_int = qmath.quantize(w, self.weight_bit, w_sf)
        bias_sf = w_sf.view(1, -1) * pre_act_sf.view(1, -1)
        b_int = None
        if bias is not None and self.quantize_bias:
            b_int = qmath.quantize(bias, self.bias_bit, bias_sf)
        return w_sf, w_int, b_int, bias_sf


class QuantBnConv2d(Module, _WeightQuantMixin):
    """Conv + BatchNorm with BN folded into per-channel symmetric integer weights — quant_modules.py:308-494."""

    def __init__(self, weight_bit=4, bias_bit=None, full_precision_flag=False, quant_mode="symmetric",
                 per_channel=False, fix_flag=False, weight_percentile=0, fix_BN=False, fix_BN_threshold=None):
        super().__init__()
        self.weight_bit = weight_bit
        self.full_precision_flag = full_precision_flag
        self.per_channel = per_channel
        self.fix_flag = fix_flag
        self.weight_percentile = weight_percentile
        self.bias_bit = bias_bit
        self.quantize_bias = bias_bit is not None
        self.quant_mode = quant_mode
        self.fix_BN = fix_BN
        self.training_BN_mode = fix_BN
        self.fix_BN_threshold = fix_BN_threshold
        self.counter = 1

    def set_param(self, conv, bn):
        self.out_channels = conv.out_channels
        self.register_buffer('convbn_scaling_factor', torch.zeros(self.out_channels))
        self.register_buffer('weight_integer', torch.zeros_like(conv.weight.data))
        self.register_buffer('bias_integer', torch.zeros_like(bn.bias))
        self.conv = conv
        self.bn = bn
        self.bn.momentum = 0.99

    def extra_repr(self):
        return "weight_bit={}, bias_bit={}, wt-channel-wise={}, quant_mode={}".format(
            self.weight_bit, self.bias_bit, self.per_channel, self.quant_mode)

    def fix(self):
        self.fix_flag = True
        self.fix_BN = True

    def unfix(self):
        self.fix_flag = False
        self.fix_BN = self.training_BN_mode
        _drop_plan(self)
        self.load_frozen_integers(None)   # stored integers belong to the frozen plan; new float weights take over

    def integer_params(self, pre_act_scaling_factor):
        """(w_sf[C], weight_integer OIHW, bias_integer[C], bias_sf[1,C]) of the folded-BN branch; also refreshes the
        buffers the reference refreshes on every forward (quant_modules.py:477-485)."""
        w, b = qmath.fold_bn(self.conv, self.bn)
        w_sf, w_int, b_int, bias_sf = self._weight_params(w, b, pre_act_scaling_factor, self.weight_percentile)
        self.convbn_scaling_factor = w_sf
        self.weight_integer = w_int
        if b_int is not None:
            self.bias_integer = b_int
        return w_sf, w_int, b_int, bias_sf

    def forward(self, x, pre_act_scaling_factor=None):
        x, pre_act_scaling_factor = _split(x, pre_act_scaling_factor)
        _check_mode(self.quant_mode)
        if self.fix_flag:
            return _frozen_dispatch(self, "conv_forward", x, pre_act_scaling_factor)
        self.counter += 1
        if self.fix_BN_threshold is None or self.counter < self.fix_BN_threshold:
            self.fix_BN = self.training_BN_mode
        else:
            self.fix_BN = True
        if not self.fix_BN:
            return self._forward_batch_stats(x)
        if self.full_precision_flag:
            raise NotImplementedError("full_precision_flag on QuantBnConv2d is not part of the integer path")
        w_sf, w_int, b_int, bias_sf = self.integer_params(pre_act_scaling_factor)
        x_int = x / pre_act_scaling_factor.view(1, -1, 1, 1)
        c = self.conv
        out = F.conv2d(x_int, w_int, b_int, c.stride, c.padding, c.dilation, c.groups)
        return (out * bias_sf.view(1, -1, 1, 1), w_sf)

    def _forward_batch_stats(self, x):
        """QAT branch with live BN statistics (quant_modules.py:417-438); training-side only."""
        c = self.conv
        w2 = c.weight.data.contiguous().view(c.out_channels, -1)
        w_sf = qmath.symmetric_scale(self.weight_bit, w2.min(dim=1).values, w2.max(dim=1).values, self.per_channel)
        w_int = qmath.quantize(c.weight, self.weight_bit, w_sf)
        y = F.conv2d(x, w_int, c.bias, c.stride, c.padding, c.dilation, c.groups) * w_sf.view(1, -1, 1, 1)
        mean, var = torch.mean(y, dim=(0, 2, 3)), torch.var(y, dim=(0, 2, 3))
        mom = self.bn.momentum
        self.bn.running_mean = self.bn.running_mean.detach() * mom + (1 - mom) * mean
        self.bn.running_var = self.bn.running_var.detach() * mom + (1 - mom) * var
        factor = self.bn.weight.view(1, -1, 1, 1) / torch.sqrt(var + self.bn.eps).view(1, -1, 1, 1)
        out = factor * (y - mean.view(1, -1, 1, 1)) + self.bn.bias.view(1, -1, 1, 1)
        return (out, w_sf.view(-1) * factor.view(-1))


class QuantConv2d(Module, _WeightQuantMixin):
    """Convolution without BN — quant_modules.py:605-736."""

    def __init__(self, weight_bit=4, bias_bit=None, full_precision_flag=False, quant_mode="symmetric",
                 per_channel=False, fix_flag=False, weight_percentile=0):
        super().__init__()
        self.full_precision_flag = full_precision_flag
        self.weight_bit = weight_bit
        self.quant_mode = quant_mode
        self.per_channel = per_channel
        self.fix_flag = fix_flag
        self.weight_percentile = weight_percentile
        self.bias_bit = bias_bit
        self.quantize_bias = bias_bit is not None

    def set_param(self, conv):
        self.in_channels, self.out_channels = conv.in_channels, conv.out_channels
        self.kernel_size, self.stride, self.padding = conv.kernel_size, conv.stride, conv.padding
        self.dilation, self.groups = conv.dilation, conv.groups
        self.conv = conv
        self.register_buffer('conv_scaling_factor', torch.zeros(self.out_channels))
        self.weight = Parameter(conv.weight.data.clone())
        self.register_buffer('weight_integer', torch.zeros_like(self.weight, dtype=torch.int8))
        self.bias = Parameter(conv.bias.data.clone()) if conv.bias is not None else None

    def fix(self):
        self.fix_flag = True

    def unfix(self):
        self.fix_flag = False
        _drop_plan(self)
        self.load_frozen_integers(None)   # stored integers belong to the frozen plan; new float weights take over

    def integer_params(self, pre_act_scaling_factor):
        w_sf, w_int, b_int, bias_sf = self._weight_params(self.weight, self.bias, pre_act_scaling_factor,
                                                          self.weight_percentile)
        self.conv_scaling_factor = w_sf
        self.weight_integer = w_int
        self.bias_integer = b_int
        return w_sf, w_int, b_int, bias_sf

    def forward(self, x, pre_act_scaling_factor=None):
        x, pre_act_scaling_factor = _split(x, pre_act_scaling_factor)
        _check_mode(self.quant_mode)
        if self.fix_flag:
            return _frozen_dispatch(self, "conv_forward", x, pre_act_scaling_factor)
        w_sf, w_int, b_int, bias_sf = self.integer_params(pre_act_scaling_factor)
        if b_int is None:
            b_int = torch.zeros_like(bias_sf.view(-1))
        x_int = x / pre_act_scaling_factor.view(1, -1, 1, 1)
        c = self.conv
        out = F.conv2d(x_int, w_int, b_int, c.stride, c.padding, c.dilation, c.groups)
        return (out * bias_sf.view(1, -1, 1, 1), w_sf)


class QuantLinear(Module, _WeightQuantMixin):
    """Fully connected classifier — quant_modules.py:12-130.  Returns the fp32 logits tensor only."""

    def __init__(self, weight_bit=4, bias_bit=None, full_precision_flag=False, quant_mode='symmetric',
                 per_channel=False, fix_flag=False, weight_percentile=0):
        super().__init__()
        self.full_precision_flag = full_precision_flag
        self.weight_bit = weight_bit
        self.quant_mode = quant_mode
        self.per_channel = per_channel
        self.fix_flag = fix_flag
        self.weight_percentile = weight_percentile
        self.bias_bit = bias_bit
        self.quantize_bias = bias_bit is not None
        self.counter = 0

    def set_param(self, linear):
        self.in_features, self.out_features = linear.in_features, linear.out_features
        self.register_buffer('fc_scaling_factor', torch.zeros(self.out_features))
        self.weight = Parameter(linear.weight.data.clone())
        self.register_buffer('weight_integer', torch.zeros_like(self.weight))
        self.register_buffer('bias_integer', torch.zeros_like(linear.bias))
        self.bias = Parameter(linear.bias.data.clone()) if linear.bias is not None else None

    def fix(self):
        self.fix_flag = True

    def unfix(self):
        self.fix_flag = False
        _drop_plan(self)
        self.load_frozen_integers(None)   # stored integers belong to the frozen plan; new float weights take over

    def integer_params(self, prev_act_scaling_factor):
        w_sf, w_int, b_int, bias_sf = self._weight_params(self.weight, self.bias, prev_act_scaling_factor, 0)
        self.fc_scaling_factor = w_sf
        self.weight_integer = w_int
        if b_int is not None:
            self.bias_integer = b_int
        return w_sf, w_int, b_int, bias_sf

    def forward(self, x, prev_act_scaling_factor=None):
        x, prev_act_scaling_factor = _split(x, prev_act_scaling_factor)
        _check_mode(self.quant_mode)
        if self.fix_flag:
            return _frozen_dispatch(self, "linear_forward", x, prev_act_scaling_factor)
        w_sf, w_int, b_int, bias_sf = self.integer_params(prev_act_scaling_factor)
        x_int = x / prev_act_scaling_factor.view(1, -1)
        return torch.round(F.linear(x_int, weight=w_int, bias=b_int)) * bias_sf[0].view(1, -1)


class QuantAveragePool2d(Module):
    """Integer average pooling: trunc(mean(x_int) + 0.01) — quant_modules.py:557-602."""

    def __init__(self, kernel_size=7, stride=1, padding=0):
        super().__init__()
        self.kernel_size, self.stride, self.padding = kernel_size, stride, padding
        self.final_pool = nn.AvgPool2d(kernel_size=kernel_size, stride=stride, padding=padding)

    def set_param(self, pool):
        self.final_pool = pool

    def forward(self, x, x_scaling_factor=None):
        x, x_scaling_factor = _split(x, x_scaling_factor)
        from .qtensor import IntActivation
        if isinstance(x, IntActivation):
            return _frozen_dispatch(self, "avgpool_forward", x, x_scaling_factor)
        if x_scaling_factor is None:
            return self.final_pool(x)
        sf = x_scaling_factor.view(-1)
        x_int = torch.trunc(self.final_pool(torch.round(x / sf)) + 0.01)
        return (x_int * sf, sf)


class QuantMaxPool2d(Module):
    """quant_modules.py:497-529."""

    def __init__(self, kernel_size=3, stride=2, padding=0):
        super().__init__()
        self.kernel_size, self.stride, self.padding = kernel_size, stride, padding
        self.pool = nn.MaxPool2d(kernel_size=kernel_size, stride=stride, padding=padding)

    def forward(self, x, x_scaling_factor=None):
        x, x_scaling_factor = _split(x, x_scaling_factor)
        return (self.pool(x), x_scaling_factor)


class QuantDropout(Module):
    """quant_modules.py:532-554."""

    def __init__(self, p=0):
        super().__init__()
        self.dropout = nn.Dropout(p)

    def forward(self, x, x_scaling_factor=None):
        x, x_scaling_factor = _split(x, x_scaling_factor)
        return (self.dropout(x), x_scaling_factor)


_QUANT_LEAVES = (QuantAct, QuantConv2d, QuantLinear, QuantBnConv2d)


def _walk(model, method):
    """Traversal rule of freeze_model / unfreeze_model (quant_modules.py:739-780): quant leaves get fix()/unfix(),
    Sequentials recurse over children, anything else recurses over attributes whose name does not contain 'norm'."""
    if type(model) in _QUANT_LEAVES:
        getattr(model, method)()
    elif type(model) == nn.Sequential:
        for _, m in model.named_children():
            _walk(m, method)
    else:
        for attr in dir(model):
            mod = getattr(model, attr)
            if isinstance(mod, nn.Module) and 'norm' not in attr:
                _walk(mod, method)


def freeze_model(model):
    """Fix activation ranges / BN statistics: switches the quant modules to the integer CUDA path."""
    _walk(model, "fix")


def unfreeze_model(model):
    _walk(model, "unfix")
