"""hawq_b200 — H100-native integer inference engine for HAWQ-quantized ResNets and MobileNetV2.

Public surface (mirrors the reference's module API for the quantized forward path):
  modules      QuantAct, QuantBnConv2d, QuantConv2d, QuantLinear, QuantAveragePool2d, QuantMaxPool2d, QuantDropout,
               freeze_model, unfreeze_model
  q_resnet     q_resnet18 / q_resnet50 / q_resnet101 (same module names / state_dict keys as the reference)
  q_mobilenetv2  q_mobilenetv2_w1 (same module names as the reference; frozen, it runs on the integer engine too)
  bit_config   bit_config_dict(), get_bit_config(arch, scheme), stamp_bit_config(model, cfg)
  engine       compile_model(model, example) -> CompiledModel (one CUDA graph per GPU), all_gather_logits
  eval_transform  PackedImages, collate_images: ragged batches of decoded images for compile_model(..., resize=256)
  engine_file  CompiledModel.save(path) -> one plan file; load_engine(path) runs it on the library's runtime, without the model
  ops / _lib   the C ABI (include/hawq_b200.h) through ctypes
The frozen path runs only on the in-tree CUDA library (sm_90a); there is no CPU or PyTorch fallback.
"""
from .modules import (QuantAct, QuantAveragePool2d, QuantBnConv2d, QuantConv2d, QuantDropout, QuantLinear,  # noqa: F401
                      QuantMaxPool2d, freeze_model, unfreeze_model)
from .q_resnet import (Q_ResBlockBn, Q_ResNet18, Q_ResNet50, Q_ResNet101, Q_ResUnitBn, q_resnet18, q_resnet50,  # noqa: F401
                       q_resnet101, quantize_arch_dict)
from .q_mobilenetv2 import Q_LinearBottleneck, Q_MobileNetV2, q_mobilenetv2_w1  # noqa: F401
from .bit_config import bit_config_dict, get_bit_config, stamp_bit_config  # noqa: F401
from .engine import CompiledModel, all_gather_logits, compile_model, shard_range  # noqa: F401
from .engine_file import LoadedEngine, load_engine  # noqa: F401
from .eval_transform import PackedImages, collate_images  # noqa: F401
from .qtensor import IntActivation  # noqa: F401
from .checkpoint import (apply_integer_checkpoint, export_tvm_params, load_quantized_checkpoint,  # noqa: F401
                         quantized_checkpoint_dict, save_quantized_checkpoint, save_tvm_params)

quantize_arch_dict = dict(quantize_arch_dict, mobilenetv2_w1=q_mobilenetv2_w1)      # reference quant_train.py:150-158

__version__ = "0.1.0"


def build_synthetic_qresnet(arch, scheme, calib_batch=4, calib_seed=0, act_ranges=None):
    """Seed-0 synthetic quantized ResNet or MobileNetV2 (``mobilenetv2_w1``) (SURVEY.md §8d): float skeleton -> quantized graph ->
    bit config -> calibration (one float forward on CPU, or ranges loaded like a checkpoint) -> frozen."""
    import torch
    from .synthetic import synthetic_batch, synthetic_float_mobilenetv2, synthetic_float_resnet
    net = synthetic_float_mobilenetv2(0) if arch == "mobilenetv2_w1" else synthetic_float_resnet(arch, 0)
    q = quantize_arch_dict[arch](net)
    cfg = get_bit_config(arch, scheme)
    matched = stamp_bit_config(q, cfg)
    if matched != len(cfg):
        raise RuntimeError("bit config matched %d of %d modules" % (matched, len(cfg)))
    q.eval()
    if act_ranges is None:
        with torch.no_grad():
            q(synthetic_batch(calib_batch, calib_seed))
    else:
        for name, m in q.named_modules():
            if isinstance(m, QuantAct):
                lo, hi = act_ranges[name]
                m.x_min.fill_(lo)
                m.x_max.fill_(hi)
    freeze_model(q)
    return q
