"""TEST INFRASTRUCTURE: an executable numpy model of hawq_resize_crop_quantize_u8 (include/hawq_b200.h), the evaluation transform of
a ragged image batch, alongside the ABI model of tests/abi_model.py, whose quantize_input_u8 it ends with.

  * ``eval_crop_u8`` restates torchvision Resize + CenterCrop on a PIL RGB image (PIL's bilinear 8-bit resample) for one image;
  * ``resize_crop_quantize_u8`` takes the same arguments as hawq_b200.ops.resize_crop_quantize_u8 and writes its output in place;
  * ``install_cpu_backend(monkeypatch)`` routes the ABI model's launchers and this one to CPU tensors;
  * ``run_both`` runs this model and the library on the same buffers, the library in guarded, poisoned allocations."""
import numpy as np
import torch

from tests import abi_model as am
from tests.util import guarded_call

I64 = np.int64


def _pil_bilinear_windows(n_in, n_out, first, count):
    """PIL's bilinear coefficients (ImagingResample, 8 bits per channel) of output samples [first, first + count) of a pass from n_in
    to n_out samples: (xmin [count], fixed-point k [count, taps], zero past each window).  numpy float64 operations are single IEEE
    operations, as in the C source."""
    scale = n_in / n_out
    fs = max(scale, 1.0)
    ss = 1.0 / fs
    center = (np.arange(first, first + count, dtype=np.float64) + 0.5) * scale
    xmin = np.maximum((center - fs + 0.5).astype(I64), 0)
    n = np.minimum((center + fs + 0.5).astype(I64), n_in) - xmin
    i = np.arange(int(n.max()))
    t = np.abs(((i[None, :] + xmin[:, None]).astype(np.float64) - center[:, None] + 0.5) * ss)
    w = np.where((t < 1.0) & (i[None, :] < n[:, None]), 1.0 - t, 0.0)
    ww = np.zeros(count)
    for j in range(w.shape[1]):                 # the sum runs in tap order
        ww = ww + w[:, j]
    w = np.divide(w, ww[:, None], out=w.copy(), where=ww[:, None] != 0.0)
    s = w * float(1 << 22)
    return xmin, np.where(w < 0.0, -0.5 + s, 0.5 + s).astype(I64)


def eval_crop_u8(img, size, crop):
    """torchvision Resize(size) (bilinear, on a PIL RGB image) + CenterCrop(crop) of one uint8 HWC image: only the crop is computed,
    horizontal pass first, each pass rounded to uint8."""
    from hawq_b200.eval_transform import center_crop_offsets, resized_size
    h, w = img.shape[:2]
    ch, cw = crop
    oh, ow = resized_size(h, w, size)
    top, left = center_crop_offsets(oh, ow, ch, cw)
    ymin, yk = _pil_bilinear_windows(h, oh, top, ch)
    xmin, xk = _pil_bilinear_windows(w, ow, left, cw)
    r0, r1 = int(ymin[0]), min(int(ymin[-1]) + yk.shape[1], h)
    tmp = np.empty((r1 - r0, cw, 3), dtype=I64)
    for a in range(r0, r1, 1024):               # horizontal pass over the rows the crop needs, in blocks
        b = min(a + 1024, r1)
        acc = np.full((b - a, cw, 3), 1 << 21, dtype=I64)
        for i in range(xk.shape[1]):
            acc += img[a:b, np.minimum(xmin + i, w - 1), :].astype(I64) * xk[None, :, i, None]
        tmp[a - r0:b - r0] = np.clip(acc >> 22, 0, 255)
    acc = np.full((ch, cw, 3), 1 << 21, dtype=I64)
    for i in range(yk.shape[1]):
        acc += tmp[np.minimum(ymin + i, r1 - 1) - r0] * yk[:, i, None, None]
    return np.clip(acc >> 22, 0, 255).astype(np.uint8)


def resize_crop_quantize_u8(pixels, table, size, crop, mean, std, scale, clamp, out):
    """hawq_resize_crop_quantize_u8: eval_crop_u8 of every present table entry (absent: zero pixels), then the ABI model's
    quantize_input_u8."""
    px = pixels.detach().cpu().numpy()
    t = table.detach().cpu()
    offs, hs, ws = t[:, 0].tolist(), t.view(torch.int32)[:, 2].tolist(), t.view(torch.int32)[:, 3].tolist()
    crops = np.zeros((len(offs), crop[0], crop[1], 3), dtype=np.uint8)
    for i, (o, h, w) in enumerate(zip(offs, hs, ws)):
        if 1 <= h <= 16384 and 1 <= w <= 16384 and 0 <= o <= px.size - 3 * h * w:
            crops[i] = eval_crop_u8(px[o:o + 3 * h * w].reshape(h, w, 3), size, crop)
    am.quantize_input_u8(torch.from_numpy(crops), mean, std, scale, clamp, out)


def install_cpu_backend(monkeypatch):
    """tests.abi_model.install_cpu_backend, with hawq_b200.ops.resize_crop_quantize_u8 routed to this model too.  Test-only."""
    from hawq_b200 import ops
    am.install_cpu_backend(monkeypatch)
    monkeypatch.setattr(ops, "resize_crop_quantize_u8", resize_crop_quantize_u8)


def run_both(args, device="cuda:0"):
    """The model, then the library on the same arguments with every tensor in a guarded, poisoned allocation (tests/util.guarded_call):
    its output must equal the model's byte for byte, every output byte must be written, and no guard byte or input may change.  The
    kernel raises no status flag.  Returns (model output, library output)."""
    from hawq_b200 import ops
    ops.reset_status(0)
    resize_crop_quantize_u8(**args)
    outs, problems = guarded_call(ops.resize_crop_quantize_u8, args, {"out": args["out"]}, device)
    assert ops.get_status(0) == 0
    assert not problems, problems
    return args["out"], outs["out"].cpu()
