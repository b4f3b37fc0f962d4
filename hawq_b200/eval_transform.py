"""Ragged batches of decoded images for the device evaluation transform (``ops.resize_crop_quantize_u8``, the head of an engine
compiled with ``resize``): torchvision's Resize(S) -> CenterCrop size and offset rules, the packed batch a ``DataLoader`` hands
over (``PackedImages``) and the ``collate_fn`` that builds it in the loader's workers (``collate_images``)."""
import numpy as np
import torch

MAX_SIDE = 16384          # largest image side the kernel accepts
MIN_RESIZE = 256          # smallest resize: a MAX_SIDE side then downsizes by at most 64 (129-tap windows)


def resized_size(h, w, size):
    """(oh, ow) of torchvision ``Resize(size)`` (an int, no max_size) for an h x w image: the short side becomes ``size``, the long one
    ``int(size * long / short)`` (an integer product, one correctly rounded division, truncated)."""
    short, long = (w, h) if w <= h else (h, w)
    new_long = int(size * long / short)
    return (new_long, size) if w <= h else (size, new_long)


def center_crop_offsets(oh, ow, ch, cw):
    """(top, left) of torchvision ``CenterCrop((ch, cw))`` on an oh x ow image that covers the crop (round half to even)."""
    if oh < ch or ow < cw:
        raise ValueError("the crop %dx%d does not fit in %dx%d (torchvision would pad)" % (ch, cw, oh, ow))
    return int(round((oh - ch) / 2.0)), int(round((ow - cw) / 2.0))


def window(in_size, out_size, xx):
    """(first, count) of the source samples output sample ``xx`` of a PIL bilinear pass from in_size to out_size reads."""
    scale = in_size / out_size
    support = max(scale, 1.0)
    center = (xx + 0.5) * scale
    first = max(int(center - support + 0.5), 0)
    return first, min(int(center + support + 0.5), in_size) - first


def source_box(h, w, size, crop):
    """(rows, cols): the source rows and columns the crop of an h x w image reads, each as a (first, count) range."""
    ch, cw = crop
    oh, ow = resized_size(h, w, size)
    top, left = center_crop_offsets(oh, ow, ch, cw)
    spans = []
    for n_in, n_out, a, n in ((h, oh, top, ch), (w, ow, left, cw)):
        first, last = window(n_in, n_out, a), window(n_in, n_out, a + n - 1)
        spans.append((first[0], last[0] + last[1] - first[0]))
    return tuple(spans)


class PackedImages:
    """A batch of RGB images of any sizes: ``pixels`` uint8 [sum of h * w * 3] (the images back to back, HWC), ``sizes`` int32 [n, 2]
    (h, w) and optional ``targets``.  ``pin_memory()`` pins the tensors (``DataLoader(pin_memory=True)`` calls it)."""

    def __init__(self, pixels, sizes, targets=None):
        sizes = torch.as_tensor(sizes, dtype=torch.int32).reshape(-1, 2)
        if pixels.dtype != torch.uint8 or pixels.dim() != 1:
            raise ValueError("pixels must be a flat uint8 tensor")
        check_sizes(sizes)
        if int((sizes[:, 0].long() * sizes[:, 1].long()).sum()) * 3 != pixels.numel():
            raise ValueError("pixels hold %d bytes, the sizes describe %d" % (pixels.numel(),
                                                                              int((sizes[:, 0].long() * sizes[:, 1].long()).sum()) * 3))
        self.pixels, self.sizes, self.targets = pixels, sizes, targets

    def __len__(self):
        return self.sizes.shape[0]

    def pin_memory(self):
        t = self.targets.pin_memory() if torch.is_tensor(self.targets) else self.targets
        return PackedImages(self.pixels.pin_memory(), self.sizes.pin_memory(), t)

    def is_pinned(self):
        return self.pixels.is_pinned()

    def offsets(self):
        """int64 [n]: byte offset of every image in ``pixels``."""
        nbytes = self.sizes[:, 0].long() * self.sizes[:, 1].long() * 3
        return torch.cumsum(nbytes, 0) - nbytes

    def table(self, slots=None):
        """The hawq_image_desc table (int64 [slots, 2]: offset, then h and w as two int32) of these images; slots past the last
        image are absent (h = 0)."""
        n = len(self)
        slots = n if slots is None else slots
        if slots < n:
            raise ValueError("%d images do not fit in %d slots" % (n, slots))
        t = torch.zeros((slots, 2), dtype=torch.int64)
        t[:n, 0] = self.offsets()
        t.view(torch.int32)[:n, 2:4] = self.sizes
        return t

    def image(self, i):
        """HWC uint8 view of image i."""
        h, w = (int(v) for v in self.sizes[i])
        o = int(self.offsets()[i])
        return self.pixels[o:o + h * w * 3].view(h, w, 3)


def check_sizes(sizes):
    bad = (sizes < 1) | (sizes > MAX_SIDE)
    if bool(bad.any()):
        i = int(torch.nonzero(bad.any(1))[0])
        raise ValueError("image %d is %dx%d: sides must lie in 1..%d" % (i, int(sizes[i, 0]), int(sizes[i, 1]), MAX_SIDE))


def _hwc(img):
    if hasattr(img, "getbands"):                            # a PIL image
        if img.mode != "RGB":
            raise ValueError("PIL images must be RGB (got mode %s): convert('RGB') first" % img.mode)
        img = np.array(img)
    t = torch.from_numpy(np.ascontiguousarray(img)) if isinstance(img, np.ndarray) else img
    if not torch.is_tensor(t) or t.dtype != torch.uint8 or t.dim() != 3 or t.shape[2] != 3:
        raise ValueError("an image must be HWC uint8 with 3 channels (numpy array, tensor or PIL RGB image)")
    return t


def collate_images(batch):
    """``DataLoader`` collate_fn: a list of images (HWC uint8 numpy arrays or tensors, or PIL RGB images), or of (image, target)
    pairs, -> ``PackedImages`` (targets collated by torch's default rule).  Raises ValueError for a side outside 1..16384."""
    pairs = len(batch) > 0 and all(isinstance(s, (tuple, list)) and len(s) == 2 for s in batch)
    imgs = [_hwc(s[0] if pairs else s) for s in batch]
    sizes = torch.tensor([[t.shape[0], t.shape[1]] for t in imgs], dtype=torch.int32).reshape(-1, 2)
    check_sizes(sizes)
    pixels = torch.cat([t.reshape(-1) for t in imgs]) if imgs else torch.empty(0, dtype=torch.uint8)
    targets = torch.utils.data.default_collate([s[1] for s in batch]) if pairs else None
    return PackedImages(pixels, sizes, targets)
