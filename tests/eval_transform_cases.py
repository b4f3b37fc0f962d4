"""The images of the evaluation-transform fixture (tests/golden/eval_transform_pil.npz, written by
tests/golden/make_eval_transform_golden.py): every case is an (h, w, kind, seed) image, regenerated from its seed where it is
checked, and a (resize, crop) setting.  kind 0: uniform noise; 1: smooth ramps that wrap around (long flat runs and sharp edges)."""
import numpy as np

FIXTURE = "eval_transform_pil.npz"
NOISE, SMOOTH = 0, 1

EDGE_SIZES = [(1, 1), (1, 5), (5, 1), (3, 700), (2, 2000), (224, 224), (256, 256), (257, 257), (255, 600), (256, 341), (256, 343),
              (4000, 3000), (500, 375), (375, 500), (333, 500), (700, 3), (2000, 2)]
UPSCALE_SIZES = [(100, 80), (150, 200), (223, 223), (64, 300), (17, 31)]
INCEPTION_SIZES = [(500, 375), (375, 500), (299, 299), (342, 342), (343, 700), (100, 150), (1200, 900)]
MAX_SIDE_CASE = 16384
EXTREME_SIZES = [(16384, 16), (16, 16384)]
LARGEST_DOWNSCALE = (16384, 16384)          # both passes downsize by 64: 129-tap windows


def cases():
    """[(h, w, kind, seed, resize, (crop_h, crop_w))]: 40 seeded random sizes in 60..700 (half noise, half smooth), the edge sizes,
    upscaled images, the InceptionV3 setting 342 / 299, 16384-px sides and the largest downscale."""
    r = np.random.RandomState(2024)
    out = [(int(r.randint(60, 701)), int(r.randint(60, 701)), i % 2, 0, 256, (224, 224)) for i in range(40)]
    out += [(h, w, NOISE, 0, 256, (224, 224)) for h, w in EDGE_SIZES]
    out += [(h, w, i % 2, 0, 256, (224, 224)) for i, (h, w) in enumerate(UPSCALE_SIZES)]
    out += [(h, w, i % 2, 0, 342, (299, 299)) for i, (h, w) in enumerate(INCEPTION_SIZES)]
    out += [(h, w, NOISE, 0, 256, (224, 224)) for h, w in EXTREME_SIZES]
    out += [LARGEST_DOWNSCALE + (SMOOTH, 0, 256, (224, 224))]
    return [(h, w, kind, 1000 + i, s, c) for i, (h, w, kind, _, s, c) in enumerate(out)]


def image(h, w, kind, seed):
    """uint8 HWC RGB image of one case."""
    r = np.random.RandomState(seed)
    if kind == NOISE:
        return r.randint(0, 256, size=(h, w, 3), dtype=np.uint8)
    a = r.randint(1, 7, size=(2, 3)).astype(np.uint8)
    ys, xs = (np.arange(h) % 256).astype(np.uint8), (np.arange(w) % 256).astype(np.uint8)
    img = np.empty((h, w, 3), dtype=np.uint8)
    for c in range(3):                       # (a0 * y + a1 * x) mod 256, in uint8 arithmetic
        img[:, :, c] = (ys * a[0, c])[:, None] + (xs * a[1, c])[None, :]
    return img
