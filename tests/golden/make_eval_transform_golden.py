"""Generate tests/golden/eval_transform_pil.npz: the reference's evaluation transform, torchvision Resize(S) -> CenterCrop(C) on PIL
RGB images, applied to the seeded images of tests/eval_transform_cases.py.

Run on CPU with torchvision and Pillow installed:  python tests/golden/make_eval_transform_golden.py
Per case it records the image (h, w, kind, seed), S and the crop, the resized size and crop offsets torchvision reports, and the
sha256 of the uint8 HWC crop; the meta entry records the Pillow and torchvision versions.  Tests need neither package: they
regenerate each image from its seed and compare digests.
"""
import hashlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from tests import eval_transform_cases as etc  # noqa: E402


def main():
    import PIL
    import torchvision
    import torchvision.transforms as T
    import torchvision.transforms.functional as F
    from PIL import Image

    Image.MAX_IMAGE_PIXELS = None            # the largest case is 16384 x 16384
    rows = []
    for h, w, kind, seed, size, crop in etc.cases():
        img = Image.fromarray(etc.image(h, w, kind, seed))
        resized = T.Resize(size)(img)
        out = np.asarray(T.CenterCrop(crop)(resized))
        assert out.shape == crop + (3,), (h, w, out.shape)
        ow, oh = resized.size
        top, left = int(round((oh - crop[0]) / 2.0)), int(round((ow - crop[1]) / 2.0))
        assert np.array_equal(np.asarray(F.crop(resized, top, left, crop[0], crop[1])), out)
        rows.append((h, w, kind, seed, size, crop[0], crop[1], oh, ow, top, left, hashlib.sha256(out.tobytes()).hexdigest()))
        print(h, w, size, crop, (oh, ow), (top, left))
    cols = list(zip(*rows))
    names = ["h", "w", "kind", "seed", "size", "crop_h", "crop_w", "oh", "ow", "top", "left"]
    arrays = {n: np.asarray(c, dtype=np.int64) for n, c in zip(names, cols[:11])}
    arrays["sha256"] = np.asarray(cols[11])
    arrays["meta"] = np.asarray(json.dumps({"pillow": PIL.__version__, "torchvision": torchvision.__version__,
                                            "transform": "Resize(size) -> CenterCrop(crop), bilinear, PIL RGB"}))
    np.savez_compressed(os.path.join(HERE, etc.FIXTURE), **arrays)
    print("wrote %d cases" % len(rows))


if __name__ == "__main__":
    main()
