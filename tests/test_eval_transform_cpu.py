"""The evaluation transform on the host: the numpy model of hawq_resize_crop_quantize_u8 (tests/eval_transform_model.py) against the
torchvision + PIL fixture and, where those packages are installed, against them live; the size and crop rules; PackedImages and
collate_images."""
import hashlib
import json
import os

import numpy as np
import pytest
import torch

from hawq_b200.eval_transform import PackedImages, center_crop_offsets, collate_images, resized_size, source_box
from tests import abi_model as am
from tests import eval_transform_cases as etc
from tests import eval_transform_model as etm
from tests.util import GOLDEN, load_golden


def fixture_rows():
    g = load_golden(etc.FIXTURE)
    names = ["h", "w", "kind", "seed", "size", "crop_h", "crop_w", "oh", "ow", "top", "left"]
    return [dict(zip(names, (int(g[n][i]) for n in names)), sha256=str(g["sha256"][i])) for i in range(len(g["h"]))], json.loads(str(g["meta"]))


def test_fixture_covers_the_cases_it_was_made_from():
    rows, meta = fixture_rows()
    assert [(r["h"], r["w"], r["kind"], r["seed"], r["size"], (r["crop_h"], r["crop_w"])) for r in rows] == etc.cases()
    assert meta["pillow"] and meta["torchvision"]
    assert len(rows) >= 57 + 1 + 2 + 1


@pytest.mark.parametrize("i", range(len(etc.cases())))
def test_model_matches_the_fixture_digest(i):
    rows, _ = fixture_rows()
    r = rows[i]
    crop = (r["crop_h"], r["crop_w"])
    oh, ow = resized_size(r["h"], r["w"], r["size"])
    assert (oh, ow) == (r["oh"], r["ow"])
    assert center_crop_offsets(oh, ow, *crop) == (r["top"], r["left"])
    out = etm.eval_crop_u8(etc.image(r["h"], r["w"], r["kind"], r["seed"]), r["size"], crop)
    assert out.shape == crop + (3,)
    assert hashlib.sha256(out.tobytes()).hexdigest() == r["sha256"], r


def test_model_matches_live_torchvision_on_random_geometries():
    Image = pytest.importorskip("PIL.Image")
    T = pytest.importorskip("torchvision.transforms")
    r = np.random.RandomState(77)
    for trial in range(200):
        size = int(r.choice([256, 256, 342, 300]))
        crop = (224, 224) if size == 256 else (299, 299) if size == 342 else (int(r.randint(1, 301)), int(r.randint(1, 301)))
        h, w = (int(v) for v in (r.randint(1, 900, size=2) if trial % 4 else r.randint(1, 120, size=2)))
        img = etc.image(h, w, trial % 2, 5000 + trial)
        want = np.asarray(T.CenterCrop(crop)(T.Resize(size)(Image.fromarray(img))))
        assert np.array_equal(etm.eval_crop_u8(img, size, crop), want), (h, w, size, crop)


def test_size_and_crop_rules_match_torchvision():
    F = pytest.importorskip("torchvision.transforms.functional")
    r = np.random.RandomState(3)
    sizes = [(h, w) for h in range(1, 41) for w in range(1, 41)] + [tuple(int(v) for v in r.randint(1, 16385, size=2)) for _ in range(3000)]
    for h, w in sizes:
        for s in (256, 342, 4097):
            assert tuple(F._compute_resized_output_size((h, w), [s])) == resized_size(h, w, s), (h, w, s)
    for oh in range(224, 300):
        for ow in (224, 225, 226, 227, 341, 343):
            grid = torch.arange(oh * ow).view(1, oh, ow)
            top_left = int(F.center_crop(grid, [224, 224])[0, 0, 0])
            assert center_crop_offsets(oh, ow, 224, 224) == divmod(top_left, ow), (oh, ow)
    assert center_crop_offsets(341, 341, 224, 224) == (58, 58)      # 58.5 rounds to even
    assert center_crop_offsets(343, 343, 224, 224) == (60, 60)      # 59.5 rounds to even
    with pytest.raises(ValueError):
        center_crop_offsets(200, 300, 224, 224)


def test_source_box_is_what_the_crop_reads():
    assert source_box(256, 256, 256, (224, 224)) == ((16, 225), (16, 225))   # scale 1: one tap of each window weighs 0
    (r0, rn), (c0, cn) = source_box(16384, 16384, 256, (224, 224))
    assert 0 <= r0 and r0 + rn <= 16384 and rn > 224 * 63


def test_collate_packs_arrays_tensors_and_pil_images_with_targets():
    r = np.random.RandomState(0)
    imgs = [r.randint(0, 256, size=(h, w, 3), dtype=np.uint8) for h, w in [(5, 7), (1, 1), (300, 2)]]
    samples = [(imgs[0], 3), (torch.from_numpy(imgs[1]), 1), (imgs[2], 4)]
    try:
        from PIL import Image
        samples[2] = (Image.fromarray(imgs[2]), 4)
    except ImportError:
        pass
    p = collate_images(samples)
    assert isinstance(p, PackedImages) and len(p) == 3
    assert p.sizes.tolist() == [[5, 7], [1, 1], [300, 2]] and p.sizes.dtype == torch.int32
    assert torch.equal(p.targets, torch.tensor([3, 1, 4]))
    assert p.pixels.numel() == sum(a.size for a in imgs)
    for i, a in enumerate(imgs):
        assert np.array_equal(p.image(i).numpy(), a)
    t = p.table(5)
    assert t.dtype == torch.int64 and t.shape == (5, 2)
    assert t[:, 0].tolist()[:3] == [0, 105, 108]
    assert t.view(torch.int32)[:, 2:4].tolist() == [[5, 7], [1, 1], [300, 2], [0, 0], [0, 0]]   # absent slots: h = 0
    with pytest.raises(ValueError):
        p.table(2)
    q = collate_images(imgs)                                        # images without targets
    assert q.targets is None and torch.equal(q.pixels, p.pixels)


@pytest.mark.parametrize("shape", [(0, 4, 3), (4, 0, 3), (16385, 1, 3), (1, 16385, 3)])
def test_collate_rejects_sides_outside_the_supported_range(shape):
    with pytest.raises(ValueError):
        collate_images([np.zeros(shape, dtype=np.uint8)])


def test_collate_accepts_the_largest_sides():
    p = collate_images([np.zeros((16384, 1, 3), dtype=np.uint8), np.zeros((1, 16384, 3), dtype=np.uint8)])
    assert p.sizes.tolist() == [[16384, 1], [1, 16384]]


@pytest.mark.parametrize("bad", [np.zeros((4, 4), np.uint8), np.zeros((4, 4, 4), np.uint8), np.zeros((4, 4, 3), np.float32),
                                 torch.zeros((3, 4, 4), dtype=torch.uint8)])
def test_collate_rejects_what_is_not_an_hwc_rgb_image(bad):
    with pytest.raises(ValueError):
        collate_images([bad])


def test_collate_rejects_pil_images_that_are_not_rgb():
    Image = pytest.importorskip("PIL.Image")
    with pytest.raises(ValueError):
        collate_images([Image.new("L", (4, 4))])
    with pytest.raises(ValueError):
        collate_images([Image.new("RGBA", (4, 4))])


def test_packed_images_check_their_sizes():
    with pytest.raises(ValueError):
        PackedImages(torch.zeros(10, dtype=torch.uint8), torch.tensor([[2, 2]], dtype=torch.int32))       # 12 bytes described
    with pytest.raises(ValueError):
        PackedImages(torch.zeros(0, dtype=torch.uint8), torch.tensor([[0, 5]], dtype=torch.int32))


def test_dataloader_pinning_reaches_packed_images(monkeypatch):
    """DataLoader(pin_memory=True) pins a batch through its pin_memory() method; PackedImages.pin_memory pins every tensor."""
    from torch.utils.data._utils import pin_memory as pm
    pinned = []
    monkeypatch.setattr(torch.Tensor, "pin_memory", lambda self, *a, **k: pinned.append(self) or self.clone())
    p = collate_images([(np.ones((3, 4, 3), np.uint8), 0), (np.ones((2, 2, 3), np.uint8), 1)])
    q = pm.pin_memory(p)
    assert isinstance(q, PackedImages) and q is not p
    assert any(t is p.pixels for t in pinned) and any(t is p.sizes for t in pinned) and any(t is p.targets for t in pinned)
    assert torch.equal(q.pixels, p.pixels) and torch.equal(q.sizes, p.sizes)


def test_model_fills_absent_and_invalid_slots_with_the_zero_pixel():
    r = np.random.RandomState(1)
    img = r.randint(0, 256, size=(300, 400, 3), dtype=np.uint8)
    p = collate_images([img])
    table = p.table(4)
    table[2, 0] = 1                                                 # image 2 would end past the arena
    table.view(torch.int32)[2, 2:4] = torch.tensor([300, 400], dtype=torch.int32)
    table.view(torch.int32)[3, 2:4] = torch.tensor([16385, 1], dtype=torch.int32)
    out = torch.zeros(4 * 224 * 224 * 3, dtype=torch.int8)
    args = dict(size=256, crop=(224, 224), mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225), scale=0.02, clamp=(-128, 127))
    etm.resize_crop_quantize_u8(p.pixels, table, out=out, **args)
    zero = torch.zeros(4 * 224 * 224 * 3, dtype=torch.int8)
    am.quantize_input_u8(torch.zeros((4, 224, 224, 3), dtype=torch.uint8), args["mean"], args["std"], args["scale"], args["clamp"], zero)
    o, z = out.view(4, -1), zero.view(4, -1)
    assert torch.equal(o[1:], z[1:]) and not torch.equal(o[0], z[0])
    crop = torch.zeros(4 * 224 * 224 * 3, dtype=torch.int8)
    am.quantize_input_u8(torch.from_numpy(etm.eval_crop_u8(img, 256, (224, 224)))[None], args["mean"], args["std"], args["scale"],
                         args["clamp"], crop[:224 * 224 * 3])
    assert torch.equal(o[0], crop.view(4, -1)[0])


def test_cpu_backend_routes_the_transform_to_the_model(monkeypatch):
    from hawq_b200 import ops
    etm.install_cpu_backend(monkeypatch)
    assert ops.resize_crop_quantize_u8 is etm.resize_crop_quantize_u8
    assert ops.quantize_input_u8 is am.quantize_input_u8
