"""-m gpu: hawq_resize_crop_quantize_u8 (Resize + CenterCrop + ToTensor + Normalize + input quantisation of ragged image batches)
against its numpy model in guarded, poisoned buffers, and engines compiled with ``resize``: bit-equal to the uint8-224 and fp32
routes fed the same crops, short batches, the pipelined call with a batch that outgrows the arena, and the overflow fallback."""
import numpy as np
import pytest
import torch

import hawq_b200 as hb
from hawq_b200.engine import IMAGENET_MEAN, IMAGENET_STD
from hawq_b200.synthetic import synthetic_batch
from tests import eval_transform_cases as etc
from tests import eval_transform_model as etm
from tests.engine_harness import golden_model
from tests.kernel_harness import DEV
from tests.util import load_net_golden

pytestmark = pytest.mark.gpu

QUANT = dict(mean=IMAGENET_MEAN, std=IMAGENET_STD, scale=0.0208, clamp=(-128, 127))     # about one int8 step per pixel step


def check_kernel(images, size=256, crop=(224, 224), slots=None, table_edit=None, quant=QUANT):
    p = hb.collate_images(images)
    table = p.table(slots)
    if table_edit is not None:
        table_edit(table)
    out = torch.zeros(table.shape[0] * crop[0] * crop[1] * 3, dtype=torch.int8)
    args = dict(pixels=p.pixels, table=table, size=size, crop=crop, out=out, **quant)
    c, g = etm.run_both(args, DEV)
    assert torch.equal(c, g), (size, crop, p.sizes.tolist())
    return g


def case_images(pred):
    return [etc.image(h, w, kind, seed) for h, w, kind, seed, s, c in etc.cases() if pred(h, w, s, c)]


def test_kernel_every_fixture_geometry_in_one_mixed_batch():
    imgs = case_images(lambda h, w, s, c: s == 256 and max(h, w) < etc.MAX_SIDE_CASE)
    assert len(imgs) >= 57 + len(etc.UPSCALE_SIZES)
    check_kernel(imgs)


def test_kernel_inception_setting_342_299():
    check_kernel(case_images(lambda h, w, s, c: s == 342), size=342, crop=(299, 299))


def test_kernel_16384_px_sides_and_the_largest_downscale():
    check_kernel(case_images(lambda h, w, s, c: max(h, w) >= etc.MAX_SIDE_CASE))


def test_kernel_absent_and_invalid_slots():
    """slots past the batch, an h = 0 entry between images and entries that leave the arena or the size limit: zero pixels."""
    imgs = case_images(lambda h, w, s, c: s == 256 and max(h, w) <= 700)[:5]

    def edit(t):
        t.view(torch.int32)[1, 2] = 0                                   # absent in the middle
        t[3, 0] = 1 << 40                                               # past the arena
        t.view(torch.int32)[4, 2:4] = torch.tensor([16385, 3], dtype=torch.int32)
    g = check_kernel(imgs, slots=8, table_edit=edit).view(8, -1)
    for i in (1, 3, 4, 5, 6, 7):
        assert torch.equal(g[i], g[7]), i
    assert not torch.equal(g[0], g[7])


def imagenet_like_sizes(r, n):
    """mostly 500 x 375, 375 x 500 and 500 x 333, some 1-3 MP images and some below 256"""
    out = []
    for _ in range(n):
        u = r.rand()
        if u < 0.75:
            out.append([(500, 375), (375, 500), (500, 333), (333, 500)][r.randint(4)])
        elif u < 0.9:
            out.append(tuple(int(v) for v in r.randint(800, 2000, size=2)))
        else:
            out.append(tuple(int(v) for v in r.randint(60, 256, size=2)))
    return out


@pytest.mark.parametrize("b", [1, 8, 128])
def test_kernel_batches(b):
    r = np.random.RandomState(b)
    imgs = [etc.image(h, w, i % 2, 7000 + i) for i, (h, w) in enumerate(imagenet_like_sizes(r, b))]
    check_kernel(imgs, quant=dict(mean=(0.5, 0.4, 0.3), std=(0.2, 0.25, 0.3), scale=0.03, clamp=(-100, 90)))


def crops_u8(imgs, size=256, crop=(224, 224)):
    return torch.from_numpy(np.stack([etm.eval_crop_u8(a, size, crop) for a in imgs]))


def torch_pipeline(u8, mean=IMAGENET_MEAN, std=IMAGENET_STD):
    """transforms.ToTensor + Normalize of uint8 NHWC crops, in torch ops (fp32 NCHW)"""
    x = u8.permute(0, 3, 1, 2).to(torch.float32).div(255)
    return x.sub(torch.tensor(mean).view(1, 3, 1, 1)).div(torch.tensor(std).view(1, 3, 1, 1))


def ragged(seed, n):
    r = np.random.RandomState(seed)
    return [etc.image(h, w, i % 2, seed * 100 + i) for i, (h, w) in enumerate(imagenet_like_sizes(r, n))]


@pytest.mark.parametrize("arch", ["resnet18", "mobilenetv2_w1"])
def test_network_logits_equal_the_uint8_and_fp32_routes(arch):
    """A ragged batch through compile_model(resize=256) == the uint8-224 engine fed the model's crops == the fp32 engine fed
    ToTensor / Normalize of those crops; a short batch (a list, then pinned PackedImages) returns the matching rows."""
    _, meta = load_net_golden(arch, "uniform8")
    q = golden_model(arch, "uniform8", meta)
    slots = 8
    imgs = ragged(11, slots)
    u8 = crops_u8(imgs)
    eng = hb.compile_model(q, torch.zeros((slots, 224, 224, 3), dtype=torch.uint8, device=DEV), resize=256)
    got = eng(imgs).clone()
    eng_u = hb.compile_model(q, u8.to(DEV))
    eng_f = hb.compile_model(q, torch_pipeline(u8).to(DEV))
    want_u, want_f = eng_u(u8.to(DEV)).clone(), eng_f(torch_pipeline(u8).to(DEV)).clone()
    assert got.shape == (slots, want_u.shape[1])
    assert torch.equal(got, want_u) and torch.equal(got, want_f)
    short = eng(imgs[:5])
    assert short.shape[0] == 5 and torch.equal(short, got[:5])
    packed = hb.collate_images(imgs[2:7]).pin_memory()
    assert packed.is_pinned()
    assert torch.equal(eng(packed), got[2:7])
    assert eng.fallbacks == 0
    with pytest.raises(ValueError):
        eng(imgs + imgs[:1])


def test_run_pipelined_grows_the_arena_and_stays_exact():
    """Ragged batches from a DataLoader (collate_images, pinned), the fourth with a 4000 x 3000 image that outgrows the arena, the
    last one short: one recapture, and every yielded tensor equals the uint8-224 engine on the model's crops."""
    _, meta = load_net_golden("resnet18", "uniform8")
    q = golden_model("resnet18", "uniform8", meta)
    slots = 8
    eng = hb.compile_model(q, torch.zeros((slots, 224, 224, 3), dtype=torch.uint8, device=DEV), resize=256)
    sizes = [(500, 375), (375, 500), (500, 333), (300, 200), (150, 90)]
    imgs = [etc.image(*sizes[i % 5], i % 2, 2100 + i) for i in range(4 * slots + 3)]
    imgs[3 * slots + 2] = etc.image(4000, 3000, 0, 99)
    loader = torch.utils.data.DataLoader([(a, i) for i, a in enumerate(imgs)], batch_size=slots, collate_fn=hb.collate_images,
                                         pin_memory=True)
    batches = list(loader)
    assert all(b.is_pinned() for b in batches) and len(batches[-1]) == 3
    assert [b.pixels.numel() > eng.arena.numel() for b in batches] == [False, False, False, True, False]
    outs = [o.clone() for o in eng.run_pipelined(batches)]
    assert eng.recaptures == 1
    eng_u = hb.compile_model(q, torch.zeros((slots, 224, 224, 3), dtype=torch.uint8, device=DEV))
    for i, b in enumerate(batches):
        u8 = crops_u8([b.image(j).numpy() for j in range(len(b))])
        want = eng_u(torch.cat([u8, torch.zeros((slots - len(b), 224, 224, 3), dtype=torch.uint8)]).to(DEV))[:len(b)].cpu()
        assert torch.equal(outs[i], want), i
        assert torch.equal(b.targets, torch.arange(i * slots, i * slots + len(b)))


def test_overflowing_batch_takes_the_exact_fallback_through_the_same_head():
    """The engine-path overflow case (ResNet-18 bops_0.25, stage2.unit2's 16-bit range shrunk to 0.75, every input at the int8
    extremes): 256 x 256 images whose centre crop is a 0 / 255 pattern, with std 0.001, drive every quantised input to the clamp.
    The resize engine falls back to its int32 graph and equals the uint8-224 engine on the same crops, which falls back too, and
    the fp32 engine on ToTensor / Normalize of them."""
    _, meta = load_net_golden("resnet18", "bops_0.25")
    q = golden_model("resnet18", "bops_0.25", meta, ("stage2.unit2.quant_act_int32", 0.75))
    slots = 8
    sign = (synthetic_batch(slots, 104) > 0).permute(0, 2, 3, 1).numpy()
    imgs = []
    for i in range(slots):
        a = np.full((256, 256, 3), 128, dtype=np.uint8)
        a[16:240, 16:240] = np.where(sign[i], 255, 0)
        imgs.append(a)
    norm = dict(mean=(0.5, 0.5, 0.5), std=(0.001, 0.001, 0.001))
    eng = hb.compile_model(q, torch.zeros((slots, 224, 224, 3), dtype=torch.uint8, device=DEV), resize=256, **norm)
    got = eng(imgs[:6]).clone()
    assert eng.fallbacks == 1 and 32 in eng.graphs
    u8 = crops_u8(imgs)
    assert np.array_equal(u8.numpy()[:, :, :, 0], np.where(sign[..., 0], 255, 0))
    eng_u = hb.compile_model(q, u8.to(DEV), **norm)
    want = eng_u(u8.to(DEV))[:6]
    assert eng_u.fallbacks == 1
    assert torch.equal(got, want)
    eng_f = hb.compile_model(q, torch_pipeline(u8, **norm).to(DEV))
    assert torch.equal(eng_f(torch_pipeline(u8, **norm).to(DEV))[:6], got)


def test_resize_arguments_are_checked():
    _, meta = load_net_golden("resnet18", "uniform8")
    q = golden_model("resnet18", "uniform8", meta)
    with pytest.raises(NotImplementedError):
        hb.compile_model(q, torch.zeros((2, 224, 224, 3), dtype=torch.uint8, device=DEV), resize=256, gather=True)
    with pytest.raises(ValueError):
        hb.compile_model(q, torch.zeros((2, 224, 224, 3), dtype=torch.uint8, device=DEV), resize=224)
    with pytest.raises(ValueError):
        hb.compile_model(q, torch.zeros((2, 3, 224, 224), dtype=torch.float32, device=DEV), resize=256)
