"""-m gpu: ragged ViT batches (images of different sizes in one forward) bit for bit with the uniform calls.

Every image's rows from dss_vit_forward_k_ragged / _cls_ragged must be torch.equal to the same image run alone through
forward_k / forward_cls, in both precision modes: one-patch and 2 x 2 crops (T = 2, 5), T = 128 and 129 (one row either
side of a 128-query attention tile), VOC shapes (T = 714), 480^2 (T = 901), ViT-B/8 at 480^2 (T = 3601) next to a T = 2
crop, a grid0 x grid0 grid from non-square pixels next to a square 224^2 image (the identity rule per image), which_block
other than -1 and a 264-image batch. Also: rows past the outputs are not written, the device positional tables of
ragged and uniform forwards are dss_pos_embed_interp_host's bits (every grid up to 64 x 64 for ragged batches), and
extract_features / extract_bbox_features write what the per-image uniform forward gives."""
import ctypes as C
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest
import torch

from conftest import load_pkg

pytestmark = pytest.mark.gpu

PRECISIONS = ("fp16", "fp32")
_MODELS = {}


def _model(name="dino_vits16", precision="fp16"):
    key = (name, precision)
    if key not in _MODELS:
        vit = load_pkg("vit")
        _MODELS[key] = vit.get_model(name, seed=0, device="cuda", precision=precision)[0]
    return _MODELS[key]


def _images(shapes, seed=0):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, 256, (H, W, 3), dtype=torch.uint8, generator=g).cuda() for H, W in shapes]


def _check_k(model, shapes, which_block=-1, seed=0):
    ims = _images(shapes, seed)
    k, rows = model.forward_k_ragged(ims, which_block=which_block)
    for im, (r0, r1) in zip(ims, rows):
        alone = model.forward_k(im[None], which_block=which_block)[0]
        assert k[r0:r1].shape == alone.shape
        assert torch.equal(k[r0:r1], alone), (tuple(im.shape), which_block)


def _check_cls(model, shapes, seed=0):
    ims = _images(shapes, seed)
    cls, _ = model.forward_cls_ragged(ims)
    for b, im in enumerate(ims):
        assert torch.equal(cls[b], model.forward_cls(im[None])[0]), tuple(im.shape)


CASES = {
    "t2_t5": [(16, 16), (32, 32), (16, 16), (47, 40)],
    "t128_t129": [(16, 127 * 16), (128, 256), (16, 127 * 16 + 15), (131, 263)],
    "voc_t714": [(375, 500), (500, 375), (16, 16), (375, 500)],
    "t901": [(480, 480), (32, 32), (480, 480)],
    "identity_rule": [(224, 232), (224, 224), (232, 224), (239, 239), (224, 224)],
}


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("case", list(CASES))
def test_ragged_equals_each_image_alone(cuda, case, precision):
    model = _model(precision=precision)
    _check_k(model, CASES[case])
    _check_cls(model, CASES[case])


@pytest.mark.parametrize("precision", PRECISIONS)
def test_vitb8_t3601_next_to_a_t2_crop(cuda, precision):
    model = _model("dino_vitb8", precision)
    shapes = [(8, 8), (480, 480), (8, 8)]
    _check_k(model, shapes)
    _check_cls(model, shapes)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_which_block(cuda, precision):
    model = _model(precision=precision)
    for which in (0, 5, -3):
        _check_k(model, [(64, 48), (224, 224), (375, 500)], which_block=which, seed=which + 10)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_264_images(cuda, precision):
    model = _model(precision=precision)
    sizes = [(16, 16), (48, 80), (224, 224), (375, 500), (130, 70), (96, 96), (33, 250), (224, 232), (160, 112)]
    shapes = [sizes[(7 * i) % len(sizes)] for i in range(264)]
    ims = _images(shapes, seed=3)
    k, rows = model.forward_k_ragged(ims)
    cls, _ = model.forward_cls_ragged(ims)
    # the uniform reference per distinct shape, batched (an image's bits do not depend on its batch)
    for key in set(shapes):
        idx = [i for i, s in enumerate(shapes) if s == key]
        batch = torch.stack([ims[i] for i in idx])
        ku, cu = model.forward_k(batch), model.forward_cls(batch)
        for j, i in enumerate(idx):
            r0, r1 = rows[i]
            assert torch.equal(k[r0:r1], ku[j]), key
            assert torch.equal(cls[i], cu[j]), key


@pytest.mark.parametrize("precision", PRECISIONS)
def test_no_rows_written_past_the_outputs(cuda, precision):
    model = _model(precision=precision)
    lib = load_pkg("_lib").load()
    vit = load_pkg("vit")
    shapes = [(375, 500), (16, 16), (128, 256)]
    packed, dims = vit.pack_images(_images(shapes, seed=5))
    n = vit.ragged_rows(dims.tolist(), 16)[-1][1]
    ws = torch.empty(lib.dss_vit_ragged_workspace_bytes(model._h, dims.data_ptr(), 3, 0), dtype=torch.uint8, device="cuda")
    ws.fill_(0xFF)   # NaN-poisoned workspace
    st = torch.cuda.current_stream().cuda_stream
    k = torch.full((n + 7, model.dim), 1234.5, device="cuda")
    assert lib.dss_vit_forward_k_ragged(model._h, packed.data_ptr(), dims.data_ptr(), 3, -1, k.data_ptr(),
                                        ws.data_ptr(), ws.numel(), st) == 0
    cls = torch.full((3 + 5, model.dim), 1234.5, device="cuda")
    assert lib.dss_vit_forward_cls_ragged(model._h, packed.data_ptr(), dims.data_ptr(), 3, cls.data_ptr(),
                                          ws.data_ptr(), ws.numel(), st) == 0
    assert bool((k[n:] == 1234.5).all()) and bool((cls[3:] == 1234.5).all())
    assert bool(torch.isfinite(k[:n]).all()) and bool(torch.isfinite(cls[:3]).all())
    ref, _ = model.forward_k_ragged(packed, dims)
    assert torch.equal(k[:n], ref)


def _host_table(lib, src, g, Hp, Wp):
    out = torch.empty(Hp * Wp + 1, src.shape[1])
    assert lib.dss_pos_embed_interp_host(src.data_ptr(), g, src.shape[1], Hp, Wp, out.data_ptr()) == 0
    return out


def _resampled(src, g, Hp, Wp):
    """interp_pos_host restated in numpy, every operation rounded on its own (taps in double, sums in fp32): the
    resampled table also for the grid0 x grid0 grid of a non-square image, for which dss_pos_embed_interp_host (the
    patch-grid rule) returns the stored grid."""
    f32, A = np.float32, -0.75
    c1 = lambda x: ((A + 2.0) * x - (A + 3.0)) * x * x + 1.0
    c2 = lambda x: ((A * x - 5.0 * A) * x + 8.0 * A) * x - 4.0 * A

    def taps(n):
        rscale = f32(1.0 / ((n + 0.1) / g))
        for o in range(n):
            real = rscale * (f32(o) + f32(0.5)) - f32(0.5)
            fl = np.floor(real)
            t = float(real - fl)
            yield int(fl), [f32(c2(t + 1.0)), f32(c1(t)), f32(c1(1.0 - t)), f32(c2(2.0 - t))]

    grid = src[1:].numpy().reshape(g, g, -1)
    clamp = lambda v: min(max(v, 0), g - 1)
    rows = [src[0].numpy()]
    for iy, wy in taps(Hp):
        for ix, wx in taps(Wp):
            o = np.zeros(src.shape[1], np.float32)
            for a in range(4):
                for b in range(4):
                    o = o + (wy[a] * wx[b]) * grid[clamp(iy - 1 + a), clamp(ix - 1 + b)]
            rows.append(o)
    return torch.from_numpy(np.stack(rows))


def test_positional_tables_match_the_host_routine(cuda):
    """Every grid up to 64 x 64 (ViT-S/16, grid0 14) against dss_pos_embed_interp_host, bit for bit: K mode (the
    identity rule by patch grid). The 14 x 14 grid of a 224 x 232 image in CLS mode is resampled, not the stored grid.
    The uniform forwards, ViT-S/16 and ViT-B/8: with zero patch weight and bias, forward_tokens(img, 0) is
    [cls + pos[0], pos[1:]] for every image of the batch, pos the host routine's table (for a grid0 x grid0 grid of
    non-square pixels, which the model's own forward resamples, its numpy restatement)."""
    model = _model()
    lib = load_pkg("_lib").load()
    vit = load_pkg("vit")
    sd = vit.random_state_dict("dino_vits16", 0)
    src = sd["pos_embed"].reshape(-1, model.dim).contiguous()
    grids = [(a, b) for a in range(1, 65) for b in range(1, 65)]
    st = torch.cuda.current_stream().cuda_stream

    with ThreadPoolExecutor(8) as pool:
        for c0 in range(0, len(grids), 256):
            chunk = grids[c0:c0 + 256]
            want = list(pool.map(lambda g: _host_table(lib, src, 14, *g), chunk))
            dims = torch.tensor([[16 * a, 16 * b] for a, b in chunk], dtype=torch.int32)
            B = len(chunk)
            ws = torch.empty(lib.dss_vit_ragged_workspace_bytes(model._h, dims.data_ptr(), B, 0), dtype=torch.uint8,
                             device="cuda")
            got = torch.empty(sum(a * b + 1 for a, b in chunk), model.dim, device="cuda")
            assert lib.dss_vit_pos_embed_ragged(model._h, dims.data_ptr(), B, 0, got.data_ptr(), ws.data_ptr(),
                                                ws.numel(), st) == 0
            got = got.cpu()
            r = 0
            for g, w in zip(chunk, want):
                assert torch.equal(got[r:r + w.shape[0]], w), g
                r += w.shape[0]
    # the identity rule per image: the stored grid for 224 x 224 in both modes and for 224 x 232 in K mode only
    dims = torch.tensor([[224, 232], [224, 224]], dtype=torch.int32)
    ws = torch.empty(lib.dss_vit_ragged_workspace_bytes(model._h, dims.data_ptr(), 2, 1), dtype=torch.uint8, device="cuda")
    for mode in (0, 1):
        got = torch.empty(2 * 197, model.dim, device="cuda")
        assert lib.dss_vit_pos_embed_ragged(model._h, dims.data_ptr(), 2, mode, got.data_ptr(), ws.data_ptr(),
                                            ws.numel(), st) == 0
        got = got.cpu()
        assert torch.equal(got[197:], src)
        assert torch.equal(got[:197], src) == (mode == 0)
        assert torch.equal(got[:197], src if mode == 0 else _resampled(src, 14, 14, 14))
        assert torch.equal(got[0], src[0])

    for name in ("dino_vits16", "dino_vitb8"):
        sd = vit.random_state_dict(name, 0)
        sd["patch_embed.proj.weight"].zero_()
        sd["patch_embed.proj.bias"].zero_()
        m = vit.DinoViT(name, sd, device="cuda")
        P, g = m.patch_size, vit.TRAIN_IMG // m.patch_size
        src = sd["pos_embed"].reshape(g * g + 1, m.dim).contiguous()
        cls = sd["cls_token"].reshape(m.dim)
        assert torch.equal(_resampled(src, g, g - 1, g + 1), _host_table(lib, src, g, g - 1, g + 1))
        grids = [(1, 1), (1, 2), (1, g), (1, 3 * g), (2, 1), (g, 1), (3 * g, 1), (g - 1, g - 1), (g, g),
                 (g + 1, g + 1), (g - 1, g), (g, g + 1), (g + 1, g), (5, 9)]
        # non-square pixels on square grids: grid0 (resampled, unlike the patch-grid rule) and grid0 - 1
        sizes = [(P * a, P * b) for a, b in grids] + [(P * g, P * g + P // 2), (P * g + P - 1, P * g),
                                                      (P * (g - 1), P * (g - 1) + 3)]
        for H, W in sizes:
            Hp, Wp = H // P, W // P
            want = _resampled(src, g, g, g) if (Hp, Wp) == (g, g) and H != W else _host_table(lib, src, g, Hp, Wp)
            img = torch.randint(0, 256, (3, H, W, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(H * W))
            got = m.forward_tokens(img.cuda(), 0).cpu()   # the 1 x 1 grid: B = 3 images of T = 2 rows
            for b in range(3):
                assert torch.equal(got[b, 0], cls + want[0]), (name, H, W, b)
                assert torch.equal(got[b, 1:], want[1:]), (name, H, W, b)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_extract_commands_write_the_uniform_forwards_bits(cuda, tmp_path, precision):
    from PIL import Image
    ex = load_pkg("extract")
    model = _model(precision=precision)
    rng = np.random.default_rng(7)
    shapes = [(375, 500), (48, 64), (224, 224), (17, 33), (500, 375), (96, 96), (64, 48)]
    names = []
    for i, (H, W) in enumerate(shapes):
        names.append(f"im{i}.png")
        Image.fromarray(rng.integers(0, 256, (H, W, 3), dtype=np.uint8)).save(tmp_path / names[-1])
    (tmp_path / "list.txt").write_text("\n".join(names) + "\n")
    ex.extract_features(str(tmp_path / "list.txt"), str(tmp_path), "dino_vits16", 3, str(tmp_path / "f"), seed=0,
                        yes=True, writer="thread", precision=precision)
    for i, name in enumerate(names):
        f = torch.load(tmp_path / "f" / f"im{i}.pth", weights_only=False)
        im = torch.from_numpy(np.asarray(Image.open(tmp_path / name).convert("RGB")).copy()).cuda()
        assert torch.equal(f["k"], model.forward_k(im[None]).cpu()), name
        assert f["shape"] == (1, 3, *shapes[i]) and int(f["indices"]) == i

    boxes = {"im0": [(0, 0, 160, 112), (10, 20, 26, 36), (0, 0, 500, 375)],
             "im4": [(5, 5, 229, 229), (0, 0, 232, 224), (33, 1, 65, 49)]}
    bbox_list = []
    for name, bb in boxes.items():
        Image.open(tmp_path / f"{name}.png").convert("RGB").save(tmp_path / f"{name}.jpg", quality=95)
        bbox_list.append({"id": name, "bboxes": bb, "bboxes_original_resolution": bb})
    torch.save(bbox_list, tmp_path / "boxes.pth")
    ex.extract_bbox_features(str(tmp_path), str(tmp_path / "boxes.pth"), "dino_vits16", str(tmp_path / "o.pth"), seed=0,
                             batch_size=4, precision=precision)
    for d in torch.load(tmp_path / "o.pth", weights_only=False):
        image = torch.from_numpy(np.asarray(Image.open(tmp_path / f"{d['id']}.jpg").convert("RGB")).copy())
        want = [model.forward_cls(image[ymin:ymax, xmin:xmax].contiguous().cuda()[None])[0].cpu()
                for xmin, ymin, xmax, ymax in d["bboxes_original_resolution"]]
        assert torch.equal(d["features"], torch.stack(want)), d["id"]
