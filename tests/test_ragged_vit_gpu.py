"""-m gpu: ragged ViT batches (images of different sizes in one forward) bit for bit with the uniform calls.

Every image's rows from dss_vit_forward_k_ragged / _cls_ragged must be torch.equal to the same image run alone through
forward_k / forward_cls, in both precision modes: one-patch and 2 x 2 crops (T = 2, 5), T = 128 and 129 (one row either
side of a 128-query attention tile), VOC shapes (T = 714), 480^2 (T = 901), ViT-B/8 at 480^2 (T = 3601) next to a T = 2
crop, a grid0 x grid0 grid from non-square pixels next to a square 224^2 image (the identity rule per image), which_block
other than -1 and a 264-image batch. Also: rows past the outputs are not written, the device positional tables are
dss_pos_embed_interp_host's bits for every grid up to 64 x 64, the handle's positional cache is untouched, and
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


def test_positional_tables_match_the_host_routine(cuda):
    """Every grid up to 64 x 64 (ViT-S/16, grid0 14) against dss_pos_embed_interp_host, bit for bit: K mode (the
    identity rule by patch grid). The 14 x 14 grid of a 224 x 232 image in CLS mode is resampled, not the stored grid."""
    model = _model()
    lib = load_pkg("_lib").load()
    vit = load_pkg("vit")
    sd = vit.random_state_dict("dino_vits16", 0)
    src = sd["pos_embed"].reshape(-1, model.dim).contiguous()
    grids = [(a, b) for a in range(1, 65) for b in range(1, 65)]
    st = torch.cuda.current_stream().cuda_stream

    def host(g):
        out = torch.empty(g[0] * g[1] + 1, model.dim)
        assert lib.dss_pos_embed_interp_host(src.data_ptr(), 14, model.dim, g[0], g[1], out.data_ptr()) == 0
        return out

    with ThreadPoolExecutor(8) as pool:
        for c0 in range(0, len(grids), 256):
            chunk = grids[c0:c0 + 256]
            want = list(pool.map(host, chunk))
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
        assert torch.equal(got[0], src[0])


def test_positional_cache_untouched(cuda):
    vit = load_pkg("vit")
    lib = load_pkg("_lib").load()
    model = vit.DinoViT("dino_vits16", vit.random_state_dict("dino_vits16", 0), device="cuda")
    assert lib.dss_vit_pos_cache_entries(model._h) == 0
    shapes = [(16 * (1 + i % 9), 16 * (1 + i % 11)) for i in range(80)]
    model.forward_k_ragged(_images(shapes))
    model.forward_cls_ragged(_images(shapes))
    assert lib.dss_vit_pos_cache_entries(model._h) == 0
    model.forward_k(_images([(64, 48)])[0][None])
    assert lib.dss_vit_pos_cache_entries(model._h) == 1
    model.forward_k_ragged(_images([(96, 96), (64, 48)]))
    assert lib.dss_vit_pos_cache_entries(model._h) == 1


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
