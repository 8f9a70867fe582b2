"""CPU: the ragged ViT forwards (dss_vit_forward_k_ragged / _cls_ragged) without a device. Argument validation happens
on the host before any device work, so an unloaded handle and never-dereferenced pointers are enough; the workspace
query, the host packing and row ranges, the writer's row-range items, and the batching of extract_features and
extract_bbox_features (a fake model counts the forwards) need no GPU either."""
import ctypes as C

import numpy as np
import pytest
import torch

from conftest import load_pkg

FAKE = 1 << 20   # a 256-byte-aligned address that is never dereferenced: validation fails first


@pytest.fixture
def handle():
    L, vit = load_pkg("_lib"), load_pkg("vit")
    lib = L.load()
    P, d, depth, heads = vit.arch("dino_vits16")
    cfg = L.VitConfig(P, d, depth, heads, vit.MLP_RATIO, vit.TRAIN_IMG // P, vit.LN_EPS)
    h = C.c_void_p()
    assert lib.dss_vit_create(C.byref(cfg), C.byref(h)) == 0
    yield lib, h
    lib.dss_vit_destroy(h)


def _dims(shapes):
    return (C.c_int * (2 * len(shapes)))(*[v for hw in shapes for v in hw])


def _k(lib, h, img, dims, B, out=FAKE, ws=FAKE, ws_bytes=1 << 40):
    return lib.dss_vit_forward_k_ragged(h, img, dims, B, -1, out, ws, ws_bytes, None)


def _cls(lib, h, img, dims, B, out=FAKE, ws=FAKE, ws_bytes=1 << 40):
    return lib.dss_vit_forward_cls_ragged(h, img, dims, B, out, ws, ws_bytes, None)


@pytest.mark.parametrize("call", [_k, _cls])
def test_argument_validation(handle, call):
    lib, h = handle
    ok = _dims([(224, 224), (37, 50)])

    def refused(msg, *a, **kw):
        assert call(lib, h, *a, **kw) == -1
        assert msg in lib.dss_last_error(), lib.dss_last_error()

    refused(b"null pointer", None, ok, 2)
    refused(b"null pointer", FAKE, ok, 2, out=None)
    refused(b"null pointer", FAKE, None, 2)
    refused(b"B must be positive", FAKE, ok, 0)
    refused(b"B must be positive", FAKE, ok, -3)
    refused(b"image 1 has negative size", FAKE, _dims([(32, 32), (-16, 32)]), 2)
    refused(b"image 2 (15x64) is smaller than one 16-pixel patch", FAKE, _dims([(32, 32), (16, 16), (15, 64)]), 3)
    refused(b"image 0 (64x8)", FAKE, _dims([(64, 8)]), 1)
    refused(b"null workspace", FAKE, ok, 2, ws=None)
    refused(b"256-byte aligned", FAKE, ok, 2, ws=FAKE + 16)
    need = lib.dss_vit_ragged_workspace_bytes(h, ok, 2, 0)
    refused(b"workspace too small", FAKE, ok, 2, ws_bytes=need - 1)
    # every argument right: the unloaded handle is refused, still before any device work
    refused(b"weights not loaded", FAKE, ok, 2, ws_bytes=need)
    assert lib.dss_vit_forward_k_ragged(None, FAKE, ok, 2, -1, FAKE, FAKE, need, None) == -1
    assert lib.dss_vit_forward_k_ragged(h, FAKE, ok, 2, 12, FAKE, FAKE, need, None) == -1
    assert b"which_block 12 out of range" in lib.dss_last_error()


def test_token_rows_past_the_tensor_map_extents_are_unsupported(handle):
    lib, h = handle
    big = 16 * 46341    # 46341^2 + 1 token rows > 2^31
    dims = _dims([(32, 32), (big, big)])
    assert lib.dss_vit_ragged_workspace_bytes(h, dims, 2, 0) == 0
    assert _k(lib, h, FAKE, dims, 2) == -4
    assert b"tensor-map extents" in lib.dss_last_error()
    assert _cls(lib, h, FAKE, dims, 2) == -4


def test_workspace_query(handle):
    lib, h = handle
    L = load_pkg("_lib")
    ws = lambda shapes, mode=0: lib.dss_vit_ragged_workspace_bytes(h, _dims(shapes), len(shapes), mode)
    base = [(224, 224), (375, 500), (16, 16)]
    w0 = ws(base)
    assert w0 > 0 and w0 % 1024 == 0
    # more images, or a larger image, never need less
    assert ws(base + [(16, 16)]) > w0
    assert ws(base + [(480, 480)]) > ws(base + [(16, 16)])
    assert ws([(224, 224), (375, 516), (16, 16)]) >= w0
    assert ws([(224, 240), (375, 500), (16, 16)]) >= w0
    prev = 0
    for n in range(1, 40):
        cur = ws([(16 * (1 + i % 7), 16 * (1 + i % 5)) for i in range(n)])
        assert cur > prev
        prev = cur
    # pixels past the patch multiples change nothing but the input
    assert ws([(239, 239), (383, 511), (31, 31)]) == w0
    # both modes lay the workspace out the same; a bad mode, B or image is 0
    assert ws(base, L.VIT_RAGGED_CLS) == w0
    assert ws(base, 2) == 0 and ws(base, -1) == 0
    assert ws([(224, 224), (8, 224)]) == 0
    assert lib.dss_vit_ragged_workspace_bytes(h, None, 2, 0) == 0
    assert lib.dss_vit_ragged_workspace_bytes(h, _dims(base), 0, 0) == 0
    # at least the uniform call's workspace for the same images; the fp32 mode needs more
    assert ws([(480, 480)] * 4) >= lib.dss_vit_workspace_bytes(h, 4, 480, 480)

    def one_image_tables():
        # both batch kinds carve the same buffers, positional table included: one image needs the uniform call's
        # workspace and the ragged tables (RaggedImage, tile prefix, patch -> token and token -> feature rows)
        for H, W in [(16, 16), (224, 224), (375, 500), (480, 480)]:
            T = (H // 16) * (W // 16) + 1
            extra = ws([(H, W)]) - lib.dss_vit_workspace_bytes(h, 1, H, W)
            assert extra % 1024 == 0 and 8 * T <= extra < 8 * T + 2048, (H, W, extra)

    one_image_tables()
    assert lib.dss_vit_set_precision(h, L.VIT_PRECISION["fp32"]) == 0
    assert ws(base) > w0
    one_image_tables()


def test_pack_images_and_row_ranges():
    vit = load_pkg("vit")
    L = load_pkg("_lib")
    g = torch.Generator().manual_seed(0)
    shapes = [(16, 16), (37, 50), (224, 224), (33, 17)]
    ims = [torch.randint(0, 256, (H, W, 3), dtype=torch.uint8, generator=g) for H, W in shapes]
    packed, dims = vit.pack_images(ims)
    assert dims.dtype == torch.int32 and dims.tolist() == [list(s) for s in shapes]
    assert packed.shape == (sum(H * W for H, W in shapes), 3) and packed.is_contiguous()
    off = 0
    for im, (H, W) in zip(ims, shapes):   # image b at pixel offset sum_{i<b} H_i W_i
        assert torch.equal(packed[off:off + H * W].reshape(H, W, 3), im)
        off += H * W
    rows = vit.ragged_rows(dims.tolist(), 16)
    assert rows == [(0, 1), (1, 7), (7, 203), (203, 205)]
    assert vit.ragged_rows([(15 + 16 * 4, 8 * 16)], 8) == [(0, 9 * 16)]
    with pytest.raises(L.DssError):
        vit.pack_images([])
    with pytest.raises(L.DssError):
        vit.pack_images([torch.zeros(4, 4, 3, dtype=torch.float32)])


def test_writer_rows_items_split_over_processes():
    """The process writer sends each process the array rows its items read: a ragged item spans n rows."""
    iop = load_pkg("io_pipeline")
    k = np.arange(10 * 2, dtype=np.float32).reshape(10, 2)
    spans = [(0, 1), (1, 7), (7, 10)]
    items = [(f"f{i}", r0, {}, {"k": ("rows1", ("k", r1 - r0))}) for i, (r0, r1) in enumerate(spans)]
    assert [iop._row_end(it) for it in items] == [1, 7, 10]
    assert iop._row_end(("p", 3, {}, {"k": ("slice", "k")})) == 4

    class Q:
        def __init__(self):
            self.msgs = []

        def put(self, m):
            self.msgs.append(m)

    w = iop.ProcessWriter.__new__(iop.ProcessWriter)
    w.procs, w.q, w.submitted = [None, None], Q(), 0
    w._check = lambda: None
    w.submit_batch({"k": k}, items)
    got = {}
    for arrays, part in w.q.msgs:
        for path, j, extra, fields in part:
            got[path] = iop._materialise(arrays, j, extra, fields)["k"]
    for i, (r0, r1) in enumerate(spans):
        assert got[f"f{i}"].shape == (1, r1 - r0, 2)
        assert torch.equal(got[f"f{i}"], torch.from_numpy(k[r0:r1]).unsqueeze(0))


class _FakeModel:
    """Stands in for DinoViT: records each ragged forward; an image's outputs are a function of that image alone."""
    P, d = 16, 4

    def __init__(self):
        self.calls = []

    @staticmethod
    def _unpack(packed, dims):
        out, off = [], 0
        for H, W in dims.tolist():
            out.append(packed[off:off + H * W].reshape(H, W, 3))
            off += H * W
        assert off == packed.shape[0]
        return out

    @classmethod
    def k_of(cls, im):
        n = (im.shape[0] // cls.P) * (im.shape[1] // cls.P)
        return float(im.double().sum()) + torch.arange(n * cls.d, dtype=torch.float32).reshape(n, cls.d)

    def forward_k_ragged(self, packed, dims, which_block=-1):
        ims = self._unpack(packed, dims)
        self.calls.append([tuple(im.shape[:2]) for im in ims])
        vit = load_pkg("vit")
        return torch.cat([self.k_of(im) for im in ims]), vit.ragged_rows(dims.tolist(), self.P)

    def forward_cls_ragged(self, packed, dims):
        ims = self._unpack(packed, dims)
        self.calls.append([tuple(im.shape[:2]) for im in ims])
        cls = torch.stack([torch.full((self.d,), float(im.double().sum()) + im.shape[0] * 1000 + im.shape[1])
                           for im in ims])
        return cls, [(b, b + 1) for b in range(len(ims))]


class _CpuRing:
    """PackedRing without page-locked memory (no device here): the same packing, the same interface."""

    def __init__(self, device, slots=2, copy_threads=8):
        pass

    def stage(self, images):
        packed, dims = load_pkg("vit").pack_images(list(images))
        return 0, packed, dims

    def to_device(self, slot, host):
        return host


def _fake(monkeypatch):
    ex = load_pkg("extract")
    model = _FakeModel()
    monkeypatch.setattr(ex, "_device", lambda: torch.device("cpu"))
    monkeypatch.setattr(ex.utils, "get_model", lambda *a, **k: (model, None, _FakeModel.P, 6))
    monkeypatch.setattr(ex.io_pipeline, "PackedRing", _CpuRing)
    return ex, model


def test_extract_features_batches_across_shapes(tmp_path, monkeypatch):
    from PIL import Image
    ex, model = _fake(monkeypatch)
    rng = np.random.default_rng(0)
    shapes = [(32, 48), (17, 16), (64, 64), (40, 33), (16, 80), (48, 32), (33, 33)]
    names = []
    for i, (H, W) in enumerate(shapes):
        names.append(f"im{i}.png")
        Image.fromarray(rng.integers(0, 256, (H, W, 3), dtype=np.uint8)).save(tmp_path / names[-1])
    (tmp_path / "list.txt").write_text("\n".join(names) + "\n")
    out = tmp_path / "features"
    ex.extract_features(str(tmp_path / "list.txt"), str(tmp_path), "dino_vits16", 3, str(out), seed=0, yes=True,
                        num_workers=0, writer="thread")
    # seven images of seven sizes: batches of 3, 3 and 1 in list order
    assert model.calls == [shapes[0:3], shapes[3:6], shapes[6:7]]
    for i, (H, W) in enumerate(shapes):
        f = torch.load(out / f"im{i}.pth", weights_only=False)
        im = torch.from_numpy(np.asarray(Image.open(tmp_path / names[i]).convert("RGB")).copy())
        assert f["k"].shape == (1, (H // 16) * (W // 16), 4)
        assert torch.equal(f["k"], _FakeModel.k_of(im).unsqueeze(0))
        assert f["shape"] == (1, 3, H, W) and int(f["indices"]) == i and f["id"] == f"im{i}"
        assert f["file"] == names[i] and f["model_name"] == "dino_vits16" and f["patch_size"] == 16
    # existing files are skipped: a second run does no forward
    model.calls.clear()
    ex.extract_features(str(tmp_path / "list.txt"), str(tmp_path), "dino_vits16", 3, str(out), seed=0, yes=True,
                        num_workers=0, writer="thread")
    assert model.calls == []


def test_extract_bbox_features_batches_across_shapes(tmp_path, monkeypatch):
    from PIL import Image
    ex, model = _fake(monkeypatch)
    rng = np.random.default_rng(1)
    boxes = {"a": [(0, 0, 32, 48), (5, 3, 21, 19), (0, 0, 64, 64)], "b": [(1, 2, 50, 30), (10, 10, 26, 26)]}
    bbox_list = []
    for name, bb in boxes.items():
        Image.fromarray(rng.integers(0, 256, (70, 80, 3), dtype=np.uint8)).save(tmp_path / f"{name}.jpg", quality=95)
        bbox_list.append({"id": name, "bboxes": bb, "bboxes_original_resolution": bb})
    torch.save(bbox_list, tmp_path / "boxes.pth")
    ex.extract_bbox_features(str(tmp_path), str(tmp_path / "boxes.pth"), "dino_vits16", str(tmp_path / "out.pth"),
                             seed=0, batch_size=2)
    sizes = [(ymax - ymin, xmax - xmin) for bb in boxes.values() for xmin, ymin, xmax, ymax in bb]
    assert model.calls == [sizes[0:2], sizes[2:4], sizes[4:5]]   # (image, box) order, two crops per forward
    got = torch.load(tmp_path / "out.pth", weights_only=False)
    for d in got:
        image = torch.from_numpy(np.asarray(Image.open(tmp_path / f"{d['id']}.jpg").convert("RGB")).copy())
        want = []
        for xmin, ymin, xmax, ymax in d["bboxes_original_resolution"]:
            crop = image[ymin:ymax, xmin:xmax]
            want.append(torch.full((4,), float(crop.double().sum()) + crop.shape[0] * 1000 + crop.shape[1]))
        assert torch.equal(d["features"], torch.stack(want))
