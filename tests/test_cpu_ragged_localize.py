"""CPU: ragged object localization without a device. dss_vit_forward_last_ragged and the ragged LOST / DINO-seg entry
points check every argument on the host before any device work, so an unloaded handle and never-dereferenced pointers
are enough; the workspace query of the padded grid, and the list-order batching of the command (a fake model and fake
box kernels), need no GPU either."""
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


def _ints(rows):
    return (C.c_int * sum(len(r) for r in rows))(*[v for r in rows for v in r])


def _last(lib, h, dims, B, img=FAKE, pad=1, which=1, feats=FAKE, n_max=196, attn=FAKE, ws=FAKE, ws_bytes=1 << 40):
    return lib.dss_vit_forward_last_ragged(h, img, dims, B, pad, which, feats, n_max, attn, ws, ws_bytes, None)


def test_forward_last_ragged_refusals(handle):
    lib, h = handle
    L = load_pkg("_lib")
    ok = _ints([(224, 224), (7, 50)])   # 14 x 14 and 1 x 4 padded grids

    def refused(msg, *a, code=-1, **kw):
        assert _last(lib, h, *a, **kw) == code
        assert msg in lib.dss_last_error(), lib.dss_last_error()

    assert lib.dss_vit_forward_last_ragged(None, FAKE, ok, 2, 1, 1, FAKE, 196, FAKE, FAKE, 1 << 40, None) == -1
    refused(b"pad must be 0 or 1", ok, 2, pad=2)
    refused(b"which must be 0 (q), 1 (k) or 2 (v)", ok, 2, which=3)
    refused(b"null pointer", ok, 2, img=None)
    refused(b"null pointer", ok, 2, feats=None, attn=None)
    refused(b"null pointer", None, 2)
    refused(b"n_max must be positive", ok, 2, n_max=0)
    refused(b"B must be positive", ok, 0)
    refused(b"image 1 has negative size", _ints([(32, 32), (-1, 32)]), 2)
    refused(b"image 1 (0x32) has no pixels", _ints([(32, 32), (0, 32)]), 2)
    # the crop refuses an image smaller than one patch, the padded grid takes it
    refused(b"image 1 (7x50) is smaller than one 16-pixel patch", ok, 2, pad=0)
    refused(b"image 0 (224x224) has 196 patches, more than n_max = 195", ok, 2, n_max=195)
    refused(b"image 0 (224x224) has 196 patches", ok, 2, pad=0, n_max=195)
    refused(b"exceed one grid column", _ints([(16, 16)] * 65536), 65536)
    refused(b"do not fit", _ints([(16, 16)] * 3), 3, n_max=1 << 30, code=-4)
    refused(b"null workspace", ok, 2, n_max=196, ws=None)
    refused(b"256-byte aligned", ok, 2, n_max=196, ws=FAKE + 16)
    need = lib.dss_vit_ragged_workspace_bytes(h, ok, 2, L.VIT_RAGGED_PAD)
    assert need > 0
    refused(b"workspace too small", ok, 2, n_max=196, ws_bytes=need - 1)
    # every argument right: the unloaded handle is refused, still before any device work
    refused(b"weights not loaded", ok, 2, n_max=196, ws_bytes=need)
    refused(b"weights not loaded", ok, 2, n_max=196, ws_bytes=need, feats=None)
    refused(b"weights not loaded", ok, 2, n_max=196, ws_bytes=need, attn=None)


def test_padded_grid_workspace_query(handle):
    lib, h = handle
    L = load_pkg("_lib")
    ws = lambda shapes, mode: lib.dss_vit_ragged_workspace_bytes(h, _ints(shapes), len(shapes), mode)
    mult = [(224, 224), (384, 512), (16, 16)]
    # on patch multiples the padded grid is the crop
    assert ws(mult, L.VIT_RAGGED_PAD) == ws(mult, L.VIT_RAGGED_K) > 0
    # one more pixel is one more patch row / column
    assert ws([(225, 224), (384, 512), (16, 16)], L.VIT_RAGGED_PAD) > ws(mult, L.VIT_RAGGED_PAD)
    assert ws([(239, 239), (383, 511), (31, 31)], L.VIT_RAGGED_PAD) == ws([(240, 240), (384, 512), (32, 32)],
                                                                           L.VIT_RAGGED_K)
    # images smaller than one patch: the padded grid only
    assert ws([(1, 1), (15, 200)], L.VIT_RAGGED_PAD) > 0
    assert ws([(1, 1), (15, 200)], L.VIT_RAGGED_K) == 0
    assert ws([(0, 5)], L.VIT_RAGGED_PAD) == 0 and ws([(16, 16)], 2) == 0
    # one image: the uniform forward_last workspace plus the ragged tables
    for H, W in [(1, 1), (17, 33), (375, 500)]:
        T = -(-H // 16) * -(-W // 16) + 1
        extra = ws([(H, W)], L.VIT_RAGGED_PAD) - lib.dss_vit_forward_last_workspace_bytes(h, 1, H, W, 1)
        assert extra % 1024 == 0 and 8 * T <= extra < 8 * T + 2048, (H, W, extra)


def test_ragged_box_refusals():
    L = load_pkg("_lib")
    lib = L.load()
    lost_ws = lib.dss_lost_ragged_workspace_bytes(2, 64)
    assert lost_ws >= 2 * 64 * 4 and lib.dss_lost_ragged_workspace_bytes(0, 64) == 0
    assert lib.dss_lost_ragged_workspace_bytes(2, 0) == 0
    din_ws = lib.dss_dinoseg_ragged_workspace_bytes(2)
    assert din_ws > 0 and lib.dss_dinoseg_ragged_workspace_bytes(0) == 0

    def lost(dims, B=2, n_max=64, ldw=64, A=FAKE, ws_bytes=lost_ws, k=100):
        return lib.dss_lost_boxes_ragged(A, B, n_max, ldw, dims, 16, k, FAKE, FAKE, FAKE, FAKE, ws_bytes, None)

    def dinoseg(dims, B=2, n_max=64, head=0, ws_bytes=din_ws, attn=FAKE):
        return lib.dss_dinoseg_boxes_ragged(attn, B, 6, n_max, head, dims, 16, FAKE, FAKE, FAKE, ws_bytes, None)

    def refused(rc, code, msg):
        assert rc == code, (rc, lib.dss_last_error())
        assert msg in lib.dss_last_error(), lib.dss_last_error()

    ok4 = _ints([(8, 8, 120, 128), (2, 3, 20, 40)])
    ok2 = _ints([(8, 8), (2, 3)])
    refused(lost(ok4, A=None), -1, b"null pointer")
    refused(lost(None), -1, b"null pointer")
    refused(lost(ok4, ldw=63), -1, b"bad shape")
    refused(lost(ok4, k=0), -1, b"k_patches")
    refused(lost(_ints([(8, 8, 120, 128), (9, 8, 130, 128)])), -1, b"image 1's 9x8 grid has more than n_max = 64")
    refused(lost(_ints([(8, 8, 120, 128), (2, 3, 0, 40)])), -1, b"image 1 has grid 2x3, size 0x40")
    refused(lost(_ints([(0, 8, 1, 128), (2, 3, 20, 40)])), -1, b"image 0 has grid 0x8")
    big = _ints([(1, 1, 16, 16), (129, 128, 2064, 2048)])
    refused(lost(big, n_max=129 * 128, ldw=129 * 128, ws_bytes=1 << 40), -4, b"image 1's 16512 cells exceed")
    refused(lost(ok4, ws_bytes=lost_ws - 1), -3, b"workspace too small")
    refused(dinoseg(ok2, attn=None), -1, b"null pointer")
    refused(dinoseg(ok2, head=6), -1, b"head 6 not in [0, 6)")
    refused(dinoseg(_ints([(8, 8), (8, 9)])), -1, b"image 1's 8x9 grid")
    refused(dinoseg(_ints([(1, 1), (129, 128)]), n_max=129 * 128, ws_bytes=1 << 40), -4, b"image 1's 16512 cells")
    refused(dinoseg(ok2, ws_bytes=din_ws - 1), -3, b"workspace too small")


def test_ragged_grids():
    vit = load_pkg("vit")
    dims = [(1, 1), (16, 16), (17, 15), (375, 500)]
    assert vit.ragged_grids(dims, 16, True) == [(1, 1, 1), (1, 1, 1), (2, 2, 1), (24 * 32, 24, 32)]
    assert vit.ragged_grids(dims, 16, False) == [(0, 0, 0), (1, 1, 1), (0, 1, 0), (23 * 31, 23, 31)]


# ------------------------------------------------------------------------------------------------ the command's batching
class _Item:
    def __init__(self, name, shape):
        self.name, self.path, self.gt, self.shape = name, None, None, shape


def _image(it):
    H, W = it.shape
    g = np.random.default_rng(int(it.name[2:]))
    return g.integers(0, 256, (H, W, 3), dtype=np.uint8)


def test_list_batches_keep_order_and_bound_pending_images():
    loc = load_pkg("localize")
    shapes = [(30 + 7 * (i % 5), 40 + 3 * (i % 3)) for i in range(23)]
    items = [_Item(f"im{i}", s) for i, s in enumerate(shapes)]
    loaded = []

    def load(it):
        loaded.append(it.name)
        return _image(it)

    got = []
    for k, (idx, imgs) in enumerate(loc._list_batches(items, 4, load, ahead=2)):
        assert idx == list(range(4 * k, min(4 * k + 4, 23)))
        assert [im.shape[:2] for im in imgs] == [shapes[j] for j in idx]
        for j, im in zip(idx, imgs):
            assert np.array_equal(im, _image(items[j]))
        # decoded or queued: this batch and at most two more
        assert len(loaded) <= 4 * (k + 3)
        got += idx
    assert got == list(range(23)) and sorted(loaded) == sorted(it.name for it in items)


class _FakeModel:
    """Records the ragged forwards the command makes; the features carry nothing but their shapes."""
    patch_size, num_heads, device = 16, 6, torch.device("cpu")

    def __init__(self):
        self.calls = []

    def forward_last_ragged(self, x, dims, which="k", pad=True, feats=True, cls_attn=False):
        vit = load_pkg("vit")
        grids = vit.ragged_grids(dims.tolist(), 16, pad)
        self.calls.append((x.clone(), dims.tolist(), which, pad, feats, cls_attn))
        n = max(g[0] for g in grids)
        f = torch.zeros(len(grids), n, 8) if feats else None
        a = torch.zeros(len(grids), 6, n) if cls_attn else None
        return f, a, grids


class _HostRing:
    """PackedRing's packing in pageable memory, without the device copy."""
    def __init__(self, device):
        pass

    def stage(self, images):
        dims = torch.tensor([[int(im.shape[0]), int(im.shape[1])] for im in images], dtype=torch.int32)
        return 0, torch.cat([torch.from_numpy(np.array(im)).reshape(-1, 3) for im in images]), dims

    def to_device(self, slot, host_batch):
        return host_batch


@pytest.mark.parametrize("method", ["lost", "dinoseg"])
@pytest.mark.parametrize("batch_size", [1, 3, 64])
def test_command_batches_in_list_order(monkeypatch, method, batch_size):
    loc = load_pkg("localize")
    shapes = [(1 + 37 * i % 500, 1 + 53 * i % 500) for i in range(1, 12)]
    items = [_Item(f"im{i}", s) for i, s in enumerate(shapes)]
    boxes_calls = []

    def fake_lost(feats, grids, sizes, P, k):
        boxes_calls.append((list(grids), [tuple(s) for s in sizes]))
        B = len(grids)
        return np.array([[g[0], g[1], s[0], s[1]] for g, s in zip(grids, sizes)]), np.zeros(B), np.zeros(B, np.int32)

    def fake_dinoseg(attn, grids, P, head):
        boxes_calls.append((list(grids), None))
        return np.array([[g[0], g[1], head, 0] for g in grids]), np.zeros(len(grids), np.int32)

    monkeypatch.setattr(loc, "lost_boxes_ragged", fake_lost)
    monkeypatch.setattr(loc, "dinoseg_boxes_ragged", fake_dinoseg)
    monkeypatch.setattr(loc.io_pipeline, "PackedRing", _HostRing)
    args = loc.parse_args(["--batch_size", str(batch_size), "--which_features", "q"]
                          + (["--dinoseg", "--dinoseg_head", "2"] if method == "dinoseg" else []))
    model = _FakeModel()
    preds = loc._from_images_ragged(args, items, model, load=_image)
    n_batches = -(-len(items) // batch_size)
    assert len(model.calls) == n_batches == len(boxes_calls)
    seen = []
    for k, (x, dims, which, pad, feats, cls_attn) in enumerate(model.calls):
        idx = list(range(k * batch_size, min((k + 1) * batch_size, len(items))))
        assert dims == [list(shapes[j]) for j in idx] and pad
        assert torch.equal(x, torch.cat([torch.from_numpy(_image(items[j])).reshape(-1, 3) for j in idx]))
        assert (which, feats, cls_attn) == (("k", False, True) if method == "dinoseg" else ("q", True, False))
        grids = [(-(-shapes[j][0] // 16), -(-shapes[j][1] // 16)) for j in idx]
        assert boxes_calls[k][0] == grids
        if method == "lost":
            assert boxes_calls[k][1] == [shapes[j] for j in idx]
        seen += idx
    assert seen == list(range(len(items)))
    for j, it in enumerate(items):
        gh, gw = -(-shapes[j][0] // 16), -(-shapes[j][1] // 16)
        want = [gh, gw, shapes[j][0], shapes[j][1]] if method == "lost" else [gh, gw, 2, 0]
        assert preds[it.name].tolist() == want


def test_command_raises_for_the_first_failing_image_in_list_order(monkeypatch):
    loc = load_pkg("localize")
    L = load_pkg("_lib")
    items = [_Item(f"im{i}", (20 + i, 30)) for i in range(7)]

    def fake_lost(feats, grids, sizes, P, k):
        st = np.array([L.LOC_SEED_IN_BACKGROUND if s[0] in (23, 25) else L.LOC_OK for s in sizes], np.int32)
        return np.zeros((len(grids), 4), np.int64), np.zeros(len(grids)), st

    monkeypatch.setattr(loc, "lost_boxes_ragged", fake_lost)
    monkeypatch.setattr(loc.io_pipeline, "PackedRing", _HostRing)
    args = loc.parse_args(["--batch_size", "4"])
    model = _FakeModel()
    with pytest.raises(ValueError, match="seed is in the background"):
        loc._from_images_ragged(args, items, model, load=_image)
    assert len(model.calls) == 1   # image 3 fails in the first batch: nothing after it runs
