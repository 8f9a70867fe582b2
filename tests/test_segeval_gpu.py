"""GPU suite for the segmentation evaluation (csrc/segeval.cu): counts bit for bit against the numpy oracle on ragged
batches of VOC shapes in every resize and crop mode, batch invariance, 64-bit carry, unsupported inputs, and both
commands reproducing the reference's printed lines on the fixture trees."""
import io

import numpy as np
import pytest
import torch

from conftest import ROOT, load_pkg
from oracle import segeval_ref
from oracle.make_segeval_golden import ROOT_MARK, build_tree

pytestmark = pytest.mark.gpu
GOLD = ROOT / "tests" / "golden"
SHAPES = segeval_ref.VOC_SHAPES + [(47, 61), (16, 16), (17, 300)]


def _semantic_items(rng, n):
    """(prediction, target, Gather, oracle's resized prediction) over every _resize_pseudolabel rule and identity."""
    se = load_pkg("segeval")
    items = []
    for i in range(n):
        H, W = SHAPES[i % len(SHAPES)]
        rule = i % 5
        ph, pw = [(H // 16, W // 16), (H // 8, W // 8), (2 * (H // 16), 2 * (W // 16)), (H, W),
                  (H // 16, W // 16 + 5)][rule]
        t = rng.integers(0, 23, (H, W)).astype(np.uint8)
        t[rng.random((H, W)) < 0.2] = 255
        t[rng.random((H, W)) < 0.02] = 200
        p = np.where(rng.random((ph, pw)) < 0.6, 0, rng.integers(0, 256, (ph, pw))).astype(np.uint8)  # background-heavy
        want = segeval_ref.resize_pseudolabel(p, H, W)
        items.append((p, t, se.semantic_gather(p.shape, (H, W), want.shape), want))
    return items


def _oracle_counts(items, n_classes):
    return segeval_ref.semantic_counts([(w, t) for _, t, _, w in items], n_classes)


@pytest.mark.parametrize("n_classes", [21, 1, 63])
def test_semantic_counts_exact_and_batch_invariant(cuda, n_classes):
    se = load_pkg("segeval")
    items = _semantic_items(np.random.default_rng(n_classes), 24)
    got = se.semantic_counts([it[:3] for it in items], n_classes, device=cuda).cpu().numpy()
    assert np.array_equal(got, _oracle_counts(items, n_classes))
    for it in items[:6]:
        solo = se.semantic_counts([it[:3]], n_classes, device=cuda).cpu().numpy()
        assert np.array_equal(solo, _oracle_counts([it], n_classes))


def test_semantic_counts_carry_past_2_32(cuda):
    se = load_pkg("segeval")
    items = _semantic_items(np.random.default_rng(7), 11)
    start = np.full((256, 22), 2 ** 32 - 3, dtype=np.int64)
    counts = torch.from_numpy(start.copy()).to(cuda)
    se.semantic_counts([it[:3] for it in items], 21, counts)
    se.semantic_counts([it[:3] for it in items], 21, counts)
    assert np.array_equal(counts.cpu().numpy(), start + 2 * _oracle_counts(items, 21))


@pytest.mark.parametrize("ds", [16, 8, None])
@pytest.mark.parametrize("crop", [False, True])
def test_object_counts_exact_and_batch_invariant(cuda, ds, crop):
    se = load_pkg("segeval")
    rng = np.random.default_rng(0 if ds is None else ds)
    items, want = [], []
    for i in range(20):
        H, W = SHAPES[i % len(SHAPES)]
        plane = rng.choice(np.array([0, 127, 128, 255], dtype=np.uint8), (H, W))
        p = (rng.random((H, W) if ds is None else (H // ds, W // ds)) < 0.5).astype(np.uint8)
        g = se.object_gather(p.shape, plane.shape, ds, crop)
        items.append((p, plane, g))
        want.append(segeval_ref.object_counts(*segeval_ref.object_prepare(p, plane, ds, crop)))
    got = se.object_counts(items, device=cuda)
    assert np.array_equal(got, np.stack(want))
    for j in (0, 7, 19):
        assert np.array_equal(se.object_counts([items[j]], device=cuda)[0], got[j])


def test_unsupported_inputs_are_rejected(cuda):
    se = load_pkg("segeval")
    _lib = load_pkg("_lib")
    lib = _lib.load()
    p = torch.zeros(4 * 4, dtype=torch.uint8, device=cuda)
    t = torch.zeros(8 * 8, dtype=torch.uint8, device=cuda)
    counts = torch.zeros(256 * 65 + 8, dtype=torch.int64, device=cuda)
    ws = torch.empty(1 << 16, dtype=torch.uint8, device=cuda)

    def call(desc, table, mode, num_classes):
        d = np.ascontiguousarray(desc, dtype=np.int64)
        tb = np.ascontiguousarray(table, dtype=np.int32)
        return lib.dss_segeval_counts(p.data_ptr(), p.numel(), t.data_ptr(), t.numel(), d.ctypes.data, 1,
                                      tb.ctypes.data, tb.size, mode, num_classes, counts.data_ptr(), ws.data_ptr(),
                                      ws.numel(), _lib.stream_ptr(cuda))
    g = se.Gather(0, 0, *[np.arange(8) // 2] * 4)                                     # a 4 x 4 map doubled
    ok = [0, 4, 4, 0, 8, 8, 0, 0, 8, 8, 0, 0, 0]
    table = g.table()
    assert call(ok, table, _lib.SEGEVAL_SEMANTIC, 21) == 0
    assert call(ok, table, _lib.SEGEVAL_SEMANTIC, 64) == _lib.DSS_ERR_UNSUPPORTED   # 65 target bins
    bad = table.copy()
    bad[3] = 4                                                                         # row 4 of a 4-row map
    assert call(ok, bad, _lib.SEGEVAL_SEMANTIC, 21) == _lib.DSS_ERR_UNSUPPORTED
    bad = table.copy()
    bad[-1] = -1
    assert call(ok, bad, _lib.SEGEVAL_BINARY, 0) == _lib.DSS_ERR_UNSUPPORTED
    crop = list(ok)
    crop[6] = 1                                                                        # rows 1 .. 8 of an 8-row target
    assert call(crop, table, _lib.SEGEVAL_BINARY, 0) == _lib.DSS_ERR_UNSUPPORTED
    off = list(ok)
    off[0] = 1                                                                         # prediction past its buffer
    assert call(off, table, _lib.SEGEVAL_BINARY, 0) == _lib.DSS_ERR_UNSUPPORTED
    torch.cuda.synchronize()


@pytest.mark.parametrize("tag", ["hungarian", "majority"])
def test_semantic_command_reproduces_reference_output(cuda, tag, tmp_path):
    se = load_pkg("segeval")
    z = np.load(GOLD / f"ref_semeval_{tag}.npz")
    build_tree(z, tmp_path)
    sub = lambda s: str(s).replace(ROOT_MARK, str(tmp_path))   # noqa: E731
    out = io.StringIO()
    stats, match = se.semantic_main([f"segments_dir={sub(z['segments_dir'])}", f"data.val_kwargs.root={sub(z['root'])}",
                                     f"n_clusters={int(z['n_clusters'])}"], out=out)
    assert out.getvalue() == "".join(sub(x) + "\n" for x in z["lines"])
    assert stats["jaccards_all_categs"] == z["jac"].tolist() and stats["mIoU"] == z["miou"]


@pytest.mark.parametrize("tag", ["ds16", "ds8", "full"])
def test_object_command_reproduces_reference_output(cuda, tag, tmp_path):
    se = load_pkg("segeval")
    z = np.load(GOLD / f"ref_objseg_{tag}.npz")
    build_tree(z, tmp_path)
    ds = int(z["downsample"])
    out = io.StringIO()
    se.object_main([f"data_root={tmp_path / 'data'}", f"predictions.root={tmp_path / 'preds'}", "predictions.run=run",
                    f"predictions.downsample={'null' if ds < 0 else ds}", "datasets=CUB,ECSSD"], out=out)
    assert out.getvalue() == "".join(x + "\n" for x in z["lines"])


def test_voc_val_sized_command_matches_oracle(cuda, tmp_path):
    """1449 VOC-val-shaped pairs through the file-based command: the same matching and mIoU as the oracle."""
    se = load_pkg("segeval")
    root, seg_dir, M = segeval_ref.synthetic_voc_tree(tmp_path, 1449, seed=3)
    out = io.StringIO()
    stats, match = se.semantic_main([f"segments_dir={seg_dir}", f"data.val_kwargs.root={root}"], out=out)
    want, want_match, lines = segeval_ref.semantic_eval(M, 21, 21)
    assert np.array_equal(np.array(match), np.array(want_match))
    assert stats["jaccards_all_categs"] == want["jaccards_all_categs"] and stats["mIoU"] == want["mIoU"]
    assert out.getvalue().endswith("\n".join(lines) + "\n")
