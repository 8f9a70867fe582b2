"""CPU suite for the segmentation evaluation: the numpy oracle (oracle/segeval_ref.py) and the package's host
arithmetic against the reference's own results (tests/golden/ref_semeval_*.npz, ref_objseg_*.npz), the gather tables
against cv2.resize, and the commands' argument, shape and value-set checks, which all run before any device work."""
import importlib.util
from pathlib import Path

import numpy as np
import pytest
from PIL import Image

from conftest import ROOT, load_pkg
from oracle import segeval_ref
from oracle.make_segeval_golden import ROOT_MARK, build_tree

GOLD = ROOT / "tests" / "golden"
SEM = ["hungarian", "majority"]
OBJ = ["ds16", "ds8", "full"]
OBJ_SETS = {"CUB": ("CUB_200_2011/test_images", "CUB_200_2011/test_segmentations", True),
            "ECSSD": ("ECSSD/images", "ECSSD/ground_truth_mask", False)}


def _sem(tag, tmp_path):
    z = np.load(GOLD / f"ref_semeval_{tag}.npz")
    build_tree(z, tmp_path)
    sub = lambda s: str(s).replace(ROOT_MARK, str(tmp_path))   # noqa: E731
    return z, sub


def _sem_arrays(z, sub):
    """(pseudo-label, target, image (H, W)) of every pair in the reference's order."""
    out = []
    for img, tgt, seg in z["pairs"]:
        with Image.open(sub(img)) as im:
            hw = (im.size[1], im.size[0])
        out.append((np.array(Image.open(sub(seg))), np.array(Image.open(sub(tgt))), hw))
    return out


def _apply(g, pred):
    """The kernel's gather on the host: output (y, x) reads pred[rows[y], cols[x]], the _in halves in the block."""
    inner = pred[np.ix_(g.rows_in, g.cols_in)]
    outer = pred[np.ix_(g.rows_out, g.cols_out)]
    y, x = np.meshgrid(np.arange(g.h), np.arange(g.w), indexing="ij")
    return np.where((y < g.block_h) & (x < g.block_w), inner, outer)


@pytest.mark.parametrize("tag", SEM)
def test_oracle_reproduces_semantic_fixture(tag, tmp_path):
    z, sub = _sem(tag, tmp_path)
    n_clusters, n_classes = int(z["n_clusters"]), int(z["num_classes"]) + 1
    pairs = [(segeval_ref.resize_pseudolabel(p, *hw), t) for p, t, hw in _sem_arrays(z, sub)]
    result, match, lines = segeval_ref.semantic_eval(segeval_ref.confusion(pairs), n_clusters, n_classes)
    assert result["jaccards_all_categs"] == z["jac"].tolist()
    assert result["mIoU"] == z["miou"]
    assert np.array_equal(np.array([[int(a), int(b)] for a, b in match]), z["match"])
    assert "\n".join(lines) == "\n".join(sub(x) for x in z["lines"][5:])   # the reference's text, split by line


@pytest.mark.parametrize("tag", SEM)
def test_package_host_arithmetic_matches_semantic_fixture(tag, tmp_path):
    """voc_pairs, the gather tables, match_clusters and semantic_miou on the oracle's binned counts give the
    reference's lines and numbers exactly."""
    se = load_pkg("segeval")
    z, sub = _sem(tag, tmp_path)
    n_clusters, n_classes = int(z["n_clusters"]), int(z["num_classes"]) + 1
    root = sub(z["root"])
    images, targets, segments, lines = se.voc_pairs(root, "2012", "val", sub(z["segments_dir"]))
    assert lines == [sub(x) for x in z["lines"][:5]]
    assert [list(p) for p in zip(images, targets, segments)] == [[sub(x) for x in p] for p in z["pairs"]]
    pairs = []
    for p, t, hw in _sem_arrays(z, sub):
        g = se.semantic_gather(p.shape, hw, t.shape)
        assert np.array_equal(_apply(g, p), segeval_ref.resize_pseudolabel(p, *hw))
        pairs.append((_apply(g, p), t))
    C = segeval_ref.semantic_counts(pairs, n_classes)
    match = se.match_clusters(C, n_clusters, n_classes)
    stats = se.semantic_miou(C, match, n_classes)
    text = "\n".join(z["lines"].tolist())
    assert f"\nOptimal matching: {match}\nEvaluation of semantic segmentation \n" in text
    assert text.endswith("\n" + str(stats))
    assert stats["jaccards_all_categs"] == z["jac"].tolist() and stats["mIoU"] == z["miou"]


def _obj(tag, tmp_path):
    z = np.load(GOLD / f"ref_objseg_{tag}.npz")
    build_tree(z, tmp_path)
    ds = int(z["downsample"])
    return z, (None if ds < 0 else ds)


@pytest.mark.parametrize("tag", OBJ)
def test_oracle_and_host_arithmetic_reproduce_object_fixture(tag, tmp_path):
    se = load_pkg("segeval")
    z, ds = _obj(tag, tmp_path)
    accs, ious, lines, counts = [], [], [], []
    for name, (img_dir, lab_dir, crop) in OBJ_SETS.items():
        images, labels = se.object_files(str(tmp_path / "data" / img_dir), str(tmp_path / "data" / lab_dir))
        pred_dir = tmp_path / "preds" / img_dir.split("/")[0] / "run"
        a_list, u_list = [], []
        for img, lab in zip(images, labels):
            pred = se.read_prediction(pred_dir / f"{img.stem}.png")
            plane = se.read_mask_plane(lab)
            p, t = segeval_ref.object_prepare(pred, plane, ds, crop)
            g = se.object_gather(pred.shape, plane.shape, ds, crop)
            assert np.array_equal(_apply(g, pred), p)
            tcrop = plane[g.top:g.top + g.h, g.left:g.left + g.w] >= 128
            assert np.array_equal(tcrop, t)
            a, u = segeval_ref.object_image_metrics(p, t)
            a_list.append(a)
            u_list.append(u)
            counts.append(segeval_ref.object_counts(p, t))
        accs += a_list
        ious += u_list
        lines += [f"[{name}] acc: {segeval_ref.mean(a_list)}", f"[{name}] iou: {segeval_ref.mean(u_list)}"]
    assert accs == z["acc"].tolist()
    assert ious == z["iou"].tolist() and [isinstance(u, int) for u in ious] == z["iou_is_int"].tolist()
    assert lines == z["lines"].tolist()
    pa, pu = se.object_metrics(np.stack(counts))
    assert pa == accs and pu == ious and [type(u) for u in pu] == [type(u) for u in ious]


def test_center_crop_offsets_are_torchvision_banker_rounding():
    import torch
    from torchvision.transforms import functional as TF
    se = load_pkg("segeval")
    assert se.center_crop_offsets(75, 70, 70) == (2, 0)    # 5 / 2 -> 2
    assert se.center_crop_offsets(70, 77, 70) == (0, 4)    # 7 / 2 -> 4
    for H in range(20, 40):
        for W in (20, 23, 31):
            S = min(H, W)
            x = torch.arange(H * W).reshape(H, W)
            top, left = se.center_crop_offsets(H, W, S)
            assert torch.equal(TF.center_crop(x, S), x[top:top + S, left:left + S])


def test_gather_tables_equal_cv2_index_maps():
    """Every resize and crop mode on an index map (cell id per prediction cell): the gather reads exactly the cells
    cv2.resize(INTER_NEAREST) and the centre crops pick."""
    se = load_pkg("segeval")
    rng = np.random.default_rng(0)
    for _ in range(300):
        H, W = int(rng.integers(16, 260)), int(rng.integers(16, 260))
        idx = lambda ph, pw: np.arange(ph * pw, dtype=np.int32).reshape(ph, pw)   # noqa: E731
        for ph in {H // 16, H // 8, 2 * (H // 16), H, int(rng.integers(1, 40))}:
            pw = {H // 16: W // 16, H // 8: W // 8}.get(ph, int(rng.integers(1, 40))) or 1
            p = idx(ph, pw)
            want = segeval_ref.resize_pseudolabel(p, H, W)
            g = se.semantic_gather(p.shape, (H, W), want.shape)
            assert np.array_equal(_apply(g, p), want)
        plane = np.zeros((H, W), dtype=np.uint8)
        for crop in (False, True):
            for ds in (16, 8, 14):
                p = idx(max(1, H // ds), max(1, W // ds))
                try:
                    want, _ = segeval_ref.object_prepare(p, plane, ds, crop)
                    want_ok = want.shape == (segeval_ref.center_crop(plane, min(H, W)) if crop else plane).shape
                except Exception:   # noqa: BLE001  (a broadcast failure of the reference's route)
                    want_ok = False
                if want_ok:
                    assert np.array_equal(_apply(se.object_gather(p.shape, (H, W), ds, crop), p), want)
                else:
                    with pytest.raises(ValueError, match="predictions.downsample=null"):
                        se.object_gather(p.shape, (H, W), ds, crop)
            want, _ = segeval_ref.object_prepare(idx(H, W), plane, None, crop)
            assert np.array_equal(_apply(se.object_gather((H, W), (H, W), None, crop), idx(H, W)), want)


def _sem_args(z, sub, *extra):
    return [f"segments_dir={sub(z['segments_dir'])}", f"data.val_kwargs.root={sub(z['root'])}",
            f"n_clusters={int(z['n_clusters'])}", *extra]


@pytest.mark.parametrize("bad", ["foo=1", "wandb=True", "cpu=True", "data.val_kwargs.download=True",
                                 "data.val_kwargs.image_set=train", "data.num_classes=63", "nokey"])
def test_semantic_command_rejects_bad_overrides(bad, tmp_path):
    se = load_pkg("segeval")
    z, sub = _sem("hungarian", tmp_path)
    with pytest.raises(ValueError):
        se.semantic_main(_sem_args(z, sub, bad))


def test_semantic_command_rejects_shape_mismatch_and_counts_before_device_work(tmp_path):
    se = load_pkg("segeval")
    z, sub = _sem("hungarian", tmp_path)
    seg = Path(sub(z["pairs"][3][2]))
    Image.fromarray(np.zeros((7, 9), dtype=np.uint8)).save(seg)
    with pytest.raises(ValueError, match=seg.name):
        se.semantic_main(_sem_args(z, sub))
    Image.fromarray(np.zeros((7, 9), dtype=np.uint8)).save(seg.parent / "99999.png")
    with pytest.raises(AssertionError):
        se.semantic_main(_sem_args(z, sub))


def _obj_args(tmp_path, ds, *extra):
    return [f"data_root={tmp_path / 'data'}", f"predictions.root={tmp_path / 'preds'}", "predictions.run=run",
            f"predictions.downsample={'null' if ds is None else ds}", "datasets=CUB,ECSSD", *extra]


@pytest.mark.parametrize("bad", ["foo=1", "wandb=True", "cpu=True", "datasets=CUB,VOC", "predictions.downsample=-2",
                                 "predictions.NOPE=x", "job_type=train"])
def test_object_command_rejects_bad_overrides(bad, tmp_path):
    se = load_pkg("segeval")
    _obj("ds16", tmp_path)
    with pytest.raises(ValueError):
        se.object_main(_obj_args(tmp_path, 16, bad))


def test_object_command_rejects_downsample_on_full_resolution_masks(tmp_path):
    se = load_pkg("segeval")
    _obj("full", tmp_path)
    with pytest.raises(ValueError, match="predictions.downsample=null"):
        se.object_main(_obj_args(tmp_path, 16))


@pytest.mark.parametrize("values", [(0, 2), (255,), (1, 255), (0, 1, 255)])
def test_object_command_rejects_bad_value_sets(values, tmp_path):
    se = load_pkg("segeval")
    _obj("ds16", tmp_path)
    f = tmp_path / "preds" / "ECSSD" / "run" / "img_001.png"
    shape = np.array(Image.open(f)).shape
    Image.fromarray(np.resize(np.array(values, dtype=np.uint8), shape)).save(f)
    with pytest.raises(ValueError, match="img_001.png"):
        se.object_main(_obj_args(tmp_path, 16))


@pytest.mark.parametrize("path", ["semantic-segmentation/eval.py", "object-segmentation/main.py"])
def test_command_shims_import(path):
    spec = importlib.util.spec_from_file_location("shim_" + path.split("/")[0].replace("-", "_"), ROOT / path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    assert callable(mod._segeval.semantic_main) and callable(mod._segeval.object_main)
