"""COCO20k in object localization, on the host: the selection list and its cache, CocoDetection's item order, the
reference's GT rule (tests/golden/ref_loc_coco.npz, written by the reference's own main.py,
oracle/make_coco_golden.py), the empty-GT and --set refusals, and the bounded decode of eigen-segmentation from
images."""
import json
import weakref
from pathlib import Path

import numpy as np
import pytest

from conftest import ROOT, load_pkg
from oracle.make_coco_golden import build_coco_tree

GOLD = ROOT / "tests" / "golden"


def _unpack(flat, offs, i, shape=None):
    a = flat[offs[i]:offs[i + 1]]
    return a.reshape(shape) if shape is not None else a


def _fixture():
    z = np.load(GOLD / "ref_loc_coco.npz")
    full = json.loads(z["full_json"].tobytes().decode())
    sizes = {int(i): tuple(int(v) for v in s) for i, s in zip(z["size_ids"], z["sizes"])}
    return z, full, sizes


def _tree(tmp_path, tag="hard", full=None, listed=None):
    z, full0, sizes = _fixture()
    ds, edir = build_coco_tree(Path(tmp_path), full or full0, list(listed or z[f"list_{tag}"]), sizes, {})
    return z, ds


def _args(ds, *extra):
    loc = load_pkg("localize")
    return loc.parse_args(["--dataset", "COCO20k", "--set", "train", "--dataset_root", str(ds), *extra])


@pytest.mark.parametrize("tag", ["hard", "nohard"])
def test_coco_reader_matches_the_reference(tmp_path, tag):
    loc = load_pkg("localize")
    z, ds = _tree(tmp_path, tag)
    name, items = loc._dataset_items(_args(ds, *(["--no_hard"] if tag == "nohard" else [])))
    assert name == "COCO20k_train" + ("-nohards" if tag == "nohard" else "")
    names = list(z[f"{tag}_names"])
    assert [it.name for it in items] == names
    for i, it in enumerate(items):
        want = _unpack(z[f"{tag}_gt"], z[f"{tag}_gt_offs"], i, (-1, 4))
        assert it.gt.dtype == np.int64 and str(it.gt.dtype) == z[f"{tag}_gt_dtypes"][i]
        assert np.array_equal(it.gt, want)
        assert it.eig_file == f"COCO_train2014_{int(it.name):012d}.pth"
        assert Path(it.path) == ds / "COCO" / "images" / "train2014" / f"COCO_train2014_{int(it.name):012d}.jpg"
        assert loc.jpeg_size(it.path) == _fixture()[2][int(it.name)]


def test_gt_rounds_half_to_even_in_float64():
    loc = load_pkg("localize")
    anns = [{"bbox": [10.5, 11.5, 20.0, 30.0], "iscrowd": 0}, {"bbox": [2.5, 3.5, 0.5, 1.5], "iscrowd": 0},
            {"bbox": [1.0, 1.0, 5.0, 5.0], "iscrowd": 1}, {"bbox": [0.0, 0.0, 3.4999997, 2], "iscrowd": 0},
            {"bbox": [1.25, 0, 2.2499997, 1], "iscrowd": 0}]
    got = loc.extract_gt_coco(anns)
    assert got.dtype == np.int64
    # x + w just below a half rounds down
    assert got.tolist() == [[10, 12, 30, 42], [2, 4, 3, 5], [0, 0, 3, 2], [1, 0, 3, 1]]
    assert loc.extract_gt_coco([{"bbox": [1, 1, 1, 1], "iscrowd": 1}]).shape == (0, 4)


def test_selection_ids_from_the_list(tmp_path):
    loc = load_pkg("localize")
    p = tmp_path / "list.txt"
    p.write_text("train2014/COCO_train2014_000000000391.jpg\nCOCO_train2014_000000000057.jpg\n"
                 "train2014/COCO_train2014_000000000391.jpg\n")
    assert loc.read_coco20k_ids(p) == [391, 57]


def test_cache_is_built_once_then_read(tmp_path):
    loc = load_pkg("localize")
    z, full, _ = _fixture()
    _, ds = _tree(tmp_path)
    cache = ds / "instances_train2014_sel20k.json"
    assert not cache.exists()
    _, items = loc._dataset_items(_args(ds))
    sel = json.loads(cache.read_text())
    ids = loc.read_coco20k_ids(ds / "coco_20k_filenames.txt")
    assert [im["id"] for im in sel["images"]] == ids
    assert sel["annotations"] == [a for a in full["annotations"] if a["image_id"] in ids]
    assert sel["categories"] == full["categories"]
    (ds / "COCO" / "annotations" / "instances_train2014.json").unlink()
    _, again = loc._dataset_items(_args(ds))
    assert [(it.name, it.gt.tolist()) for it in again] == [(it.name, it.gt.tolist()) for it in items]


def _refused(tmp_path, text, match):
    loc = load_pkg("localize")
    _, ds = _tree(tmp_path)
    cache = ds / "instances_train2014_sel20k.json"
    cache.write_text(text)
    with pytest.raises(ValueError, match=match) as e:
        loc._dataset_items(_args(ds))
    assert str(cache) in str(e.value) and "delete it" in str(e.value)
    assert cache.read_text() == text


def test_cache_in_the_reference_defective_format_is_refused_and_kept(tmp_path):
    _, full, _ = _fixture()
    anns = [a for a in full["annotations"] if a["image_id"] == 391]
    # what the reference's select_coco_20k writes: lists of annotation dicts for both images and annotations
    bad = json.dumps({"images": [[anns[-1]]], "annotations": [anns], "categories": full["categories"]})
    _refused(tmp_path, bad, "image records")


def test_cache_with_other_ids_is_refused_and_kept(tmp_path):
    _, full, _ = _fixture()
    other = json.dumps({"images": [im for im in full["images"] if im["id"] in (391, 77)], "annotations": [],
                        "categories": full["categories"]})
    _refused(tmp_path, other, "ids differ")


def test_set_other_than_train_is_refused():
    loc = load_pkg("localize")
    for s in ("trainval", "val", "test"):
        with pytest.raises(ValueError, match="COCO20k.*--set train"):
            loc.check_supported(loc.parse_args(["--dataset", "COCO20k", "--set", s]))
    loc.check_supported(loc.parse_args(["--dataset", "COCO20k", "--set", "train"]))


def test_listed_id_without_image_record_is_refused(tmp_path):
    loc = load_pkg("localize")
    z, _, _ = _fixture()
    _, ds = _tree(tmp_path, listed=list(z["list_hard"]) + ["train2014/COCO_train2014_000000123456.jpg"])
    with pytest.raises(ValueError, match="123456"):
        loc._dataset_items(_args(ds))
    assert not (ds / "instances_train2014_sel20k.json").exists()


@pytest.mark.parametrize("kind", ["all crowd", "no annotation"])
def test_image_without_a_box_needs_no_hard(tmp_path, kind):
    loc = load_pkg("localize")
    _lib = load_pkg("_lib")
    z, full, _ = _fixture()
    if kind == "all crowd":
        iid = 4410
    else:
        iid = 77
        full = dict(full, annotations=[a for a in full["annotations"] if a["image_id"] != iid])
    listed = list(z["list_hard"]) + [f"train2014/COCO_train2014_{iid:012d}.jpg"]
    _, ds = _tree(tmp_path, full=full, listed=listed)
    n0 = _lib.load().dss_kernel_launch_count()
    with pytest.raises(ValueError, match=f"{iid}.*--no_hard"):
        loc.main(["--dataset", "COCO20k", "--set", "train", "--dataset_root", str(ds), "--eigenseg",
                  "--precomputed_eigs_dir", str(tmp_path / "none"), "--output_dir", str(tmp_path / "out")])
    assert _lib.load().dss_kernel_launch_count() == n0
    assert not (tmp_path / "out").exists()
    _, items = loc._dataset_items(_args(ds, "--no_hard"))
    assert [it.name for it in items] == list(z["hard_names"])
    _, items = loc._dataset_items(_args(ds, "--no_evaluation"))
    assert str(iid) in [it.name for it in items]


def test_voc_items_keep_their_eigenvector_file_names():
    loc = load_pkg("localize")
    assert loc._Item("000005.jpg", "x/000005.jpg", None).eig_file == "000005.pth"
    assert loc._Item("9", "x.jpg", None, "COCO_train2014_000000000009.pth").eig_file == "COCO_train2014_000000000009.pth"


class _Tracked(np.ndarray):
    pass


def test_eigenseg_decode_is_bounded_over_many_sizes(tmp_path):
    from PIL import Image
    loc = load_pkg("localize")
    rng = np.random.default_rng(3)
    shapes = [(16 + 8 * (i % 13), 24 + 8 * (i % 7)) for i in range(60)]    # 60 images, 13 x 7 coprime: many sizes
    items = []
    for i, (H, W) in enumerate(shapes):
        p = tmp_path / f"{i}.png"
        Image.fromarray(rng.integers(0, 256, (H, W, 3), dtype=np.uint8)).save(p)
        items.append(loc._Item(f"{i}", str(p), None))
    assert len(set(shapes)) > 30
    alive = [0]
    peak = [0]

    def load(it):
        img = loc.load_rgb(it.path).view(_Tracked)
        alive[0] += 1
        peak[0] = max(peak[0], alive[0])
        weakref.finalize(img, lambda: alive.__setitem__(0, alive[0] - 1))
        return img

    bs, ahead = 4, 2
    seen = []
    for idx, batch in loc._image_batches(items, bs, load, ahead=ahead):
        assert alive[0] <= bs * (ahead + 1)
        assert len(idx) <= bs and all(shapes[j] == batch.shape[1:3] for j in idx)
        for t, j in enumerate(idx):
            assert np.array_equal(batch[t], loc.load_rgb(items[j].path))
        seen += idx
    assert sorted(seen) == list(range(60))
    assert peak[0] <= bs * (ahead + 1)


def test_eigenseg_batches_keep_the_streaming_order():
    loc = load_pkg("localize")
    sizes = [(1, 1), (2, 2), (1, 1), (1, 1), (3, 3), (2, 2), (2, 2), (1, 1), (3, 3)]
    assert loc._size_batches(sizes, 3) == [[0, 2, 3], [1, 5, 6], [4, 8], [7]]
