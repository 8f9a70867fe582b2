"""COCO20k object localization on the GPU: the precomputed-eigenvector route byte for byte against the reference's own
main.py (tests/golden/ref_loc_coco.npz), the same images through the COCO20k and the VOC layouts, eigen-segmentation
from images under any decode bound, and extract_all's eigenvectors read back by the command."""
import functools
import json
import pickle
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from conftest import ROOT, load_pkg
from oracle.make_coco_golden import build_coco_tree, coco_file_name
from oracle.make_localize_golden import build_tree, voc_xml

pytestmark = pytest.mark.gpu
GOLD = ROOT / "tests" / "golden"


def _unpack(flat, offs, i, shape=None):
    a = flat[offs[i]:offs[i + 1]]
    return a.reshape(shape) if shape is not None else a


def _run_main(cwd, argv):
    cmd = [sys.executable, str(ROOT / "object-localization" / "main.py")] + argv
    return subprocess.run(cmd, cwd=cwd, capture_output=True, text=True, check=True)


@pytest.mark.parametrize("tag", ["hard", "nohard"])
def test_main_coco_precomputed_matches_reference(cuda, tmp_path, tag):
    z = np.load(GOLD / "ref_loc_coco.npz")
    full = json.loads(z["full_json"].tobytes().decode())
    sizes = {int(i): tuple(int(v) for v in s) for i, s in zip(z["size_ids"], z["sizes"])}
    K = z["eig_K"]
    eigs = {int(iid): _unpack(z["eigs"], z["eig_offs"], i, (int(K[i]), -1)) for i, iid in enumerate(z["eig_ids"])}
    # no selection cache: the command builds it from the full train2014 file
    _, edir = build_coco_tree(tmp_path, full, list(z[f"list_{tag}"]), sizes, eigs)
    extra = ["--no_hard"] if tag == "nohard" else []
    r = _run_main(tmp_path, ["--dataset", "COCO20k", "--set", "train", "--eigenseg", "--precomputed_eigs_dir",
                             str(edir), "--output_dir", "outputs"] + extra)
    folder = tmp_path / "outputs" / ("COCO20k_train" + ("-nohards" if extra else "")) / "LOST-vit_small16_k"
    assert (folder / "results.txt").read_bytes() == z[f"{tag}_results"].tobytes()
    assert "corloc:" in r.stdout
    preds = pickle.loads((folder / "preds.pkl").read_bytes())
    gt = pickle.loads((folder / "gt.pkl").read_bytes())
    names = list(z[f"{tag}_names"])
    assert list(preds) == names and list(gt) == names
    for i, n in enumerate(names):
        assert preds[n].dtype == np.int64 and np.array_equal(preds[n], z[f"{tag}_preds"][i])
        g = _unpack(z[f"{tag}_gt"], z[f"{tag}_gt_offs"], i, (-1, 4))
        assert gt[n].dtype == np.int64 and np.array_equal(gt[n], g)


# (image id, (H, W)): COCO's shapes, an odd one, and one below a ViT-B/8 grid of 128 x 128
SHAPES = [(9, (480, 640)), (57, (640, 480)), (233, (359, 481)), (391, (427, 640)), (786, (612, 612)),
          (1204, (640, 640)), (5012, (480, 640)), (6000, (333, 500))]
GRAY, CMYK = 57, 786


def _same_images_in_both_layouts(root: Path):
    """One set of JPEG files written as a COCO20k tree and as a VOC07 tree (same bytes, VOC ids in COCO's id order);
    one box per image, the same box in both (VOC: 1-based inclusive, COCO: x, y, w, h)."""
    from PIL import Image
    synth = load_pkg("synth")
    full = {"images": [], "annotations": [], "categories": [{"id": 1, "name": "thing", "supercategory": "thing"}]}
    listed, sizes, xmls = [], {}, []
    jpegs = {}
    for k, (iid, (H, W)) in enumerate(SHAPES):
        im = Image.fromarray(synth.blobs_image(H, W, 40 + k).numpy())
        if iid == GRAY:
            im = im.convert("L")
        elif iid == CMYK:
            im = im.convert("CMYK")
        x0, y0, x1, y1 = W // 5, H // 6, W // 5 + W // 2, H // 6 + H // 2
        full["images"].append({"id": iid, "file_name": coco_file_name(iid), "height": H, "width": W})
        full["annotations"].append({"id": k + 1, "image_id": iid, "category_id": 1, "iscrowd": 0,
                                    "bbox": [float(x0), float(y0), float(x1 - x0), float(y1 - y0)]})
        listed.append(f"train2014/{coco_file_name(iid)}")
        sizes[iid] = (H, W)
        xmls.append(voc_xml(f"{iid:06d}.jpg", H, W, [("thing", 0, 0, x0 + 1, y0 + 1, x1, y1)]))
        jpegs[iid] = im
    coco_ds, _ = build_coco_tree(root / "coco", full, listed, sizes, {})
    ids = [f"{iid:06d}" for iid, _ in SHAPES]
    voc_ds, _ = build_tree(root / "voc", ids, xmls, [s for _, s in SHAPES], [np.zeros((1, 1), np.float32)] * len(ids))
    for iid, im in jpegs.items():   # the same bytes under both layouts
        p = coco_ds / "COCO" / "images" / "train2014" / coco_file_name(iid)
        im.save(p, format="JPEG", quality=90)
        (voc_ds / "VOCdevkit" / "VOC2007" / "JPEGImages" / f"{iid:06d}.jpg").write_bytes(p.read_bytes())
    return coco_ds, voc_ds


def _corloc_line(preds, gt):
    loc = load_pkg("localize")
    hits = [bool(torch.any(loc.bbox_iou(torch.from_numpy(preds[n]), torch.from_numpy(gt[n])) >= 0.5)) for n in preds]
    return "corloc,%.1f,,\n" % (100 * np.sum(hits) / len(hits))


@pytest.mark.parametrize("arch,patch", [("vit_small", 16), ("vit_base", 8)])
def test_coco_and_voc_layouts_give_the_same_boxes(cuda, tmp_path, arch, patch):
    loc = load_pkg("localize")
    coco_ds, voc_ds = _same_images_in_both_layouts(tmp_path)
    methods = {"lost": [], "dinoseg": ["--dinoseg"], "eigenseg": ["--eigenseg", "--which_matrix", "laplacian"]}
    for method, flags in methods.items():
        got = {}
        for layout, argv in (("coco", ["--dataset", "COCO20k", "--set", "train", "--dataset_root", str(coco_ds)]),
                             ("voc", ["--dataset", "VOC07", "--dataset_root", str(voc_ds)])):
            out = tmp_path / f"out_{layout}_{method}"
            score = loc.main(argv + flags + ["--arch", arch, "--patch_size", str(patch), "--seed", "5",
                                             "--batch_size", "3", "--output_dir", str(out)])
            folder = next(out.glob("*/*"))
            preds = pickle.loads((folder / "preds.pkl").read_bytes())
            gt = pickle.loads((folder / "gt.pkl").read_bytes())
            line = _corloc_line(preds, gt)
            assert (folder / "results.txt").read_text() == line and abs(score - float(line.split(",")[1])) < 0.051
            got[layout] = (preds, gt)
        (cp, cg), (vp, vg) = got["coco"], got["voc"]
        assert list(cp) == [str(iid) for iid, _ in SHAPES] and list(vp) == [f"{iid:06d}.jpg" for iid, _ in SHAPES]
        for iid, _ in SHAPES:
            a, b = cp[str(iid)], vp[f"{iid:06d}.jpg"]
            assert a.dtype == b.dtype == np.int64 and np.array_equal(a, b), (method, iid, a, b)
            assert np.array_equal(cg[str(iid)], vg[f"{iid:06d}.jpg"])


def test_eigenseg_decode_bound_leaves_the_boxes_unchanged(cuda, tmp_path, monkeypatch):
    loc = load_pkg("localize")
    coco_ds, _ = _same_images_in_both_layouts(tmp_path)
    args = loc.parse_args(["--dataset", "COCO20k", "--set", "train", "--dataset_root", str(coco_ds), "--eigenseg",
                           "--which_matrix", "laplacian", "--batch_size", "2", "--seed", "5"])
    _, items = loc._dataset_items(args)
    vit = load_pkg("vit")
    model, _, _, _ = vit.get_model("dino_vits16", seed=5)
    image_batches = loc._image_batches
    got = []
    for ahead in (0, 64):
        monkeypatch.setattr(loc, "_image_batches", functools.partial(image_batches, ahead=ahead))
        got.append(loc._from_images(args, items, model))
    assert list(got[0]) and sorted(got[0]) == sorted(got[1]) == sorted(it.name for it in items)
    for n in got[0]:
        assert np.array_equal(got[0][n], got[1][n])


def test_extract_all_then_coco_eigenseg(cuda, tmp_path):
    extract = load_pkg("extract")
    coco_ds, _ = _same_images_in_both_layouts(tmp_path)
    # colour-free extract_all decodes every file as RGB, the grayscale and CMYK ones included
    extract.extract_all(images_list=str(coco_ds / "coco_20k_filenames.txt"), images_root=str(coco_ds / "COCO" / "images"),
                        model_name="dino_vits16", features_dir=None, eigs_dir=str(tmp_path / "eigs"), K=4, seed=5,
                        batch_size=3, writer="thread", yes=True)
    edir = tmp_path / "eigs" / "train2014"
    assert sorted(p.name for p in edir.iterdir()) == sorted(f"COCO_train2014_{iid:012d}.pth" for iid, _ in SHAPES)
    _run_main(tmp_path, ["--dataset", "COCO20k", "--set", "train", "--dataset_root", str(coco_ds), "--eigenseg",
                         "--precomputed_eigs_dir", str(edir), "--which_matrix", "laplacian", "--output_dir", "outputs"])
    folder = tmp_path / "outputs" / "COCO20k_train" / "LOST-vit_small16_k"
    preds = pickle.loads((folder / "preds.pkl").read_bytes())
    assert sorted(preds) == sorted(str(iid) for iid, _ in SHAPES)
    assert (folder / "results.txt").read_text() == _corloc_line(preds, pickle.loads((folder / "gt.pkl").read_bytes()))
