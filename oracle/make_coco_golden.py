"""Writes tests/golden/ref_loc_coco.npz by running the reference's OWN object-localization/main.py with
``--dataset COCO20k --set train --eigenseg --precomputed_eigs_dir ...`` (read-only, dev container only), under the
stubs of make_localize_golden.py plus two more:

  pycocotools.coco.COCO -> a stand-in with the members torchvision's CocoDetection reads (imgs, getAnnIds, loadAnns,
                           loadImgs), in pycocotools' order: an image's annotations in their order in the JSON file;
  datasets/instances_train2014_sel20k.json is written correctly formatted before the run, so the reference's
                           defective select_coco_20k is never called (DESIGN §5); the --no_hard run also gets an empty
                           datasets/hard_COCO20k_train_2014.txt, without which its get_hards crashes.

The fixture holds data only: the full train2014 JSON of the synthetic tree, the two selection lists, the image sizes,
the eigenvectors and the reference's preds.pkl / gt.pkl / results.txt of both runs. The tests rebuild the tree with
build_coco_tree. The synthetic tree has image ids listed out of order (and one listed twice), boxes with .5
coordinates and with x + w that rounds differently in float32, crowd annotations among normal ones, annotations of
several images interleaved in the file, images the list does not select, COCO's image shapes and an odd one, and an
image whose annotations are all crowd (in the --no_hard run only: the reference crashes on it otherwise).

    python -m oracle.make_coco_golden
"""
from __future__ import annotations

import json
import pickle
import tempfile
from pathlib import Path

import numpy as np
import torch

from .make_localize_golden import GOLDEN, _blob_vector, _pack, load_reference, run_reference_main
from .ref_shim import _stub

# (image id, (H, W), patch size of its eigenvectors), in selection-list order
IMAGES = [(391, (480, 640), 16), (57, (640, 480), 8), (1204, (427, 640), 16), (9, (640, 640), 8),
          (786, (612, 612), 16), (233, (359, 481), 8), (5012, (640, 427), 16)]
ALL_CROWD = (4410, (480, 640), 16)      # every annotation is crowd: listed for the --no_hard run only
UNSELECTED = [(77, (480, 640)), (3000, (500, 375))]
HALF_EVEN = [[10.5, 11.5, 20.0, 30.0], [2.5, 3.5, 0.5, 1.5]]   # -> [10, 12, 30, 42] and [2, 4, 3, 5]


def coco_file_name(image_id: int) -> str:
    return f"COCO_train2014_{image_id:012d}.jpg"


def _float32_flip(rng, W):
    """(x, w) whose float64 sum x + w rounds to another integer than the float32 sum: the sum is 3e-7 below k + 0.5
    for an odd k, which float32 rounds to k + 0.5 and then half to even up to k + 1."""
    for _ in range(100):
        x = round(float(rng.uniform(0, W / 2)), 2)
        k = 2 * int(rng.integers(int(x) // 2 + 1, W // 2)) + 1
        w = k + 0.5 - x - 3e-7
        if round(x + w) != round(float(np.float32(x) + np.float32(w))):
            return x, w
    raise AssertionError("no float32 rounding flip found")


def synthetic_coco(rng):
    """(full train2014 dict, selection list lines of the --no_hard run, the same without the all-crowd image)."""
    images, anns = [], []
    for iid, (H, W), _ in IMAGES + [ALL_CROWD]:
        images.append({"id": iid, "file_name": coco_file_name(iid), "height": H, "width": W})
    for iid, (H, W) in UNSELECTED:
        images.append({"id": iid, "file_name": coco_file_name(iid), "height": H, "width": W})
    sizes = {im["id"]: (im["height"], im["width"]) for im in images}
    for k, (iid, (H, W), _) in enumerate(IMAGES):
        n = int(rng.integers(2, 5))
        for t in range(n):
            crowd = int(t > 0 and rng.random() < 0.35)
            if t == 0 and k < len(HALF_EVEN):
                box = list(HALF_EVEN[k])
            elif t == 0 and k == len(HALF_EVEN):
                x, w = _float32_flip(rng, W)
                box = [x, round(float(rng.uniform(0, H / 2)), 2), w, round(float(rng.uniform(1, H / 2)), 2)]
            else:
                x, y = rng.uniform(0, W - 2), rng.uniform(0, H - 2)
                w, h = rng.uniform(1, W - x), rng.uniform(1, H - y)
                box = [float(np.round(v * 2) / 2) if rng.random() < 0.3 else round(float(v), 2) for v in (x, y, w, h)]
            anns.append({"image_id": iid, "category_id": int(rng.integers(1, 91)), "bbox": box, "iscrowd": crowd})
    for iid, (H, W) in [(ALL_CROWD[0], ALL_CROWD[1])] * 2 + UNSELECTED:
        anns.append({"image_id": iid, "category_id": 1, "bbox": [5.0, 6.0, W / 3, H / 4],
                     "iscrowd": int(iid == ALL_CROWD[0])})
    order = rng.permutation(len(anns))     # several images' annotations interleaved in the file
    anns = [dict(anns[j], id=100 + i, area=float(anns[j]["bbox"][2] * anns[j]["bbox"][3])) for i, j in enumerate(order)]
    full = {"images": images, "annotations": anns,
            "categories": [{"id": c, "name": f"class{c}", "supercategory": "thing"} for c in range(1, 91)]}
    listed = [f"train2014/{coco_file_name(iid)}" for iid, _, _ in IMAGES]
    listed.insert(3, listed[1])           # an id listed twice counts once
    nohard = listed[:4] + [f"train2014/{coco_file_name(ALL_CROWD[0])}"] + listed[4:]
    return full, nohard, listed, sizes


def build_coco_tree(root: Path, full: dict, listed, sizes, eigs: dict, eig_dir_name="laplacian_dino_vits16",
                    cache: bool = False):
    """{root}/datasets as the reference lays COCO20k out (datasets.py:50-66) and the eigenvector files
    COCO_train2014_{id:012d}.pth (main.py:257-258); also used by the tests. The images are flat colour, one of them
    grayscale. With cache=True the selection cache is written too, correctly formatted."""
    from PIL import Image
    ds = root / "datasets"
    (ds / "COCO" / "images" / "train2014").mkdir(parents=True, exist_ok=True)
    (ds / "COCO" / "annotations").mkdir(parents=True, exist_ok=True)
    (ds / "COCO" / "annotations" / "instances_train2014.json").write_text(json.dumps(full))
    (ds / "coco_20k_filenames.txt").write_text("".join(f"{s}\n" for s in listed))
    for im in full["images"]:
        H, W = sizes[im["id"]]
        mode, colour = ("L", 128) if im["id"] == IMAGES[2][0] else ("RGB", (90, 120, 150))
        Image.new(mode, (int(W), int(H)), colour).save(ds / "COCO" / "images" / "train2014" / im["file_name"])
    if cache:
        ids = list(dict.fromkeys(int(s.split("_")[-1].split(".")[0]) for s in listed))
        sel = {"images": [next(im for im in full["images"] if im["id"] == i) for i in ids],
               "annotations": [a for a in full["annotations"] if a["image_id"] in ids],
               "categories": full["categories"]}
        (ds / "instances_train2014_sel20k.json").write_text(json.dumps(sel))
    edir = root / eig_dir_name
    edir.mkdir(parents=True, exist_ok=True)
    for iid, ev in eigs.items():
        torch.save({"eigenvalues": torch.zeros(ev.shape[0]), "eigenvectors": torch.from_numpy(ev)},
                   edir / f"COCO_train2014_{int(iid):012d}.pth")
    return ds, edir


class _COCO:
    """pycocotools.coco.COCO as CocoDetection reads it: imgs, getAnnIds(image id), loadAnns, loadImgs."""

    def __init__(self, annotation_file):
        with open(annotation_file) as f:
            d = json.load(f)
        self.imgs = {im["id"]: im for im in d["images"]}
        self.anns = {a["id"]: a for a in d["annotations"]}
        self.img_to_anns = {}
        for a in d["annotations"]:
            self.img_to_anns.setdefault(a["image_id"], []).append(a)

    def getAnnIds(self, imgIds=()):
        ids = imgIds if isinstance(imgIds, (list, tuple)) else [imgIds]
        return [a["id"] for i in ids for a in self.img_to_anns.get(i, [])]

    def loadAnns(self, ids):
        return [self.anns[i] for i in ids]

    def loadImgs(self, ids):
        return [self.imgs[i] for i in (ids if isinstance(ids, (list, tuple)) else [ids])]


def make_coco(ref_main, rng):
    full, nohard_list, hard_list, sizes = synthetic_coco(rng)
    eigs = {}
    for iid, (H, W), P in IMAGES + [ALL_CROWD]:
        eigs[iid] = np.stack([_blob_vector(rng, H // P, W // P) for _ in range(3)]).astype(np.float32)
    ids = sorted(eigs)
    out = {"full_json": np.frombuffer(json.dumps(full).encode(), dtype=np.uint8),
           "list_hard": np.array(hard_list), "list_nohard": np.array(nohard_list),
           "size_ids": np.array(sorted(sizes)), "sizes": np.array([sizes[i] for i in sorted(sizes)]),
           "eig_ids": np.array(ids), "eig_K": np.array([eigs[i].shape[0] for i in ids])}
    out["eigs"], out["eig_offs"] = _pack([eigs[i] for i in ids])
    for tag, listed, extra in (("hard", hard_list, []), ("nohard", nohard_list, ["--no_hard"])):
        with tempfile.TemporaryDirectory() as td:
            td = Path(td)
            ds, edir = build_coco_tree(td, full, listed, sizes, eigs, cache=True)
            if extra:
                (ds / "hard_COCO20k_train_2014.txt").write_text("")
            run_reference_main(ref_main, td, ["--dataset", "COCO20k", "--set", "train", "--eigenseg",
                                              "--precomputed_eigs_dir", str(edir), "--output_dir",
                                              str(td / "outputs")] + extra)
            folder = td / "outputs" / ("COCO20k_train" + ("-nohards" if extra else "")) / "LOST-vit_small16_k"
            preds = pickle.loads((folder / "preds.pkl").read_bytes())
            gt = pickle.loads((folder / "gt.pkl").read_bytes())
            assert list(gt) == list(preds)
            out[f"{tag}_names"] = np.array(list(preds))
            out[f"{tag}_preds"] = np.stack([preds[k] for k in preds])
            gflat, goffs = _pack([gt[k] for k in preds])
            out[f"{tag}_gt"], out[f"{tag}_gt_offs"] = gflat.astype(np.int64), goffs
            out[f"{tag}_gt_dtypes"] = np.array([str(gt[k].dtype) for k in preds])
            out[f"{tag}_results"] = np.frombuffer((folder / "results.txt").read_bytes(), dtype=np.uint8)
    np.savez_compressed(GOLDEN / "ref_loc_coco.npz", **out)
    return len(out["hard_names"]), len(out["nohard_names"])


def main():
    _, _, ref_main = load_reference()
    _stub("pycocotools")
    _stub("pycocotools.coco", COCO=_COCO)
    rng = np.random.default_rng(20261018)
    print("COCO20k images (hard, nohard)", make_coco(ref_main, rng))


if __name__ == "__main__":
    main()
