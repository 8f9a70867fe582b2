"""Writes tests/golden/ref_semeval_*.npz and ref_objseg_*.npz by running the reference's OWN evaluation code
(semantic-segmentation/eval.py evaluate + dataset/voc.py, object-segmentation/main.py evaluate_predictions + metrics.py
+ dataset.py; read-only, dev container only) on seeded synthetic trees, under inert stubs for what is not installed:
hydra, omegaconf, accelerate, wandb, albumentations (imported by dataset/__init__.py), matplotlib and skimage (only
the unused visualize() calls them). joblib's multiprocessing pool of eval_utils is kept.

The fixtures hold data only: every file of the tree (relative path + bytes), the reference's results and its captured
stdout with the tree's root written as <ROOT>. The tests rebuild the tree in a temporary directory.

    python -m oracle.make_segeval_golden
"""
from __future__ import annotations

import contextlib
import io
import sys
import tempfile
import types
from pathlib import Path

import numpy as np
from PIL import Image

from .ref_shim import _stub

REF = Path("/root/reference")
GOLDEN = Path(__file__).resolve().parents[1] / "tests" / "golden"
ROOT_MARK = "<ROOT>"


class AttrDict(dict):
    __getattr__ = dict.__getitem__


def _stubs():
    def _never(*a, **k):
        raise RuntimeError("stubbed dependency called")
    _stub("hydra", main=lambda **k: (lambda f: f))
    _stub("wandb", init=_never)
    _stub("accelerate", Accelerator=_never)
    _stub("omegaconf", DictConfig=dict, OmegaConf=types.SimpleNamespace(to_yaml=_never))
    _stub("albumentations")
    _stub("albumentations.pytorch")
    _stub("matplotlib")
    _stub("matplotlib.cm", get_cmap=_never)
    _stub("skimage")
    _stub("skimage.color", label2rgb=_never)


def _import_from(app: str, names):
    """Imports the reference modules of one app (its util / dataset names collide with the other app's)."""
    for n in ("util", "dataset", "dataset.voc", "metrics", "main", "eval", "eval_utils"):
        sys.modules.pop(n, None)
    sys.path.insert(0, str(REF / app))
    try:
        return [__import__(n, fromlist=["_"]) for n in names]
    finally:
        sys.path.remove(str(REF / app))


# ------------------------------------------------------------------------------------------------ trees
def save_png(path: Path, arr, mode=None, palette=None):
    path.parent.mkdir(parents=True, exist_ok=True)
    im = Image.fromarray(arr) if mode is None else Image.fromarray(arr).convert(mode)
    if palette is not None:
        im = Image.frombytes("P", arr.shape[::-1], np.ascontiguousarray(arr).tobytes())
        im.putpalette(palette)
    im.save(path)


def save_jpeg(path: Path, H: int, W: int, rng):
    path.parent.mkdir(parents=True, exist_ok=True)
    Image.fromarray(np.full((H, W, 3), rng.integers(0, 256, 3), dtype=np.uint8)).save(path, quality=50)


def tree_files(root: Path):
    files = sorted(p for p in root.rglob("*") if p.is_file())
    names = np.array([str(p.relative_to(root)) for p in files])
    data = [np.frombuffer(p.read_bytes(), dtype=np.uint8) for p in files]
    offs = np.cumsum([0] + [len(d) for d in data]).astype(np.int64)
    return names, np.concatenate(data), offs


def build_tree(z, root: Path) -> Path:
    """Writes the files of a fixture under root."""
    for i, name in enumerate(z["file_names"]):
        p = root / str(name)
        p.parent.mkdir(parents=True, exist_ok=True)
        p.write_bytes(z["file_blob"][z["file_offs"][i]:z["file_offs"][i + 1]].tobytes())
    return root


VOC_PALETTE = [v for i in range(256) for v in ((i * 37) % 256, (i * 91) % 256, (i * 151) % 256)]


def _voc_target(rng, H, W, n_classes, absent):
    t = np.zeros((H, W), dtype=np.uint8)
    classes = [c for c in range(1, n_classes) if c != absent]
    for _ in range(int(rng.integers(1, 4))):
        h, w = int(rng.integers(H // 5, H // 2)), int(rng.integers(W // 5, W // 2))
        y, x = int(rng.integers(0, H - h)), int(rng.integers(0, W - w))
        t[max(0, y - 2):y + h + 2, max(0, x - 2):x + w + 2] = 255   # the VOC "void" border
        t[y:y + h, x:x + w] = rng.choice(classes)
    t[rng.random((H, W)) < 0.01] = rng.choice([30, 200])           # values outside the classes
    return t


def _pseudolabel(rng, t, ph, pw, n_clusters, perm, extra):
    """A pseudo-label correlated with the target: the permuted class of the nearest cell, with noise, values >=
    n_clusters (255 included) and `extra` unused cluster values reserved for the tie."""
    H, W = t.shape
    ys, xs = (np.arange(ph) * H) // ph, (np.arange(pw) * W) // pw
    cell = t[np.ix_(ys, xs)].astype(np.int64)
    p = perm[np.where(cell < len(perm), cell, 0)]
    noise = rng.random(p.shape)
    p = np.where(noise < 0.1, rng.integers(0, n_clusters - extra, p.shape), p)
    p = np.where(noise > 0.97, rng.choice([n_clusters, 255], p.shape), p)
    return p.astype(np.uint8)


def semantic_case(tmp: Path, seed: int, n_clusters: int, num_classes: int = 20):
    rng = np.random.default_rng(seed)
    n_classes = num_classes + 1
    voc = tmp / "VOC" / "VOCdevkit" / "VOC2012"
    seg_dir = tmp / "segments"
    absent = 17
    perm = rng.permutation(n_clusters - 2)[:n_classes] if n_clusters == n_classes else rng.permutation(n_clusters)[:n_classes]
    # (H, W, pseudo-label shape rule): H // 16, H // 8, 2 (H // 16), full resolution, a height that matches the rule
    # with a width that does not, a map that matches no rule at the image size (identity)
    specs = [(75, 90, "h16"), (64, 80, "h8"), (100, 67, "2h16"), (50, 53, "full"), (81, 120, "h16w"),
             (66, 70, "h8"), (90, 75, "h16"), (47, 53, "full"), (120, 97, "2h16"), (40, 40, "tie")]
    extra_stems = ["2008_000001", "2009_000500", "2010_000020"]   # JPEGImages outside the split
    stems = [f"2007_{1000 + 37 * i:06d}" for i in range(len(specs))]
    all_stems = sorted(stems + extra_stems)
    pairs = {}
    for i, (H, W, rule) in enumerate(specs):
        t = _voc_target(rng, H, W, n_classes, absent)
        if rule == "tie":   # clusters n_clusters-2 and n_clusters-1 overlap class 3 identically and nothing else
            t[:] = 255
            t[10:30, 10:30] = 3
            p = np.full((H, W), 255, dtype=np.uint8)
            p[10:20, 10:30] = n_clusters - 2
            p[20:30, 10:30] = n_clusters - 1
        else:
            ph, pw = {"h16": (H // 16, W // 16), "h8": (H // 8, W // 8), "2h16": (2 * (H // 16), 2 * (W // 16)),
                      "full": (H, W), "h16w": (H // 16, W // 16 + 3)}[rule]
            p = _pseudolabel(rng, t, ph, pw, n_clusters, perm, 2 if n_clusters == n_classes else 0)
        pairs[stems[i]] = (H, W, t, p)
    for k, stem in enumerate(all_stems):
        if stem in pairs:
            H, W, t, p = pairs[stem]
            save_png(voc / "SegmentationClass" / f"{stem}.png", t, palette=VOC_PALETTE)
        else:
            H, W = int(rng.integers(40, 90)), int(rng.integers(40, 90))
            p = rng.integers(0, n_clusters, (H // 16, W // 16)).astype(np.uint8)
        save_jpeg(voc / "JPEGImages" / f"{stem}.jpg", H, W, rng)
        save_png(seg_dir / f"{k:05d}.png", p)
    (voc / "ImageSets" / "Segmentation").mkdir(parents=True, exist_ok=True)
    (voc / "ImageSets" / "Segmentation" / "val.txt").write_text("".join(f"{s}\n" for s in stems))
    return tmp / "VOC", seg_dir


def run_semantic(root: Path, seg_dir: Path, n_clusters: int, num_classes: int = 20):
    eval_mod, voc_mod = _import_from("semantic-segmentation", ["eval", "dataset.voc"])
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        ds = voc_mod.VOCSegmentationWithPseudolabels(root=str(root), year="2012", image_set="val",
                                                     download=False, segments_dir=str(seg_dir), transform=None)
        cfg = AttrDict(data=AttrDict(num_classes=num_classes))
        stats, match = eval_mod.evaluate(cfg=cfg, dataset_val=ds, n_clusters=n_clusters)
        print(stats)
    pairs = [(ds.images[i], ds.masks[i], ds.segments[i]) for i in range(len(ds))]
    return stats, match, buf.getvalue().splitlines(), pairs


# ------------------------------------------------------------------------------------------------ object segmentation
def _mask(rng, H, W, mode):
    """A mask whose R channel (after convert('RGB')) holds 0, 127, 128 and 255."""
    v = np.zeros((H, W), dtype=np.uint8)
    y, x = int(rng.integers(0, H // 2)), int(rng.integers(0, W // 2))
    v[y:y + H // 2, x:x + W // 2] = 255
    v[rng.random((H, W)) < 0.05] = 127
    v[rng.random((H, W)) < 0.05] = 128
    if mode == "1":
        return Image.fromarray(v >= 128)
    if mode == "RGB":
        return Image.fromarray(np.stack([v, 255 - v, rng.integers(0, 256, (H, W), dtype=np.uint8)], -1))
    if mode == "P":
        idx = np.select([v == 255, v == 128, v == 127], [1, 2, 3], 0).astype(np.uint8)
        im = Image.frombytes("P", (W, H), idx.tobytes())
        im.putpalette([0, 9, 9, 255, 0, 0, 128, 200, 1, 127, 255, 255] + [0] * (256 * 3 - 12))
        return im
    return Image.fromarray(v)


OBJ_SPECS = {   # name: (layout, crop, [(H, W)])
    "CUB": ("folders", True, [(70, 65), (65, 72), (100, 65), (48, 81), (33, 33), (65, 100)]),
    "ECSSD": ("flat", False, [(60, 75), (47, 47), (90, 50), (33, 70), (50, 50)]),
}


def object_case(tmp: Path, seed: int, downsample):
    rng = np.random.default_rng(seed)
    data, preds = tmp / "data", tmp / "preds"
    sets = [{0, 255}, {0, 1}, {0}]
    modes = ["L", "RGB", "P", "1"]
    k = 0
    sub = {"CUB": ("CUB_200_2011/test_images", "CUB_200_2011/test_segmentations", "CUB_200_2011"),
           "ECSSD": ("ECSSD/images", "ECSSD/ground_truth_mask", "ECSSD")}
    for name, (layout, crop, sizes) in OBJ_SPECS.items():
        img_dir, lab_dir, pred_sub = sub[name]
        for i, (H, W) in enumerate(sizes):
            stem = f"img_{i:03d}"
            folder = f"{i % 2:03d}.class/" if layout == "folders" else ""
            save_jpeg(data / img_dir / f"{folder}{stem}.jpg", H, W, rng)
            m = _mask(rng, H, W, modes[k % 4])
            empty = name == "ECSSD" and i == len(sizes) - 1
            if empty:   # empty prediction on an empty ground truth: union 0 -> IoU 0
                m = Image.fromarray(np.zeros((H, W), dtype=np.uint8))
            (data / lab_dir / folder).mkdir(parents=True, exist_ok=True)
            m.save(data / lab_dir / f"{folder}{stem}.png")
            shape = (H, W) if downsample is None else (H // downsample, W // downsample)
            vals = sorted({0} if empty else sets[k % 3])
            p = np.where(rng.random(shape) < 0.5, vals[-1], vals[0]).astype(np.uint8)
            save_png(preds / pred_sub / "run" / f"{stem}.png", p)
            k += 1
    return data, preds


def run_object(data: Path, preds: Path, downsample):
    main_mod, metrics_mod, dataset_mod = _import_from("object-segmentation", ["main", "metrics", "dataset"])
    from torch.utils.data import DataLoader
    per_image = []
    compute = metrics_mod.compute_metrics

    def recording(**kw):
        r = compute(**kw)
        per_image.append((r["acc"][0], r["iou"][0]))
        return r
    main_mod.metrics.compute_metrics = recording
    sub = {"CUB": ("CUB_200_2011/test_images", "CUB_200_2011/test_segmentations", "CUB_200_2011"),
           "ECSSD": ("ECSSD/images", "ECSSD/ground_truth_mask", "ECSSD")}
    cfg = AttrDict(predictions=AttrDict(downsample=downsample, **{n: str(preds / s[2] / "run") for n, s in sub.items()}))
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        for name, (layout, crop, _) in OBJ_SPECS.items():
            ds = dataset_mod.SegmentationDataset(images_dir=str(data / sub[name][0]), labels_dir=str(data / sub[name][1]),
                                                 crop=crop, image_size=None, name=name)
            main_mod.evaluate_predictions(cfg=cfg, dataloader_val=DataLoader(ds, batch_size=1, num_workers=0),
                                          accelerator=None)
    main_mod.metrics.compute_metrics = compute
    return buf.getvalue().splitlines(), per_image


def main():
    _stubs()
    GOLDEN.mkdir(parents=True, exist_ok=True)
    for tag, seed, n_clusters in (("hungarian", 0, 21), ("majority", 1, 27)):
        with tempfile.TemporaryDirectory() as d:
            tmp = Path(d)
            root, seg_dir = semantic_case(tmp, seed, n_clusters)
            stats, match, lines, pairs = run_semantic(root, seg_dir, n_clusters)
            names, blob, offs = tree_files(tmp)
            rel = lambda s: str(s).replace(str(tmp), ROOT_MARK)   # noqa: E731
            np.savez_compressed(
                GOLDEN / f"ref_semeval_{tag}.npz", file_names=names, file_blob=blob, file_offs=offs,
                n_clusters=n_clusters, num_classes=20, root=rel(root), segments_dir=rel(seg_dir),
                pairs=np.array([[rel(a), rel(b), rel(c)] for a, b, c in pairs]),
                lines=np.array([rel(x) for x in lines]), jac=np.array(stats["jaccards_all_categs"], dtype=np.float64),
                miou=np.float64(stats["mIoU"]), match=np.array([[int(a), int(b)] for a, b in match], dtype=np.int64))
            print(tag, "\n".join(lines))
    for tag, seed, ds in (("ds16", 2, 16), ("ds8", 3, 8), ("full", 4, None)):
        with tempfile.TemporaryDirectory() as d:
            tmp = Path(d)
            data, preds = object_case(tmp, seed, ds)
            lines, per_image = run_object(data, preds, ds)
            names, blob, offs = tree_files(tmp)
            np.savez_compressed(
                GOLDEN / f"ref_objseg_{tag}.npz", file_names=names, file_blob=blob, file_offs=offs,
                downsample=-1 if ds is None else ds, lines=np.array(lines),
                acc=np.array([a for a, _ in per_image], dtype=np.float64),
                iou=np.array([u for _, u in per_image], dtype=np.float64),
                iou_is_int=np.array([isinstance(u, int) for _, u in per_image]))
            print(tag, "\n".join(lines))


if __name__ == "__main__":
    main()
