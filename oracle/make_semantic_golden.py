"""Generates the semantic-segmentation fixtures under tests/golden/ (ref_bboxes.npz, ref_bbox_clusters.npz,
ref_semantic_segmaps.npz) by running the reference's OWN ``_extract_bbox``, ``extract_bbox_clusters`` and
``extract_semantic_segmentations`` (imported from /root/reference through oracle/ref_shim.py) on small seeded inputs.
Run in the dev container only:

    python -m oracle.make_semantic_golden

skimage is not installed there: its binary_erosion / binary_dilation (extract_utils.py:116) are supplied by the
scipy.ndimage restatement of oracle/bbox_ref.py while the reference's module is imported. scikit-learn is the real one.
tests/test_cpu_semantic.py checks the box oracle and the host semantic maps against these fixtures;
tests/test_semantic_gpu.py checks the CUDA boxes against them."""
from __future__ import annotations

import importlib.machinery
import sys
import tempfile
import types
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from oracle import bbox_ref, ref_shim  # noqa: E402

GOLDEN = ROOT / "tests" / "golden"


def load_reference_with_morphology():
    """ref_shim.load_reference() with skimage.morphology mapped to the oracle/bbox_ref.py restatement (the shim alone
    stubs it with functions that must never be called). The stand-in modules are removed again after the import."""
    added = []
    try:
        import skimage.morphology  # noqa: F401
    except Exception:
        for name, attrs in (("skimage", {}), ("skimage.morphology", {"binary_erosion": bbox_ref.binary_erosion,
                                                                     "binary_dilation": bbox_ref.binary_dilation})):
            m = types.ModuleType(name)
            m.__spec__ = importlib.machinery.ModuleSpec(name, loader=None)
            for k, v in attrs.items():
                setattr(m, k, v)
            sys.modules[name] = m
            added.append(name)
    try:
        ref = ref_shim.load_reference()
    finally:
        for name in added:
            sys.modules.pop(name, None)
    if added:
        assert ref.utils.binary_erosion is bbox_ref.binary_erosion, \
            "the reference was imported before the morphology restatement was installed"
    return ref


def semantic_label_maps():
    """Small label maps for the box / semantic-map fixtures: segments touching the border, a one-pixel-wide segment that
    erosion would empty, a one-pixel segment, a {0, 255} binary map and a seeded random blob map."""
    a = np.zeros((9, 12), np.uint8)
    a[:4, :5] = 1              # top-left corner block (touches two borders)
    a[5:, 3:11] = 2            # touches the bottom border
    a[1:8, 8] = 3              # one pixel wide: every erosion empties it
    a[7, 1] = 7                # one pixel
    a[0, 11] = 9               # one pixel in the corner
    b = np.zeros((8, 10), np.uint8)
    b[2:6, 3:9] = 255          # binary foreground saved as 255
    rng = np.random.default_rng(5)
    c = np.zeros((13, 11), np.uint8)
    for v in range(1, 6):
        y, x = rng.integers(0, 13), rng.integers(0, 11)
        h, w = rng.integers(2, 7), rng.integers(2, 7)
        c[y:y + h, x:x + w] = v
    return {"corners": a, "binary": b, "blobs": c}


BBOX_CASES = [  # num_erode, num_dilate, skip_bg_index, downsample_factor
    (2, 3, True, None), (1, 2, False, None), (0, 0, True, 8), (3, 5, True, None), (2, 5, False, 16)]


def make_semantic_golden():
    """Outputs of the reference's own _extract_bbox, extract_bbox_clusters and extract_semantic_segmentations on small
    seeded inputs (skimage's morphology through the oracle/bbox_ref.py restatement, real scikit-learn)."""
    import os
    from PIL import Image
    os.environ["TORCH_FORCE_NO_WEIGHTS_ONLY_LOAD"] = "1"   # the reference's torch.load calls predate weights_only
    ref = load_reference_with_morphology()
    maps = semantic_label_maps()
    boxes = {}
    with tempfile.TemporaryDirectory() as td:
        fdir, sdir = Path(td) / "f", Path(td) / "s"
        fdir.mkdir(); sdir.mkdir()
        for name, m in maps.items():
            P = 16
            torch.save({"k": torch.zeros(1, m.size, 4), "indices": torch.tensor(0), "file": f"{name}.jpg", "id": name,
                        "model_name": "dino_vits16", "patch_size": P, "shape": (1, 3, m.shape[0] * P + 5, m.shape[1] * P)},
                       fdir / f"{name}.pth")
            Image.fromarray(m).save(sdir / f"{name}.png")
        inputs = ref.utils.get_paired_input_files(str(fdir), str(sdir))
        for ci, (ne, nd, skip, ds) in enumerate(BBOX_CASES):
            for inp in inputs:
                out = ref._extract_bbox(inp, num_erode=ne, num_dilate=nd, skip_bg_index=skip, downsample_factor=ds)
                rows = [[s, *b, *o] for s, b, o in zip(out["segment_indices"], out["bboxes"],
                                                       out["bboxes_original_resolution"])]
                boxes[f"case{ci}_{out['id']}"] = np.array(rows, dtype=np.int64).reshape(-1, 9)
                boxes[f"types_case{ci}_{out['id']}"] = np.array(repr(
                    (type(out["segment_indices"][0]).__name__, type(out["bboxes"][0][0]).__name__,
                     type(out["bboxes_original_resolution"][0][0]).__name__, out["format"])))
    np.savez_compressed(GOLDEN / "ref_bboxes.npz", cases=np.array(repr(BBOX_CASES)),
                        **{f"map_{k}": v for k, v in maps.items()}, **boxes)

    # clusters: a well separated planted mixture (5 groups in 24 dims) spread over 12 box dicts
    g = np.random.default_rng(11)
    centres = g.normal(size=(5, 24)) * 4.0
    counts = g.integers(2, 9, size=12)
    truth = g.integers(0, 5, size=int(counts.sum()))
    feats = (centres[truth] + 0.05 * g.normal(size=(len(truth), 24))).astype(np.float32)
    bbox_list, o = [], 0
    for i, n in enumerate(counts.tolist()):
        bbox_list.append({"id": f"im{i}", "bboxes": [[0, 0, 1, 1]] * n, "bboxes_original_resolution": [[0, 0, 16, 16]] * n,
                          "segment_indices": list(range(1, n + 1)), "format": "(xmin, ymin, xmax, ymax)",
                          "features": torch.from_numpy(feats[o:o + n].copy())})
        o += n
    with tempfile.TemporaryDirectory() as td:
        torch.save(bbox_list, Path(td) / "feats.pth")
        ref.extract_bbox_clusters(str(Path(td) / "feats.pth"), str(Path(td) / "clusters.pth"), num_clusters=5, seed=0,
                                  pca_dim=4)
        out = torch.load(Path(td) / "clusters.pth", weights_only=False)
    np.savez_compressed(GOLDEN / "ref_bbox_clusters.npz", features=feats, counts=counts, truth=truth,
                        clusters=np.concatenate([d["clusters"] for d in out]),
                        cluster_dtype=np.array(str(out[0]["clusters"].dtype)),
                        has_features=np.array(any("features" in d for d in out)))

    # semantic maps: the skip_bg_index boxes of the label maps with seeded cluster ids
    sem = {}
    with tempfile.TemporaryDirectory() as td:
        sdir, odir = Path(td) / "s", Path(td) / "o"
        sdir.mkdir()
        bbox_list = []
        for j, (name, m) in enumerate(maps.items()):
            Image.fromarray(m).save(sdir / f"{name}.png")
            binary = set(np.unique(m).tolist()) <= {0, 255}
            vals = [v for v in np.unique((m > 0).astype(np.uint8) if binary else m).tolist() if v > 0]
            clusters = np.random.default_rng(30 + j).integers(0, 21, size=len(vals)).astype(np.int32)
            bbox_list.append({"id": name, "bboxes": [[0, 0, 1, 1]] * len(vals), "segment_indices": vals,
                              "clusters": clusters})
            sem[f"segment_indices_{name}"] = np.array(vals, dtype=np.int64)
            sem[f"clusters_{name}"] = clusters
        torch.save(bbox_list, Path(td) / "clusters.pth")
        ref.extract_semantic_segmentations(str(sdir), str(Path(td) / "clusters.pth"), str(odir))
        for name in maps:
            sem[f"semantic_{name}"] = np.array(Image.open(odir / f"{name}.png"))
    np.savez_compressed(GOLDEN / "ref_semantic_segmaps.npz", **{f"map_{k}": v for k, v in maps.items()}, **sem)
    print("semantic fixtures:", sorted(boxes)[:3], "...", np.bincount(out[0]["clusters"]) if len(out) else None)


if __name__ == "__main__":
    assert ref_shim.available(), "reference sources not present"
    make_semantic_golden()
