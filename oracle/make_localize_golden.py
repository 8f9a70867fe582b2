"""Writes tests/golden/ref_loc_*.npz by running the reference's OWN object localization code (object-localization/
object_discovery.py, datasets.py, main.py; read-only, dev container only) under stubs for what is not installed:

  skimage.measure.label -> scipy.ndimage.label with ones((3, 3)) (skimage's default connectivity = ndim)
  skimage.io, traitlets, matplotlib, dino.vision_transformer (-> the oracle ViT), torch.hub.load_state_dict_from_url
  (-> a seeded state dict); Tensor.cuda is a no-op on a GPU-less box (as ref_shim.py does).

The fixtures hold data only: inputs, the reference's outputs, and the tree of the end-to-end run (annotation XML,
image sizes, eigenvectors), which the tests rebuild in a temporary directory.

    python -m oracle.make_localize_golden
"""
from __future__ import annotations

import contextlib
import io
import os
import pickle
import sys
import tempfile
from pathlib import Path

import numpy as np
import scipy.ndimage
import torch

from . import dino_vit, localize_ref
from .ref_shim import _stub

REF_DIR = Path("/root/reference/object-localization")
GOLDEN = Path(__file__).resolve().parents[1] / "tests" / "golden"
_mods = None


def load_reference():
    """(object_discovery, datasets, main) of the reference, imported under the stubs."""
    global _mods
    if _mods is not None:
        return _mods

    def _never(*a, **k):
        raise RuntimeError("stubbed dependency called")

    _stub("skimage")
    _stub("skimage.io", imread=_never)
    _stub("skimage.measure", label=lambda m: scipy.ndimage.label(m, structure=localize_ref.EIGHT)[0])
    _stub("traitlets")
    _stub("traitlets.traitlets", default=_never)
    _stub("matplotlib")
    _stub("matplotlib.pyplot")

    def vit(name):
        def make(patch_size=16, num_classes=0):
            return dino_vit.build(name.replace("16", str(patch_size)), seed=0)
        return make

    _stub("dino")
    _stub("dino.vision_transformer", vit_small=vit("dino_vits16"), vit_base=vit("dino_vitb16"))
    torch.hub.load_state_dict_from_url = lambda url, **k: dino_vit.build(
        {"deitsmall16": "dino_vits16", "deitsmall8": "dino_vits8", "vitbase16": "dino_vitb16",
         "vitbase8": "dino_vitb8"}[url.split("/")[-1].split("_")[1]], seed=0).state_dict()
    if not torch.cuda.is_available():
        torch.Tensor.cuda = lambda self, *a, **k: self
    sys.path.insert(0, str(REF_DIR))
    try:
        import datasets as ref_datasets
        import main as ref_main
        import object_discovery as ref_od
    finally:
        sys.path.remove(str(REF_DIR))
    _mods = (ref_od, ref_datasets, ref_main)
    return _mods


def _pack(arrays):
    flat = np.concatenate([np.asarray(a).reshape(-1) for a in arrays]) if arrays else np.zeros(0)
    offs = np.cumsum([0] + [np.asarray(a).size for a in arrays]).astype(np.int64)
    return flat, offs


def _blob_vector(rng, h, w, n_blobs=2):
    yy, xx = np.mgrid[0:h, 0:w]
    v = rng.normal(0, 0.3, (h, w))
    for _ in range(n_blobs):
        cy, cx, r = rng.uniform(0, h), rng.uniform(0, w), rng.uniform(1, max(h, w) / 2)
        v += np.exp(-((yy - cy) ** 2 + (xx - cx) ** 2) / (2 * r * r)) * rng.choice([-2, 2])
    return v.astype(np.float32).reshape(-1)


def make_eigseg(ref_od, rng):
    cases = []   # (H, W, v)
    for (H, W) in [(375, 500), (333, 500), (224, 224), (100, 37), (61, 250)]:
        for P in (8, 16):
            cases.append((H, W, _blob_vector(rng, H // P, W // P)))
        cases.append((H, W, _blob_vector(rng, 2 * (H // 16), 2 * (W // 16))))     # the third case (P 8 on a P 16 grid)
        cases.append((H, W, _blob_vector(rng, 4 * (H // 32), 4 * (W // 32))))     # the fourth case
    cases.append((64, 64, -np.ones(64, np.float32)))                 # empty mask: the whole image
    cases.append((64, 64, np.ones(64, np.float32)))                  # full mask (mean 1: not flipped)
    v = -np.ones((8, 8), np.float32); v[:5, :] = 1                   # mean 0.625: flipped
    cases.append((64, 64, v.reshape(-1)))
    v = -np.ones((8, 8), np.float32); v[:4, :] = 1                   # mean exactly 0.5: not flipped
    cases.append((64, 64, v.reshape(-1)))
    v = -np.ones((8, 8), np.float32); v[0, 0:2] = 1; v[5, 5:7] = 1; v[7, 0:2] = 1   # three components of size 2: tie
    cases.append((64, 64, v.reshape(-1)))
    v = -np.ones((6, 6), np.float32); v[1, 1] = 1; v[2, 2] = 1; v[3, 1] = 1          # diagonal contacts: 8-connected
    cases.append((96, 96, v.reshape(-1)))
    cases.append((16, 16, np.ones(1, np.float32)))                   # 1 x 1
    cases.append((50, 50, np.ones(7, np.float32)))                   # no grid with 7 cells
    for _ in range(30):                                              # random masks over densities
        H, W = int(rng.integers(16, 400)), int(rng.integers(16, 400))
        P = int(rng.choice([8, 16]))
        dens = rng.uniform(0.05, 0.95)
        cases.append((H, W, np.where(rng.random((H // P) * (W // P)) < dens, 1.0, -1.0).astype(np.float32)))
    boxes, err = [], []
    for H, W, v in cases:
        try:
            b = np.asarray(ref_od.get_bbox_from_patch_mask(torch.from_numpy(v > 0), (3, H, W)), dtype=np.int64)
            e = False
        except ValueError:
            b, e = np.zeros(4, np.int64), True
        if not e:
            assert np.array_equal(b, localize_ref.eigseg_box(v, H, W)), (H, W)
        boxes.append(b); err.append(e)
    flat, offs = _pack([c[2] for c in cases])
    np.savez_compressed(GOLDEN / "ref_loc_eigseg.npz", v=flat.astype(np.float32), offs=offs,
                        H=np.array([c[0] for c in cases]), W=np.array([c[1] for c in cases]), boxes=np.stack(boxes),
                        err=np.array(err))
    return len(cases)


def make_lost(ref_od, rng):
    cases = []   # (feats [N, d] int-valued, gh, gw, H, W, P, k)
    for (H, W, P, d, k) in [(60, 90, 16, 16, 100), (100, 37, 8, 8, 100), (64, 64, 16, 32, 100), (45, 70, 8, 24, 5),
                            (333, 500, 16, 16, 100), (48, 48, 16, 8, 100), (200, 150, 16, 64, 1000)]:
        gh, gw = -(-H // P), -(-W // P)
        for _ in range(3):
            f = rng.integers(-4, 5, (gh * gw, d)).astype(np.float32)
            cases.append((f, gh, gw, H, W, P, k))
    # a zero seed feature: no similar patch, M[seed] = 0 -> the seed is in the background
    f = rng.integers(-4, 5, (12, 8)).astype(np.float32); f[5] = 0
    cases.append((f, 3, 4, 40, 60, 16, 100))
    boxes, seeds, err = [], [], []
    kept = []
    for f, gh, gw, H, W, P, k in cases:
        feats = torch.from_numpy(f)[None]
        try:
            pred, A, M, scores, seed = ref_od.lost(feats, (gh, gw), [P, P], (3, H, W), k_patches=k)
            b, s, e = np.asarray(pred, dtype=np.int64), int(seed), False
        except ValueError as ex:
            assert "background" in str(ex)
            b, s, e = np.zeros(4, np.int64), int(localize_ref.lost_order(f @ f.T)[0]), True
        # the reference's unstable argsort must agree with the stable-ties restatement on every kept fixture
        A = f @ f.T
        if e:
            try:
                localize_ref.lost_box(A, (gh, gw), (H, W), P, k)
                agree = False
            except ValueError:
                agree = True
        else:
            ob, os_ = localize_ref.lost_box(A, (gh, gw), (H, W), P, k)
            agree = np.array_equal(ob, b) and os_ == s
        if not agree:
            continue
        kept.append((f, gh, gw, H, W, P, k)); boxes.append(b); seeds.append(s); err.append(e)
    # the fixtures are the cases where the two orders agree; the seed-in-background case must be among them
    assert len(kept) >= len(cases) // 2 and err[-1], f"stable ties disagree with the reference on {len(cases) - len(kept)} cases"
    flat, offs = _pack([c[0] for c in kept])
    np.savez_compressed(GOLDEN / "ref_loc_lost.npz", feats=flat.astype(np.float32), offs=offs,
                        d=np.array([c[0].shape[1] for c in kept]), gh=np.array([c[1] for c in kept]),
                        gw=np.array([c[2] for c in kept]), H=np.array([c[3] for c in kept]),
                        W=np.array([c[4] for c in kept]), P=np.array([c[5] for c in kept]),
                        k=np.array([c[6] for c in kept]), boxes=np.stack(boxes), seeds=np.array(seeds), err=np.array(err))
    return len(kept), len(cases)


def _cells(gh, gw, rects):
    m = np.zeros((gh, gw), bool)
    for y0, y1, x0, x1 in rects:
        m[y0:y1, x0:x1] = True
    return m.reshape(-1)


def _attn_with_kept(rng, kept, heads):
    """Attention rows whose kept set (cumulative mass of the ascending values > 0.4) is exactly `kept`: the others
    have value ~1 and total mass <= 0.4 of the row, each kept value ~b with the first one crossing 0.4."""
    nb, nk = int((~kept).sum()), int(kept.sum())
    b = 1.575 * nb / nk
    assert nk <= 2 or b < 0.6 * nb / (0.4 * nk - 1)
    rows = []
    for _ in range(heads):
        a = np.where(kept, b, 1.0) * (1 + 1e-4 * rng.random(kept.size))
        rows.append(a / a.sum())
    return np.asarray(rows, np.float32)


def make_dinoseg(ref_od, rng):
    cases = []   # (attn [heads, N], gh, gw, P, head)
    for (gh, gw, P, heads) in [(24, 32, 16, 6), (31, 40, 8, 6), (14, 14, 16, 12), (5, 9, 8, 6)]:
        for _ in range(3):
            s = rng.normal(0, 2, (heads, gh * gw))
            a = np.exp(s) / np.exp(s).sum(1, keepdims=True)
            cases.append((a.astype(np.float32), gh, gw, P, int(rng.integers(0, heads))))
    # hand-made kept sets, values distinct (the order of tied values is unspecified in the reference's sort)
    for kept, P, head in [(_cells(8, 8, [(2, 5, 2, 5)]), 16, 4),                   # n = 1: label 0, the background
                          (_cells(8, 8, [(0, 1, 0, 1), (4, 8, 4, 8)]), 16, 4),     # n = 2, the uncounted one larger
                          (_cells(8, 8, [(0, 1, 0, 2), (3, 4, 0, 5), (6, 8, 6, 8)]), 8, 1)]:   # n = 3
        cases.append((_attn_with_kept(rng, kept, 6), 8, 8, P, head))
    # every patch kept (1 x 2 grid): the selected background is empty
    cases.append((np.array([[0.5, 0.5]] * 6, np.float32), 1, 2, 16, 0))
    boxes, err = [], []
    for a, gh, gw, P, head in cases:
        attn = torch.from_numpy(a)[None, :, None, :].expand(1, a.shape[0], 2, a.shape[1])
        attn = torch.cat([torch.zeros(1, a.shape[0], 2, 1), attn], dim=3).contiguous()   # the CLS column, dropped
        try:
            b, e = np.asarray(ref_od.dino_seg(attn, (gh, gw), P, head=head), dtype=np.int64), False
        except ValueError:
            b, e = np.zeros(4, np.int64), True
        if not e:
            assert np.array_equal(b, localize_ref.dinoseg_box(a[head], (gh, gw), P))
        boxes.append(b); err.append(e)
    flat, offs = _pack([c[0] for c in cases])
    np.savez_compressed(GOLDEN / "ref_loc_dinoseg.npz", attn=flat.astype(np.float32), offs=offs,
                        heads=np.array([c[0].shape[0] for c in cases]), gh=np.array([c[1] for c in cases]),
                        gw=np.array([c[2] for c in cases]), P=np.array([c[3] for c in cases]),
                        head=np.array([c[4] for c in cases]), boxes=np.stack(boxes), err=np.array(err))
    return len(cases)


def make_iou(ref_datasets, rng):
    """Boxes whose IoU with a GT box is within a few float32 ulps of 0.5, and the reference's float32 IoUs."""
    preds, gts, ious = [], [], []
    while len(preds) < 200:
        p = np.sort(rng.integers(0, 60, (2, 2)), axis=0).T.reshape(-1)[[0, 2, 1, 3]]
        g = np.sort(rng.integers(0, 60, (2, 2)), axis=0).T.reshape(-1)[[0, 2, 1, 3]]
        if p[2] <= p[0] or p[3] <= p[1] or g[2] <= g[0] or g[3] <= g[1]:
            continue
        if abs(localize_ref.iou_float64(p, g)[0] - 0.5) > 2e-7:
            continue
        preds.append(p.astype(np.int64)); gts.append(g.astype(np.int64))
        ious.append(float(ref_datasets.bbox_iou(torch.from_numpy(preds[-1]), torch.from_numpy(gts[-1][None]))[0]))
    np.savez_compressed(GOLDEN / "ref_loc_iou.npz", pred=np.stack(preds), gt=np.stack(gts), iou=np.array(ious, np.float32))
    return len(preds)


# ------------------------------------------------------------------------------------------------ end to end
SIZES = [(375, 500), (333, 500), (500, 375), (360, 480), (375, 500), (64, 48), (281, 500), (500, 333)]
CLASSES = ["dog", "cat", "person", "car", "bird"]


def voc_xml(name, H, W, objects):
    objs = "".join(
        f"<object><name>{c}</name><pose>Unspecified</pose><truncated>{t}</truncated><difficult>{d}</difficult>"
        f"<bndbox><xmin>{x0}</xmin><ymin>{y0}</ymin><xmax>{x1}</xmax><ymax>{y1}</ymax></bndbox></object>"
        for c, t, d, x0, y0, x1, y1 in objects)
    return (f"<annotation><folder>VOC2007</folder><filename>{name}</filename><size><width>{W}</width>"
            f"<height>{H}</height><depth>3</depth></size><segmented>0</segmented>{objs}</annotation>")


def synthetic_tree(rng):
    ids, xmls, eigs = [], [], []
    for i, (H, W) in enumerate(SIZES):
        iid = f"{i * 7 + 5:06d}"
        objs = []
        for _ in range(int(rng.integers(1, 4))):
            x0, x1 = sorted(rng.integers(1, W + 1, 2)); y0, y1 = sorted(rng.integers(1, H + 1, 2))
            objs.append((str(rng.choice(CLASSES)), int(rng.random() < 0.3), int(rng.random() < 0.2), int(x0), int(y0),
                         int(max(x1, x0 + 1)), int(max(y1, y0 + 1))))
        if i == 2:   # only hard objects: dropped under --no_hard
            objs = [(c, 1, d, *b) for c, t, d, *b in objs]
        ids.append(iid)
        xmls.append(voc_xml(f"{iid}.jpg", H, W, objs))
        P = 16 if i % 3 else 8
        ev = np.stack([_blob_vector(rng, H // P, W // P) for _ in range(3)])
        eigs.append(ev.astype(np.float32))
    return ids, xmls, eigs


def build_tree(root: Path, ids, xmls, sizes, eigs, eig_dir_name="laplacian_dino_vits16"):
    """VOCdevkit/VOC2007 tree under root/datasets/VOC2007 and the eigenvector files (also used by the tests)."""
    from PIL import Image
    voc = root / "datasets" / "VOC2007" / "VOCdevkit" / "VOC2007"
    for sub in ("Annotations", "JPEGImages", "ImageSets/Main"):
        (voc / sub).mkdir(parents=True, exist_ok=True)
    (voc / "ImageSets" / "Main" / "trainval.txt").write_text("".join(f"{i}\n" for i in ids))
    edir = root / eig_dir_name
    edir.mkdir(parents=True, exist_ok=True)
    for i, x, (H, W), ev in zip(ids, xmls, sizes, eigs):
        (voc / "Annotations" / f"{i}.xml").write_text(x)
        Image.new("RGB", (int(W), int(H)), (90, 120, 150)).save(voc / "JPEGImages" / f"{i}.jpg")
        torch.save({"eigenvalues": torch.zeros(ev.shape[0]), "eigenvectors": torch.from_numpy(ev)}, edir / f"{i}.pth")
    return root / "datasets" / "VOC2007", edir


def run_reference_main(ref_main, cwd: Path, argv):
    old_cwd, old_argv = os.getcwd(), sys.argv
    os.chdir(cwd)
    sys.argv = ["main.py"] + argv
    try:
        with contextlib.redirect_stdout(io.StringIO()), contextlib.redirect_stderr(io.StringIO()):
            ref_main.main()
    finally:
        os.chdir(old_cwd)
        sys.argv = old_argv


def make_main(ref_main, rng):
    ids, xmls, eigs = synthetic_tree(rng)
    out = {"ids": np.array(ids), "sizes": np.array(SIZES), "xml": np.array(xmls)}
    flat, offs = _pack(eigs)
    out.update(eigs=flat.astype(np.float32), eig_offs=offs, eig_K=np.array([e.shape[0] for e in eigs]))
    for tag, extra in (("hard", []), ("nohard", ["--no_hard"])):
        with tempfile.TemporaryDirectory() as td:
            td = Path(td)
            _, edir = build_tree(td, ids, xmls, SIZES, eigs)
            run_reference_main(ref_main, td, ["--eigenseg", "--precomputed_eigs_dir", str(edir), "--output_dir",
                                              str(td / "outputs")] + extra)
            name = "VOC07_trainval" + ("-nohards" if extra else "")
            folder = td / "outputs" / name / "LOST-vit_small16_k"
            preds = pickle.loads((folder / "preds.pkl").read_bytes())
            gt = pickle.loads((folder / "gt.pkl").read_bytes())
            out[f"{tag}_names"] = np.array(list(preds))
            out[f"{tag}_preds"] = np.stack([preds[k] for k in preds])
            gflat, goffs = _pack([gt[k] for k in preds])
            out[f"{tag}_gt"], out[f"{tag}_gt_offs"] = gflat.astype(np.int64), goffs
            out[f"{tag}_results"] = np.frombuffer((folder / "results.txt").read_bytes(), dtype=np.uint8)
    np.savez_compressed(GOLDEN / "ref_loc_main.npz", **out)
    return len(ids)


def main():
    ref_od, ref_datasets, ref_main = load_reference()
    rng = np.random.default_rng(20261015)
    print("eigseg cases", make_eigseg(ref_od, rng))
    print("lost cases (kept, generated)", make_lost(ref_od, rng))
    print("dinoseg cases", make_dinoseg(ref_od, rng))
    print("iou cases", make_iou(ref_datasets, rng))
    print("main images", make_main(ref_main, rng))


if __name__ == "__main__":
    main()
