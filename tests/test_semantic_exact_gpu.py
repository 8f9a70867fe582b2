"""-m gpu: the semantic-segmentation stages exactly (extract_bboxes -> extract_bbox_features -> extract_bbox_clusters).

- Segment boxes bit for bit against the scipy restatement of the reference (oracle/bbox_ref.py) at every grid edge the
  kernel supports (1 x 1, 1 x 16384, 16384 x 1, 2 x 8192, 127 x 129, 128 x 128), on hand-built maps (every label
  value, only 0 / 255, 1-pixel lines, checkerboards, squares that erosion empties at a chosen step, segments on every
  border), at morphology counts past the point where the masks stop changing, and in batches many waves deep. Outputs
  land in sentinel-filled buffers with guard rows; a grid past 16384 cells is refused before anything is launched.
- Box-crop CLS features: with a zero patch embedding, forward_tokens(img, 0) is exactly CLS + the positional embedding,
  compared with the upstream restatement on UNCROPPED pixel sizes (a 14 x 14 patch grid from a 224 x 232 crop is
  resampled upstream; the library used to hand it the stored grid). extract_bbox_features on JPEG sets whose boxes come
  from extract_bboxes at downsample factors 16 and 8: every row bitwise forward_cls of its crop alone, in (image, box)
  order, and within the fp32 oracle's 3e-3 on the crop fed uncropped.
- PCA against float64 numpy.linalg.eigh of the same float32 rows: Rayleigh quotients against the top eigenvalues,
  residuals, orthonormality and Davis-Kahan subspace angles, at d 65 / 384 / 768 and pca_dim 1 / 32 / 64 on power-law,
  clustered (equal, 1e-3 and 1e-6 apart across the cut) and L2-normalised spectra; the solver's retry with the largest
  Krylov space; rank-deficient data.
- extract_bbox_clusters composed exactly: the K-means oracle of tests/test_kmeans_gpu.py run on the device's own PCA
  output must give the same labels, centres and iteration count."""
import numpy as np
import pytest
import torch
from PIL import Image

from conftest import load_pkg
from oracle import bbox_ref
from test_kmeans_gpu import _oracle
from test_semantic_gpu import _rows

pytestmark = pytest.mark.gpu

SENT = -12345
GUARD = 3


# ------------------------------------------------------------------------------------------------- segment boxes
def _raw_boxes(maps_dev, ne, nd, B=None):
    """dss_segment_bboxes into sentinel buffers with GUARD images of guard rows; returns (rc, boxes, present) after
    checking the guards."""
    _lib = load_pkg("_lib")
    B = maps_dev.shape[0] if B is None else B
    H, W = maps_dev.shape[1:]
    boxes = torch.full(((B + GUARD) * 256 * 4,), SENT, dtype=torch.int32, device=maps_dev.device)
    present = torch.full(((B + GUARD) * 256,), 0xA5, dtype=torch.uint8, device=maps_dev.device)
    rc = _lib.load().dss_segment_bboxes(maps_dev.data_ptr(), B, H, W, ne, nd, boxes.data_ptr(), present.data_ptr(),
                                        _lib.stream_ptr(maps_dev.device))
    torch.cuda.synchronize()
    assert (boxes[B * 1024:] == SENT).all(), "a guard row after the boxes changed"
    assert (present[B * 256:] == 0xA5).all(), "a guard row after the presence flags changed"
    return rc, boxes[:B * 1024].view(B, 256, 4).cpu().numpy(), present[:B * 256].view(B, 256).cpu().numpy()


def _oracle_rows(m, ne, nd):
    """(rows with skip_bg_index=False, rows with True): the reference skips segment 0 and nothing else."""
    rows = _rows(bbox_ref.extract_bbox(m, "x", 16, ne, nd, False))
    return rows, rows[rows[:, 0] != 0]


def _check_maps(maps, boxes, present, ne, nd, what):
    ex = load_pkg("extract")
    for b, m in enumerate(maps):
        assert np.array_equal(np.flatnonzero(present[b]), np.unique(m)), (what, b)
        assert np.all(boxes[b][present[b] == 0] == 0), (what, b)          # absent values get zero boxes
        want_all, want_skip = _oracle_rows(m, ne, nd)
        for skip, want in ((False, want_all), (True, want_skip)):
            got = ex._bbox_dict("x", 16, boxes[b], present[b].astype(bool), skip)
            assert np.array_equal(_rows(got), want), (what, b, ne, nd, skip)


MORPH = [(0, 0), (0, 2), (2, 0), (1, 1), (2, 3), (3, 1), (5, 0), (0, 5)]
GRIDS = [(1, 1), (1, 16384), (16384, 1), (2, 8192), (127, 129), (128, 128)]


@pytest.mark.parametrize("H,W", GRIDS)
def test_segment_boxes_at_grid_edges(cuda, H, W):
    """Every hand-built map of oracle.bbox_ref.edge_maps, through cluster.segment_bboxes and extract._bbox_dict, with
    and without skip_bg_index. The squares have sides 1, 3, ..., so num_erode = 5 empties them at steps 1 to 5 (the
    side-9 square at the last step) and the kernel must keep the last non-empty mask; (40, 0) / (0, 40) run far past
    the point where the masks stop changing (a 128-cell strip fills after 127 dilations, so (0, 200) on 1 x 128)."""
    cluster = load_pkg("cluster")
    names, maps = zip(*bbox_ref.edge_maps(H, W, seed=H * 7 + W).items())
    maps = np.stack(maps)
    dev = torch.from_numpy(maps).to(cuda)
    morph = MORPH + ([(40, 0), (0, 40), (40, 40)] if H * W <= 128 * 129 and min(H, W) > 2 else [(40, 0), (12, 12)])
    for ne, nd in morph:
        boxes, present = cluster.segment_bboxes(dev, ne, nd)
        _check_maps(maps, boxes.cpu().numpy(), present.cpu().numpy(), ne, nd, (H, W, names))
        rc, raw_boxes, raw_present = _raw_boxes(dev, ne, nd)             # the same bits into guarded buffers
        assert rc == 0
        assert np.array_equal(raw_boxes, boxes.cpu().numpy()) and np.array_equal(raw_present, present.cpu().numpy())
    if H == 1 and W == 16384:
        strip = np.stack([bbox_ref.edge_maps(1, 128, seed=1)[k] for k in ("squares", "lines", "border")])
        boxes, present = cluster.segment_bboxes(torch.from_numpy(strip).to(cuda), 0, 200)
        _check_maps(strip, boxes.cpu().numpy(), present.cpu().numpy(), 0, 200, "strip fill")


def test_segment_boxes_single_cells_and_border_rules(cuda):
    """Erosion counts pixels outside the image as set and dilation as unset, so a segment on a border survives erosion
    from that side and grows only inwards; an isolated cell erodes empty at step 1 and is kept. Hand-checked boxes."""
    cluster = load_pkg("cluster")
    m = np.zeros((6, 9), np.uint8)
    m[0, :] = 1          # the top row: survives any erosion (outside counts as set, the row below is 0 -> eroded)
    m[:, 8] = 2          # the right column
    m[3, 3] = 3          # an isolated cell
    m[5, 0:3] = 255      # the bottom-left run
    maps = m[None]
    boxes, present = cluster.segment_bboxes(torch.from_numpy(maps).to(cuda), 1, 0)
    boxes, present = boxes.cpu().numpy()[0], present.cpu().numpy()[0]
    _check_maps(maps, boxes[None], present[None], 1, 0, "hand")
    assert boxes[3].tolist() == [3, 3, 4, 4]                           # erosion emptied it: the step is discarded
    boxes, _ = cluster.segment_bboxes(torch.from_numpy(maps).to(cuda), 0, 1)
    assert boxes.cpu().numpy()[0, 3].tolist() == [2, 2, 5, 5]          # one dilation of the cross
    assert boxes.cpu().numpy()[0, 255].tolist() == [0, 4, 4, 6]        # grows up and right, not past the borders


def test_segment_boxes_many_waves_equal_solo_runs(cuda):
    """B = 48 maps of 128 x 128 (12 288 CTAs with 32 KB of shared memory each: many waves over the SMs), each image
    bitwise its solo run, and the batch against the oracle on a sample."""
    cluster = load_pkg("cluster")
    g = np.random.default_rng(5)
    pool = list(bbox_ref.edge_maps(128, 128, seed=3).values())
    maps = np.stack([pool[i % len(pool)] if i % 3 else g.integers(0, 256, size=(128, 128), dtype=np.uint8)
                     for i in range(48)])
    dev = torch.from_numpy(maps).to(cuda)
    sms = torch.cuda.get_device_properties(cuda).multi_processor_count
    assert 48 * 256 > 8 * sms
    rc, boxes, present = _raw_boxes(dev, 2, 3)
    assert rc == 0
    for b in range(48):
        _, one_b, one_p = _raw_boxes(dev[b:b + 1].contiguous(), 2, 3)
        assert np.array_equal(one_b[0], boxes[b]) and np.array_equal(one_p[0], present[b]), b
    _check_maps(maps[::7], boxes[::7], present[::7], 2, 3, "waves")


@pytest.mark.parametrize("H,W", [(1, 16385), (16385, 1), (129, 128), (128, 129)])
def test_segment_boxes_refuse_grids_past_16384_cells(cuda, H, W):
    """16 385 cells and more: DSS_ERR_UNSUPPORTED, no kernel launched, the output buffers untouched."""
    _lib = load_pkg("_lib")
    maps = torch.zeros(2, H, W, dtype=torch.uint8, device=cuda)
    boxes = torch.full((2 * 256 * 4,), SENT, dtype=torch.int32, device=cuda)
    present = torch.full((2 * 256,), 0xA5, dtype=torch.uint8, device=cuda)
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    rc = _lib.load().dss_segment_bboxes(maps.data_ptr(), 2, H, W, 2, 3, boxes.data_ptr(), present.data_ptr(),
                                        _lib.stream_ptr(cuda))
    torch.cuda.synchronize()
    assert rc == _lib.DSS_ERR_UNSUPPORTED
    assert _lib.launch_count() == n0
    assert (boxes == SENT).all() and (present == 0xA5).all()
    assert b"16384" in _lib.load().dss_last_error()


# --------------------------------------------------------------------------------------------- positional embedding
# (H, W) pixel sizes, uncropped. The first two rows are the suspected case: a grid0 x grid0 patch grid from a
# non-square input, which upstream resamples with scale (grid0 + 0.1) / grid0. The others: square inputs (stored grid),
# 1 x n / n x 1, 196 patches as 7 x 28 / 28 x 7, grid0 +- 1, sizes that are not patch multiples.
POS_SIZES_16 = [(224, 232), (239, 224), (224, 224), (231, 231), (16, 16), (16, 17), (16, 400), (400, 31), (112, 448),
                (448, 127), (208, 208), (240, 255), (224, 232), (224, 224)]
POS_SIZES_8 = [(224, 231), (224, 224), (8, 640), (640, 15), (216, 216), (232, 239)]


@pytest.mark.parametrize("name,sizes", [("dino_vits16", POS_SIZES_16), ("dino_vitb8", POS_SIZES_8)])
def test_positional_embedding_of_uncropped_inputs(cuda, name, sizes):
    """Zero patch-embedding weight and bias: forward_tokens(img, 0) = [cls + pos[0], pos[1:]] in fp32, exactly the
    tokens upstream prepare_tokens builds before the first block. Sizes repeat in the list, so each call must get the
    table its own pixel sizes need, whatever the calls before it."""
    from oracle import dino_vit
    vit = load_pkg("vit")
    ref = dino_vit.build(name, seed=11)
    sd = {k: v.clone() for k, v in ref.state_dict().items()}
    sd["patch_embed.proj.weight"].zero_()
    sd["patch_embed.proj.bias"].zero_()
    mine = vit.DinoViT(name, sd, device=cuda)
    P, g = ref.cfg.patch, ref.cfg.grid0
    worst = 0.0
    for H, W in sizes:
        img = torch.randint(0, 256, (1, H, W, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(H * W))
        got = mine.forward_tokens(img.to(cuda), 0)[0].cpu()
        Hp, Wp = H // P, W // P
        pos = ref.interpolate_pos_encoding(Hp * Wp, H, W)[0]
        want = torch.cat([ref.cls_token[0] + pos[:1], pos[1:]])
        err = (got - want).abs().max().item()
        worst = max(worst, err / 2e-6)
        if Hp == g and Wp == g and H == W:
            assert torch.equal(got, want), (H, W)                          # the stored grid, bit for bit
        else:
            assert err <= 2e-6, (H, W, err)                                # the bicubic weights' fp32 rounding
        if Hp == g and Wp == g and H != W:
            assert (want[1:] - ref.pos_embed[0, 1:]).abs().max().item() > 1e-4   # upstream really resamples
    print(f"{name}: worst |pos error| / 2e-6 = {worst:.3f}")


# -------------------------------------------------------------------------------------------- box-crop CLS features
def _crop_layouts(ds):
    """(pixel H, W, label map at 1/ds) per image; label blocks chosen so that crop shapes repeat across images, and at
    ds = 8 include 224 x 232 and 232 x 224 crops (14 x 14 patches, non-square pixels), 1 x n and n x 1 patch grids."""
    if ds == 8:
        m0 = np.zeros((32, 32), np.uint8); m0[0:28, 0:29] = 1; m0[2:6, 2:6] = 2; m0[29:32, :] = 3; m0[0:28, 30:32] = 4
        m1 = np.zeros((30, 40), np.uint8); m1[0:4, 0:4] = 5; m1[10:14, 10:14] = 6; m1[20:30, :] = 7; m1[5:9, 20:24] = 8
        m2 = np.zeros((29, 28), np.uint8); m2[:, :] = 9; m2[0:4, 0:4] = 10
        m3 = np.zeros((28, 28), np.uint8); m3[:, :] = 11; m3[8:12, 8:12] = 12
        return [(256, 256, m0), (240, 320, m1), (232, 224, m2), (224, 224, m3)]
    assert ds == 16
    m0 = np.zeros((16, 16), np.uint8); m0[0:14, 0:15] = 1; m0[2:4, 2:4] = 2; m0[15:16, :] = 3
    m1 = np.zeros((15, 20), np.uint8); m1[0:2, 0:2] = 5; m1[5:7, 5:7] = 6; m1[10:15, :] = 7; m1[3:5, 10:12] = 8
    m2 = np.zeros((14, 14), np.uint8); m2[:, :] = 9; m2[0:2, 0:2] = 10
    return [(256, 256, m0), (240, 320, m1), (224, 224, m2)]


@pytest.mark.parametrize("ds", [16, 8])
def test_extract_bbox_features_rows_are_solo_crops(cuda, tmp_path, ds):
    from oracle import dino_vit
    ex = load_pkg("extract"); vit = load_pkg("vit"); synth = load_pkg("synth")
    images, fdir, sdir = tmp_path / "images", tmp_path / "f", tmp_path / "s"
    for d in (images, fdir, sdir):
        d.mkdir()
    for i, (H, W, m) in enumerate(_crop_layouts(ds)):
        name = f"im{i}"
        Image.fromarray(synth.blobs_image(H, W, 70 + i).numpy()).save(images / f"{name}.jpg", quality=92)
        assert m.shape == (H // ds, W // ds)
        torch.save({"id": name, "patch_size": 16, "shape": (1, 3, H, W), "k": torch.zeros(1)}, fdir / f"{name}.pth")
        Image.fromarray(m).save(sdir / f"{name}.png")
    ex.extract_bboxes(str(fdir), str(sdir), str(tmp_path / "boxes.pth"), num_erode=0, num_dilate=0,
                      downsample_factor=ds)
    ex.extract_bbox_features(str(images), str(tmp_path / "boxes.pth"), "dino_vits16", str(tmp_path / "feats.pth"),
                             seed=0, batch_size=2)
    out = torch.load(tmp_path / "feats.pth", weights_only=False)
    model = vit.get_model("dino_vits16", seed=0, device=cuda)[0]
    ref = dino_vit.DinoViT(dino_vit.cfg_for("dino_vits16")).eval()
    ref.load_state_dict(vit.random_state_dict("dino_vits16", 0))
    ref = ref.to(cuda)
    shapes, checked, worst = {}, {}, 0.0
    for d in out:
        image = torch.from_numpy(np.asarray(Image.open(images / f"{d['id']}.jpg").convert("RGB")).copy())
        f = d["features"]
        assert f.dtype == torch.float32 and tuple(f.shape) == (len(d["bboxes"]), 384)
        for j, (x0, y0, x1, y1) in enumerate(d["bboxes_original_resolution"]):
            crop = image[y0:y1, x0:x1].contiguous()
            shapes[tuple(crop.shape[:2])] = shapes.get(tuple(crop.shape[:2]), 0) + 1
            solo = model.forward_cls(crop[None].to(cuda)).cpu()[0]
            assert torch.equal(f[j], solo), (d["id"], j, tuple(crop.shape))
            if checked.get(tuple(crop.shape[:2]), 0) < 2:
                checked[tuple(crop.shape[:2])] = checked.get(tuple(crop.shape[:2]), 0) + 1
                want = ref(dino_vit.preprocess_u8(crop, 1).to(cuda))[0].cpu()      # uncropped, as the reference
                rel = ((f[j] - want).norm() / want.norm()).item()
                worst = max(worst, rel / 3e-3)
                assert rel <= 3e-3, (d["id"], j, tuple(crop.shape), rel)
    assert max(shapes.values()) > 2                                  # one shape spans more than one batch of 2
    if ds == 8:
        assert {(224, 232), (232, 224), (224, 224), (24, 256), (224, 16)} <= set(shapes)
    print(f"ds {ds}: crop shapes {shapes}; worst CLS rel-L2 / 3e-3 = {worst:.3f}")


# ------------------------------------------------------------------------------------------------------------- PCA
# |Rayleigh quotient - lambda_i| <= EIG_TOL ||C|| and ||C v - rho v|| <= RESID_TOL ||C||, each plus the measured
# ||C_device - C_float64||_2. The solver stops when its residual estimate is <= tol * anorm, tol = 1e-6, with
# anorm = max(1, max_j |alpha_j| + beta_j) <= 2 ||C|| once pca_components has scaled C so that ||C|| >= 1: at most
# 2e-6 ||C||. RESID_TOL = 5 x that leaves room for the fp32 rounding of the matrix-vector products and of the vectors.
# (Without the scaling the 1 in anorm makes the stop absolute: 2e-4 ||C|| on L2-normalised rows at d = 384.)
SOLVER_TOL = 1e-6
EIG_TOL = 1e-5
RESID_TOL = 5 * 2 * SOLVER_TOL
ORTH_TOL = 1e-5


def _rows_with_spectrum(lam, M, seed, offset=0.5):
    """float32 rows whose sample covariance (ddof 1) is Q diag(lam) Q^T up to their float32 rounding."""
    g = np.random.default_rng(seed)
    d = len(lam)
    U = np.linalg.qr(np.concatenate([np.ones((M, 1)), g.normal(size=(M, d))], axis=1))[0][:, 1:]   # centred columns
    Q = np.linalg.qr(g.normal(size=(d, d)))[0]
    return ((U * np.sqrt(lam * (M - 1))) @ Q.T + offset).astype(np.float32)


def _spectrum(kind, d, p):
    i = np.arange(1, d + 1, dtype=np.float64)
    lam = i ** -1.5
    if kind == "power":
        return lam
    gap = {"equal": 0.0, "gap1e-3": 1e-3, "gap1e-6": 1e-6}[kind]
    lo, hi = max(0, p - 3), min(d, p + 3)                           # a cluster of 6 straddling the cut at p
    lam[lo:hi] = lam[lo] * (1.0 - gap * np.arange(hi - lo))
    return lam


def _check_components(X, V, p, what, cov=None):
    """V [p, d] (device) against numpy.linalg.eigh of the float64 covariance of the same float32 rows. The solver works
    on the device's fp32 covariance ``cov`` [d, >= d], so the eigenvalue and residual bounds add its measured distance
    ||C_device - C||_2 to the solver's 1e-5 ||C||. Returns the worst error / tolerance ratio per check."""
    C = np.cov(X.astype(np.float64), rowvar=False)
    lam, U = np.linalg.eigh(C)
    lam, U = lam[::-1], U[:, ::-1]
    V = V.astype(np.float64)
    assert V.shape == (p, C.shape[0]) and np.isfinite(V).all(), what
    norm = lam[0]
    d = C.shape[0]
    dC = 0.0 if cov is None else np.linalg.norm(cov.cpu().numpy()[:, :d].astype(np.float64) - C, 2)
    rho = np.einsum("id,de,ie->i", V, C, V)
    R = C @ V.T - V.T * rho                                           # [d, p] residual columns
    ratios = {"eig": np.abs(rho - lam[:p]).max() / (EIG_TOL * norm + dC),
              "resid": np.linalg.norm(R, axis=0).max() / (RESID_TOL * norm + dC),
              "orth": np.abs(V @ V.T - np.eye(p)).max() / ORTH_TOL}
    gap = rho.min() - lam[p] if p < len(lam) else 0.0
    if gap > 10 * np.linalg.norm(R):                                  # a clear gap after pca_dim: Davis-Kahan sin(theta)
        sin = np.linalg.svd(U[:, p:].T @ V.T, compute_uv=False).max()
        ratios["dk"] = sin / (np.linalg.norm(R) / gap * 1.01 + 1e-12)
    for k, r in ratios.items():
        assert r <= 1.0, (what, k, r)
    return ratios


# Six eigenvalues equal or 1e-6 apart across the cut: the single-vector Lanczos of dss_eigsh_topk reports convergence
# before it has resolved every copy, so pca_components returns vectors from below the cluster in place of copies and
# the top-p Rayleigh quotients fall short of the float64 eigenvalues by far more than EIG_TOL. The solver's restart
# handles exact Lanczos breakdown, not near-degenerate clusters that do not break down (the limitation is stated with
# info[b,1] in include/dss_b200.h). Strict xfail: a fix makes these pass and the marks must go.
_MISSES_COPIES = pytest.mark.xfail(strict=True, reason="dss_eigsh_topk misses copies of a near-repeated eigenvalue")
PCA_CASES = [(65, 64, "power"), (65, 1, "power"), (384, 32, "power"), (384, 64, "power"), (768, 1, "power"),
             (768, 32, "power"), (768, 64, "power"), (384, 32, "gap1e-3"), (768, 64, "gap1e-3"),
             pytest.param(384, 32, "equal", marks=_MISSES_COPIES), pytest.param(384, 32, "gap1e-6", marks=_MISSES_COPIES),
             pytest.param(768, 64, "equal", marks=_MISSES_COPIES), pytest.param(768, 64, "gap1e-6", marks=_MISSES_COPIES),
             pytest.param(65, 32, "gap1e-6", marks=_MISSES_COPIES)]


@pytest.mark.parametrize("d,p,kind", PCA_CASES)
def test_pca_components_match_float64(cuda, d, p, kind):
    cluster = load_pkg("cluster")
    X = _rows_with_spectrum(_spectrum(kind, d, p), 3 * d, seed=d + p)
    mean, cov = cluster.covariance(torch.from_numpy(X).to(cuda))
    V = cluster.pca_components(cov, d, p).cpu().numpy()
    r = _check_components(X, V, p, (d, p, kind), cov)
    print(f"PCA d={d} p={p} {kind}: " + " ".join(f"{k} {v:.3f}" for k, v in r.items()))


@pytest.mark.parametrize("d,p", [(384, 1), (384, 32), (768, 64)])
def test_pca_of_l2_normalised_rows(cuda, d, p):
    """The spectrum extract_bbox_clusters feeds: L2-normalised rows of a smooth mixture decay without a clean gap.
    pca() is covariance + components + projection; its output is checked bitwise against that composition."""
    cluster = load_pkg("cluster"); spectral = load_pkg("spectral")
    g = np.random.default_rng(d * p)
    F = (g.normal(size=(4000, d)) * np.linspace(2.0, 0.2, d) + g.normal(size=d)) * g.uniform(1, 10, size=(4000, 1))
    Xn = spectral.normalize_rows(torch.from_numpy(F.astype(np.float32)).to(cuda))
    mean, cov = cluster.covariance(Xn)
    V = cluster.pca_components(cov, d, p)
    r = _check_components(Xn.cpu().numpy(), V.cpu().numpy(), p, ("l2", d, p), cov)
    assert torch.equal(cluster.pca(Xn, p), cluster.pca_project(Xn, mean, V))
    print(f"PCA of normalised rows d={d} p={p}: " + " ".join(f"{k} {v:.3f}" for k, v in r.items()))


def test_pca_components_retry_with_the_largest_krylov_space(cuda, monkeypatch):
    """A spectrum the default step budget (min(d - 1, 320) Lanczos steps) does not resolve to the solver's tolerance:
    768 eigenvalues spread over a relative 1e-4, so the top 64 are separated by ~1e-7 of ||C||. pca_components must
    see the first solve fail, retry with d - 1 steps, and return eigenpairs."""
    cluster = load_pkg("cluster"); spectral = load_pkg("spectral")
    d, p = 768, 64
    g = np.random.default_rng(0)
    lam = 1.0 + 1e-4 * np.linspace(1.0, 0.0, d)
    Q = np.linalg.qr(g.normal(size=(d, d)))[0]
    C = ((Q * lam) @ Q.T).astype(np.float32)
    cov = torch.zeros(d, spectral.pitch(d), dtype=torch.float32)
    cov[:, :d] = torch.from_numpy(C)
    calls = []
    real = spectral.eigsh_topk

    def spy(A, N, K, tol=0.0, max_steps=0):
        out = real(A, N, K, tol=tol, max_steps=max_steps)
        calls.append((max_steps, int(out[2][0, 1])))
        return out

    monkeypatch.setattr(spectral, "eigsh_topk", spy)
    V = cluster.pca_components(cov.to(cuda), d, p).cpu().numpy()
    assert [c[0] for c in calls] == [0, d - 1] and calls[0][1] != 1 and calls[1][1] == 1, calls
    C64 = C.astype(np.float64)
    lam64 = np.linalg.eigvalsh(C64)[::-1]
    rho = np.einsum("id,de,ie->i", V, C64, V)
    assert np.abs(rho - lam64[:p]).max() <= EIG_TOL * lam64[0]
    assert np.linalg.norm(C64 @ V.T - V.T * rho, axis=0).max() <= RESID_TOL * lam64[0]
    assert np.abs(V.astype(np.float64) @ V.T - np.eye(p)).max() <= ORTH_TOL


@pytest.mark.parametrize("M,p", [(32, 32), (33, 32), (2, 1), (64, 64)])
def test_pca_of_rank_deficient_data(cuda, M, p):
    """M - 1 < pca_dim <= M (scikit-learn accepts pca_dim <= min(M, d)): the centred rows span M - 1 directions; the
    components past them are null directions of the covariance and every row projects onto them as ~0."""
    cluster = load_pkg("cluster")
    d = 384
    g = np.random.default_rng(M)
    X = (g.normal(size=(M, d)) * 3 + 1).astype(np.float32)
    Y = cluster.pca(torch.from_numpy(X).to(cuda), p).cpu().numpy()
    assert Y.shape == (M, p) and np.isfinite(Y).all()
    r = M - 1                                                        # rank of the centred data
    scale = np.abs(Y[:, :min(r, p)]).max()
    if p > r:
        assert np.abs(Y[:, r:]).max() <= 1e-5 * scale, np.abs(Y[:, r:]).max() / scale
    Xc = X.astype(np.float64) - X.astype(np.float64).mean(0)
    s = np.linalg.svd(Xc, compute_uv=False)
    got = np.linalg.svd(Y[:, :min(r, p)].astype(np.float64), compute_uv=False)
    assert np.allclose(got, s[:min(r, p)], rtol=1e-4, atol=0), (got[:4], s[:4])


@pytest.mark.parametrize("M,p", [(31, 32), (1, 1), (10, 64)])
def test_pca_refuses_more_components_than_rows(cuda, M, p):
    cluster = load_pkg("cluster")
    with pytest.raises(ValueError, match="rows"):
        cluster.pca(torch.ones(M, 384, device=cuda), p)


def test_normalize_rows_of_zero_rows(cuda):
    spectral = load_pkg("spectral")
    g = np.random.default_rng(3)
    F = g.normal(size=(300, 384)).astype(np.float32) * g.uniform(1e-3, 1e3, size=(300, 1)).astype(np.float32)
    F[[0, 17, 299]] = 0.0
    _lib = load_pkg("_lib")
    x = torch.from_numpy(F).to(cuda)
    out = torch.full((300 + GUARD, 384), float("nan"), device=cuda)      # the kernel writes into it: guard rows after
    assert _lib.load().dss_normalize_rows(x.data_ptr(), 300, 384, out.data_ptr(), _lib.stream_ptr(cuda)) == 0
    torch.cuda.synchronize()
    assert torch.isnan(out[300:]).all(), "a guard row after the output changed"
    got = out[:300].cpu().numpy()
    assert torch.equal(out[:300], spectral.normalize_rows(x))
    assert np.array_equal(got[[0, 17, 299]], np.zeros((3, 384), np.float32))
    F64 = F.astype(np.float64)
    n = np.linalg.norm(F64, axis=1, keepdims=True)
    want = np.divide(F64, n, out=np.zeros_like(F64), where=n > 0)
    assert np.abs(got - want).max() <= 4 * 2.0 ** -24 * np.sqrt(384)


# ------------------------------------------------------------------------------------------- extract_bbox_clusters
def _cluster_features(seed, n_images=1200, d=384, k_true=21):
    """~30 000 box rows over n_images dicts (some with 0 boxes, some with 1) from k_true well-separated directions with
    per-row magnitudes, so the L2 normalisation matters and the K-means decisions have wide margins."""
    g = np.random.default_rng(seed)
    counts = g.integers(2, 49, size=n_images)
    counts[::97] = 0
    counts[1::89] = 1
    dirs = g.normal(size=(k_true, d))
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    out = []
    for i, n in enumerate(counts):
        lab = g.integers(0, k_true, size=n)
        f = (dirs[lab] + 0.03 * g.normal(size=(n, d))) * g.uniform(0.5, 20.0, size=(n, 1))
        out.append({"id": f"im{i:05d}", "bboxes": [[0, 0, 1, 1]] * int(n), "features": torch.from_numpy(f.astype(np.float32))})
    return out


@pytest.mark.parametrize("pca_dim,seed", [(32, 0), (0, 1)])
def test_extract_bbox_clusters_composed_exactly(cuda, tmp_path, pca_dim, seed):
    """The device's PCA output read back and clustered by the float64 K-means oracle (tests/test_kmeans_gpu.py's
    _oracle, same seed and stream key 0) gives the device's labels, centres and iteration count. The oracle's margin
    asserts are unchanged; on this real-valued mixture they hold by construction (21 directions 1.4 apart with noise of
    norm ~0.6 before normalisation). Exact agreement of the k-means++ draws also rests on the device's float32 squared
    distances, whose rounding is far below the spacing of the D^2 prefix sums over 30 000 rows; the bitwise label
    comparison is what checks it. The first E step is on real-valued centres too, so its margin is asserted as well."""
    ex = load_pkg("extract"); cluster = load_pkg("cluster"); spectral = load_pkg("spectral")
    k = 21
    dicts = _cluster_features(100 + pca_dim)
    M = sum(len(d["bboxes"]) for d in dicts)
    assert 25000 <= M <= 35000
    assert any(len(d["bboxes"]) == 0 for d in dicts) and any(len(d["bboxes"]) == 1 for d in dicts)
    torch.save(dicts, tmp_path / "feats.pth")
    ex.extract_bbox_clusters(str(tmp_path / "feats.pth"), str(tmp_path / "clusters.pth"), num_clusters=k, seed=seed,
                             pca_dim=pca_dim)
    out = torch.load(tmp_path / "clusters.pth", weights_only=False)
    assert [d["id"] for d in out] == [d["id"] for d in dicts]
    file_labels = np.concatenate([d["clusters"] for d in out])
    for d in out:
        assert "features" not in d and d["clusters"].dtype == np.int32 and len(d["clusters"]) == len(d["bboxes"])
    feats = torch.cat([d["features"] for d in dicts]).to(cuda)
    Xn = spectral.normalize_rows(feats)
    if pca_dim:
        mean, cov = cluster.covariance(Xn)
        V = cluster.pca_components(cov, Xn.shape[1], pca_dim)
        Y = cluster.pca_project(Xn, mean, V)
        assert torch.equal(Y, cluster.pca(Xn, pca_dim))
        r = _check_components(Xn.cpu().numpy(), V.cpu().numpy(), pca_dim, "clusters", cov)
        # the projection against float64 on the same operands (fp32 X - mean, d fp32 FMAs per output)
        Xc = Xn.cpu().double().numpy() - mean.cpu().double().numpy()
        V64 = V.cpu().double().numpy()
        want = Xc @ V64.T
        bound = 4 * Xn.shape[1] * 2.0 ** -24 * (np.abs(Xc) @ np.abs(V64).T) + 1e-30
        err = np.abs(Y.cpu().double().numpy() - want) / bound
        assert err.max() <= 1.0, err.max()
        r["project"] = err.max()
        print("device PCA: " + " ".join(f"{kk} {v:.3f}" for kk, v in r.items()))
    else:
        Y = Xn
    labels, centres, info, _ = cluster.kmeans(Y, k, seed=seed)
    assert np.array_equal(file_labels, labels.cpu().numpy())             # the file's slices, in dict order
    X = Y.cpu().numpy()
    _, o = _oracle(X, k, seed, 0, 300, 1e-4)
    assert o["e_margin"][0] > 1.0, o["e_margin"][0]
    assert np.array_equal(labels.cpu().numpy(), o["labels"])
    assert np.array_equal(centres.cpu().numpy().view(np.uint32), o["centers"].astype(np.float32).view(np.uint32))
    assert (int(info[0]), int(info[1])) == (o["n_iter"], int(o["converged"]))
    print(f"pca_dim {pca_dim}: {o['n_iter']} iterations, min E margin {o['e_margin'].min():.3g}, "
          f"tol gap {o['tol_gap'].min(initial=np.inf):.3g}")
