"""Host side of the semantic-segmentation kernels (csrc/cluster.cu): segment bounding boxes of label maps, the
covariance-eigh PCA and the data-set K-means of the reference's extract_bboxes / extract_bbox_clusters
(extract/extract.py:429-599)."""
from __future__ import annotations

import math
from typing import Tuple

import torch

from . import _lib, spectral

KMEANS_MAX_K = 64         # at dims <= 768 ...
KMEANS_MAX_K_NARROW = 256  # ... and at dims <= 64
PCA_MAX_DIM = 64           # dss_eigsh_topk computes at most 64 eigenpairs


@torch.no_grad()
def segment_bboxes(segmaps: torch.Tensor, num_erode: int, num_dilate: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """segmaps [B, H, W] uint8 CUDA -> (boxes [B, 256, 4] int32 = (xmin, ymin, xmax + 1, ymax + 1) of every label value
    after num_erode erosions and num_dilate dilations, present [B, 256] bool)."""
    _lib.require_cuda(segmaps, "segmaps")
    if segmaps.dtype != torch.uint8 or segmaps.dim() != 3:
        raise ValueError(f"segmaps must be uint8 [B, H, W], got {segmaps.dtype} {tuple(segmaps.shape)}")
    s = segmaps.contiguous()
    B, H, W = s.shape
    dev = s.device
    with torch.cuda.device(dev):
        boxes = torch.empty(B, 256, 4, dtype=torch.int32, device=dev)
        present = torch.empty(B, 256, dtype=torch.uint8, device=dev)
        _lib.check(_lib.load().dss_segment_bboxes(s.data_ptr(), B, H, W, int(num_erode), int(num_dilate), boxes.data_ptr(),
                                                  present.data_ptr(), _lib.stream_ptr(dev)), "dss_segment_bboxes")
    return boxes, present.bool()


@torch.no_grad()
def covariance(X: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """X [M, d] fp32 CUDA -> (column mean [d], covariance [d, pitch(d)] with ddof 1; columns >= d are zero)."""
    _lib.require_cuda(X, "X")
    x = X.to(torch.float32).contiguous()
    M, d = x.shape
    lib = _lib.load()
    dev = x.device
    with torch.cuda.device(dev):
        mean = torch.empty(d, dtype=torch.float32, device=dev)
        cov = torch.zeros(d, spectral.pitch(d), dtype=torch.float32, device=dev)
        ws = spectral._scratch.get("cov", int(lib.dss_covariance_workspace_bytes(M, d)), dev)
        _lib.check(lib.dss_covariance(x.data_ptr(), M, d, mean.data_ptr(), cov.data_ptr(), cov.shape[1], ws.data_ptr(),
                                      ws.numel(), _lib.stream_ptr(dev)), "dss_covariance")
    return mean, cov


@torch.no_grad()
def pca_components(cov: torch.Tensor, d: int, pca_dim: int) -> torch.Tensor:
    """Top ``pca_dim`` eigenvectors [pca_dim, d] of the covariance (dss_eigsh_topk). Like the eigenvector commands, a
    solve that does not reach its tolerance is retried with the largest Krylov space, and then fails loudly.

    The solver stops at residual <= tol * max(1, ||A||): an absolute 1e-6 for a covariance with ||C|| < 1, which is
    what L2-normalised rows give (||C|| ~ 3e-3 at d = 768). So the covariance is first multiplied by the power of two
    that brings its largest diagonal entry into [1, 2). That is exact in fp32 and leaves the eigenvectors unchanged, and
    since lambda_1 >= max C_ii the tolerance is then relative to ||C||.

    Limitation: a cluster of distinct but nearly equal eigenvalues straddling pca_dim (relative spread ~1e-6) does not
    break the Lanczos recurrence down, so the solver can report convergence with copies from the cluster missing and
    return vectors from below it instead (see dss_eigsh_topk in include/dss_b200.h)."""
    if pca_dim > PCA_MAX_DIM:
        raise _lib.DssError(f"pca_dim={pca_dim} > {PCA_MAX_DIM}: the device eigensolver computes at most "
                            f"{PCA_MAX_DIM} eigenpairs")
    if not 1 <= pca_dim < d:
        raise ValueError(f"pca_dim={pca_dim} must be in [1, {d})")
    top = float(torch.diagonal(cov[:, :d]).max())
    if math.isfinite(top) and top > 0.0:
        cov = cov * math.ldexp(1.0, 1 - math.frexp(top)[1])       # max C_ii * 2^k in [1, 2)
    evals, evecs, info, _ = spectral.eigsh_topk(cov[None], d, pca_dim)
    if int(info[0, 1]) != 1 or not bool(torch.isfinite(evecs).all()):
        evals, evecs, info, _ = spectral.eigsh_topk(cov[None], d, pca_dim, max_steps=d - 1)
        if int(info[0, 1]) != 1 or not bool(torch.isfinite(evecs).all()):
            raise _lib.DssError(f"PCA: the eigensolver did not converge for the {d} x {d} covariance")
    return evecs[0]


@torch.no_grad()
def pca_project(X: torch.Tensor, mean: torch.Tensor, V: torch.Tensor) -> torch.Tensor:
    """(X - mean) V^T: X [M, d], V [p, d] -> [M, p]."""
    _lib.require_cuda(X, "X")
    x, m, v = (t.to(torch.float32).contiguous() for t in (X, mean, V))
    M, d = x.shape
    p = v.shape[0]
    assert v.shape[1] == d and m.shape == (d,)
    with torch.cuda.device(x.device):
        y = torch.empty(M, p, dtype=torch.float32, device=x.device)
        _lib.check(_lib.load().dss_pca_project(x.data_ptr(), M, d, m.data_ptr(), v.data_ptr(), p, y.data_ptr(),
                                               _lib.stream_ptr(x.device)), "dss_pca_project")
    return y


@torch.no_grad()
def pca(X: torch.Tensor, pca_dim: int) -> torch.Tensor:
    """scikit-learn PCA(pca_dim).fit_transform(X) by the covariance-eigh route (component signs may differ).
    Like scikit-learn, pca_dim may not exceed the number of rows: with M rows the centred data span at most M - 1
    directions, and the components past them are null directions of the covariance, onto which every row projects to
    ~0. A small data set can hit this, so it is an error of the input (ValueError), not a device failure."""
    M = X.shape[0]
    if M < 2 or pca_dim > M:
        raise ValueError(f"pca_dim={pca_dim} needs at least max(2, pca_dim) rows, got {M}")
    mean, cov = covariance(X)
    return pca_project(X, mean, pca_components(cov, X.shape[1], pca_dim))


@torch.no_grad()
def kmeans(X: torch.Tensor, k: int, seed: int = 0, max_iter: int = 300, tol: float = 1e-4):
    """K-means of the rows of X [M, dims] fp32 CUDA on the whole GPU (csrc/cluster.cu).
    Returns (labels int32 [M], centres [k, dims], info int32 [2] = {iterations, converged}, inertia fp32 [1])."""
    _lib.require_cuda(X, "X")
    x = X.to(torch.float32).contiguous()
    M, dims = x.shape
    lib = _lib.load()
    dev = x.device
    with torch.cuda.device(dev):
        labels = torch.empty(M, dtype=torch.int32, device=dev)
        centres = torch.empty(k, dims, dtype=torch.float32, device=dev)
        info = torch.empty(2, dtype=torch.int32, device=dev)
        inertia = torch.empty(1, dtype=torch.float32, device=dev)
        ws = spectral._scratch.get("kmeans", int(lib.dss_kmeans_workspace_bytes(M, dims, k)), dev)
        _lib.check(lib.dss_kmeans(x.data_ptr(), M, dims, int(k), int(seed) & 0xFFFFFFFF, int(max_iter), float(tol),
                                  centres.data_ptr(), labels.data_ptr(), info.data_ptr(), inertia.data_ptr(),
                                  ws.data_ptr(), ws.numel(), _lib.stream_ptr(dev)), "dss_kmeans")
    return labels, centres, info, inertia
