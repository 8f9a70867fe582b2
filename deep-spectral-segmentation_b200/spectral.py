"""Host side of the affinity / colour-KNN / eigensolver stage (mirror of the arithmetic in
extract/extract.py:148,191-240 and extract/extract_utils.py:151-220). Device work: csrc/affinity.cu, knn.cu, eigsh.cu."""
from __future__ import annotations

from typing import Optional, Tuple

import torch

from . import _lib


class _Scratch:
    """Grow-only device scratch buffers keyed by purpose (caller-owned workspaces of the C ABI)."""

    def __init__(self):
        self.bufs = {}

    def get(self, key, nbytes, device):
        b = self.bufs.get((key, device))
        if b is None or b.numel() < nbytes:
            b = torch.empty(max(int(nbytes), 256), dtype=torch.uint8, device=device)
            self.bufs[(key, device)] = b
        return b


_scratch = _Scratch()


def pitch(N: int) -> int:
    """Row pitch of the affinity matrix: rows padded to a multiple of 4 floats (16 B) for vector loads."""
    return (N + 3) // 4 * 4


@torch.no_grad()
def knn_color_counts(rgb_lr: torch.Tensor, Hl: int, Wl: int) -> torch.Tensor:
    """rgb_lr [B, Hl*Wl, 3] fp32 CUDA in [0,1] -> dense KNN colour affinity counts [B, N, N] uint8."""
    _lib.require_cuda(rgb_lr, "rgb_lr")
    lib = _lib.load()
    rgb = rgb_lr.to(torch.float32).contiguous()
    B, N, _ = rgb.shape
    assert N == Hl * Wl
    with torch.cuda.device(rgb.device):
        # bytes are updated with 32-bit atomics: capacity rounded up to a whole word (any N, odd included)
        flat = torch.empty((B * N * N + 3) // 4 * 4, dtype=torch.uint8, device=rgb.device)
        _lib.check(lib.dss_knn_color_counts(rgb.data_ptr(), B, Hl, Wl, flat.data_ptr(), None, 0,
                                            _lib.stream_ptr(rgb.device)), "dss_knn_color_counts")
    return flat[:B * N * N].view(B, N, N)


@torch.no_grad()
def affinity(feats: torch.Tensor, normalize=True, threshold_at_zero=True, color_counts: Optional[torch.Tensor] = None,
             color_lambda: float = 0.0, out: Optional[torch.Tensor] = None, scale_by_max: bool = True,
             degree: Optional[torch.Tensor] = None) -> torch.Tensor:
    """feats [B, N, d] fp32 CUDA -> W [B, N, pitch(N)] fp32 (columns >= N are zero). If ``degree`` [B, N] fp32 is
    given it receives the row sums of W, accumulated in the affinity kernel's epilogue (get_diagonal's row_sum)."""
    _lib.require_cuda(feats, "feats")
    lib = _lib.load()
    f = feats.to(torch.float32).contiguous()
    B, N, d = f.shape
    ldw = pitch(N)
    dev = f.device
    with torch.cuda.device(dev):
        if out is None:
            out = torch.empty(B, N, ldw, dtype=torch.float32, device=dev)
        need = int(lib.dss_affinity_workspace_bytes(B, N, d))
        ws = _scratch.get("aff", need, dev)
        flags = ((_lib.AFF_NORMALIZE if normalize else 0) | (_lib.AFF_THRESHOLD_AT_ZERO if threshold_at_zero else 0)
                 | (0 if scale_by_max else _lib.AFF_NO_MAX_SCALE))
        cc = None
        if color_counts is not None and color_lambda > 0:
            cc = color_counts.contiguous()
            assert cc.dtype == torch.uint8 and tuple(cc.shape) == (B, N, N)
        if degree is not None:
            assert degree.dtype == torch.float32 and degree.is_contiguous() and tuple(degree.shape) == (B, N)
        _lib.check(lib.dss_affinity(f.data_ptr(), B, N, d, flags, _lib.ptr(cc), float(color_lambda), out.data_ptr(), ldw,
                                    _lib.ptr(degree), ws.data_ptr(), ws.numel(), _lib.stream_ptr(dev)), "dss_affinity")
    return out


DEFAULT_MAX_STEPS = 320   # the solver's step budget for max_steps <= 0 (at most N - 1, N for eigsh_topk)


def max_steps(N: int, mode: int = 0) -> int:
    """Largest step budget the solver accepts at N: its Lanczos tridiagonal (3 doubles per step) lives in shared memory.
    At most N - 1 (mode 0 / 1, eigsh_laplacian) or N (mode 2, eigsh_topk); 0 when not even one step fits."""
    return int(_lib.load().dss_eigsh_max_steps(N, mode))


@torch.no_grad()
def eigsh_laplacian(W: torch.Tensor, N: int, K: int, lapnorm=True, tol: float = 0.0, max_steps: int = 0,
                    degree: Optional[torch.Tensor] = None
                    ) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
    """W [B, N, ldw] fp32 CUDA (symmetric; the upper triangle is what is read) -> (eigenvalues [B,K], eigenvectors
    [B,K,N], info [B,4] int32, resid [B,K]). ``degree`` [B, N]: row sums of W from affinity(), or None."""
    _lib.require_cuda(W, "W")
    lib = _lib.load()
    assert W.dtype == torch.float32 and W.is_contiguous() and W.dim() == 3 and W.shape[1] == N
    B, _, ldw = W.shape
    dev = W.device
    with torch.cuda.device(dev):
        evals = torch.empty(B, K, dtype=torch.float32, device=dev)
        evecs = torch.empty(B, K, N, dtype=torch.float32, device=dev)
        info = torch.empty(B, 4, dtype=torch.int32, device=dev)
        resid = torch.empty(B, K, dtype=torch.float32, device=dev)
        need = int(lib.dss_eigsh_workspace_bytes(B, N, K, max_steps))
        ws = _scratch.get("eig", need, dev)
        if degree is not None:
            assert degree.dtype == torch.float32 and degree.is_contiguous() and tuple(degree.shape) == (B, N)
        _lib.check(lib.dss_eigsh_laplacian(W.data_ptr(), _lib.ptr(degree), ldw, B, N, K, 1 if lapnorm else 0, float(tol),
                                           int(max_steps),
                                           evals.data_ptr(), evecs.data_ptr(), info.data_ptr(), resid.data_ptr(),
                                           ws.data_ptr(), ws.numel(), _lib.stream_ptr(dev)), "dss_eigsh_laplacian")
    return evals, evecs, info, resid


@torch.no_grad()
def eigsh_topk(A: torch.Tensor, N: int, K: int, tol: float = 0.0, max_steps: int = 0):
    """A [B, N, lda] symmetric fp32 CUDA -> K algebraically largest pairs, descending:
    (eigenvalues [B,K], eigenvectors [B,K,N] unit 2-norm with the sign rule, info [B,4], resid [B,K])."""
    _lib.require_cuda(A, "A")
    lib = _lib.load()
    assert A.dtype == torch.float32 and A.is_contiguous() and A.dim() == 3 and A.shape[1] == N
    B, _, lda = A.shape
    dev = A.device
    with torch.cuda.device(dev):
        evals = torch.empty(B, K, dtype=torch.float32, device=dev)
        evecs = torch.empty(B, K, N, dtype=torch.float32, device=dev)
        info = torch.empty(B, 4, dtype=torch.int32, device=dev)
        resid = torch.empty(B, K, dtype=torch.float32, device=dev)
        need = int(lib.dss_eigsh_workspace_bytes(B, N, K, max_steps))
        ws = _scratch.get("eig", need, dev)
        _lib.check(lib.dss_eigsh_topk(A.data_ptr(), lda, B, N, K, float(tol), int(max_steps), evals.data_ptr(),
                                      evecs.data_ptr(), info.data_ptr(), resid.data_ptr(), ws.data_ptr(), ws.numel(),
                                      _lib.stream_ptr(dev)), "dss_eigsh_topk")
    return evals, evecs, info, resid


@torch.no_grad()
def normalize_rows(feats: torch.Tensor) -> torch.Tensor:
    """F.normalize(p=2, dim=-1) of [..., d] fp32 CUDA features (extract.py:148)."""
    _lib.require_cuda(feats, "feats")
    f = feats.to(torch.float32).contiguous()
    out = torch.empty_like(f)
    with torch.cuda.device(f.device):
        _lib.check(_lib.load().dss_normalize_rows(f.data_ptr(), f.numel() // f.shape[-1], f.shape[-1], out.data_ptr(),
                                                  _lib.stream_ptr(f.device)), "dss_normalize_rows")
    return out


@torch.no_grad()
def upsample_bilinear(feats: torch.Tensor, Hp: int, Wp: int, Hl: int, Wl: int) -> torch.Tensor:
    """feats [B, Hp*Wp, d] -> [B, Hl*Wl, d]: F.interpolate(bilinear, align_corners=False) of extract.py:185-188."""
    _lib.require_cuda(feats, "feats")
    f = feats.to(torch.float32).contiguous()
    B, N, d = f.shape
    assert N == Hp * Wp
    out = torch.empty(B, Hl * Wl, d, dtype=torch.float32, device=f.device)
    with torch.cuda.device(f.device):
        _lib.check(_lib.load().dss_upsample_bilinear(f.data_ptr(), B, Hp, Wp, d, Hl, Wl, out.data_ptr(),
                                                     _lib.stream_ptr(f.device)), "dss_upsample_bilinear")
    return out


@torch.no_grad()
def affinity_eigs(feats: torch.Tensor, K: int, which_matrix: str = "affinity", normalize=True, threshold_at_zero=True,
                  tol: float = 0.0, max_steps: int = 0):
    """The reference's which_matrix='affinity' (eigsh(W, which='LM'), extract.py:166-172) and 'affinity_svd'
    (torch.linalg.svd(feats), extract.py:160-163) branches for a batch. Returns descending (values, vectors, info);
    for 'affinity_svd' the values are singular values sqrt(eig(F^ F^T))."""
    if which_matrix == "affinity":
        A = affinity(feats, normalize, threshold_at_zero, scale_by_max=False)
    elif which_matrix == "affinity_svd":
        A = affinity(feats, normalize, False, scale_by_max=False)
    else:
        raise ValueError(which_matrix)
    evals, evecs, info, _ = eigsh_topk(A, feats.shape[1], K, tol, max_steps)
    if which_matrix == "affinity_svd":
        evals = evals.clamp_min(0).sqrt()
    return evals, evecs, info


RW_COEF = 900.0   # pymatting's _rw_laplacian hard-codes exp(-900 ||zi - zj||^2); its sigma argument (0.033) is unused


@torch.no_grad()
def rw_affinity_add(W: torch.Tensor, degree: Optional[torch.Tensor], rgb_u8: torch.Tensor, Hl: int, Wl: int,
                    color_lambda: float, coef: float = RW_COEF) -> None:
    """W [B, N, ldw] += lambda * random-walk colour affinity of the uint8 low-res images rgb_u8 [B, N, 3]
    (which_color_matrix='rw', extract_utils.py:191-204); degree [B, N] is updated with the added row sums."""
    _lib.require_cuda(W, "W")
    assert rgb_u8.dtype == torch.uint8 and rgb_u8.is_cuda and rgb_u8.is_contiguous()
    B, N, ldw = W.shape
    assert N == Hl * Wl and tuple(rgb_u8.shape) == (B, N, 3)
    with torch.cuda.device(W.device):
        _lib.check(_lib.load().dss_rw_affinity_add(rgb_u8.data_ptr(), B, Hl, Wl, float(color_lambda), float(coef),
                                                   W.data_ptr(), ldw, _lib.ptr(degree), _lib.stream_ptr(W.device)),
                   "dss_rw_affinity_add")


@torch.no_grad()
def laplacian_eigs(feats: torch.Tensor, K: int, normalize=True, threshold_at_zero=True, lapnorm=True,
                   rgb_lr: Optional[torch.Tensor] = None, lr_size: Optional[Tuple[int, int]] = None,
                   color_lambda: float = 0.0, tol: float = 0.0, max_steps: int = 0, which_color_matrix: str = "knn"):
    """which_matrix='laplacian' of the reference for a batch: feats [B,N,d] -> (eigenvalues [B,K], eigenvectors [B,K,N]).
    rgb_lr: the low-resolution image of extract.py:199-204 -- fp32 [B,N,3] in [0,1] for 'knn', the uint8 pixels
    [B,N,3] (before the /255) for 'rw'."""
    cc = None
    if color_lambda > 0:
        if rgb_lr is None or lr_size is None:
            raise ValueError("image_color_lambda > 0 needs the low-resolution image (rgb_lr, lr_size)")
        if which_color_matrix == "knn":
            cc = knn_color_counts(rgb_lr, lr_size[0], lr_size[1])
        elif which_color_matrix != "rw":
            raise ValueError(f"unknown which_color_matrix={which_color_matrix!r}")
    deg = torch.empty(feats.shape[0], feats.shape[1], dtype=torch.float32, device=feats.device)
    W = affinity(feats, normalize, threshold_at_zero, cc, color_lambda, degree=deg)
    if color_lambda > 0 and which_color_matrix == "rw":
        rw_affinity_add(W, deg, rgb_lr, lr_size[0], lr_size[1], color_lambda)
    evals, evecs, info, resid = eigsh_laplacian(W, feats.shape[1], K, lapnorm, tol, max_steps, degree=deg)
    return evals, evecs, info, resid


@torch.no_grad()
def get_eigenvectors_from_features(feats: torch.Tensor, which_matrix: str = "laplacian", K: int = 2):
    """Second caller of the eigensolver in the reference: object-localization/object_discovery.py:16-42
    (``get_eigenvectors_from_features``: A = F F^T on the features AS GIVEN, relu, /max, degree, eigsh(D - A, sigma=0,
    M=D) in float64, K=2, no sign rule). feats [N, d] CUDA -> (eigenvalues [K], eigenvectors [K, N]) on the device.
    The sign of each vector is the library's (the reference returns ARPACK's arbitrary sign there)."""
    if which_matrix == "affinity_torch":
        raise RuntimeError("which_matrix='affinity_torch' calls torch.eig, which PyTorch removed (dead in the reference)")
    if which_matrix == "affinity":
        ev, vec, _ = affinity_eigs(feats[None], K, "affinity", normalize=False, threshold_at_zero=False)
        return ev[0].flip(0), vec[0]          # the reference leaves eigsh's ascending values next to flipped vectors
    if which_matrix == "laplacian":
        ev, vec, _, _ = laplacian_eigs(feats[None], K, normalize=False, threshold_at_zero=True, lapnorm=True)
        return ev[0], vec[0]
    raise NotImplementedError(which_matrix)   # 'matting_laplacian' raises in the reference as well (:44-46)
