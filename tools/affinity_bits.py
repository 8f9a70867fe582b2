"""SHA-256 digests of the affinity build's output bytes (dss_affinity: W with its pitch padding, and the degree) on
seeded features, written as the fixture that tests/test_affinity_bits_gpu.py recomputes and compares: a change to the
affinity GEMM that must keep its bits is checked against digests taken before it.

    python tools/affinity_bits.py [--out tests/golden/affinity_bits.json]

Cases (B, N, d, flags, colour counts, row pitch):
  - N in {1, 63, 64, 65, 127, 128, 129, 196, 713, 900, 901, 1024, 3600} at B = 3, d = 384, normalised rows: every
    width class of an image's last column tile (1 .. 128 columns) and last row tiles with at most and with more than
    64 rows;
  - B = 1 and d in {64, 768} at N = 900;
  - every combination of the DSS_AFF_* flags at N = 900 (and the LOST form, DSS_AFF_NO_MAX_SCALE alone, at N = 129);
  - colour counts with lambda = 10 at N = 129 and 900;
  - row pitches wider than N: inside the last column tile (N = 65, 900) and past it (N = 129, 713).
Features are N(0, 1) with a per-row scale in [0.25, 4), so that the Gram matrix has negative entries (for the relu
threshold) and the un-normalised paths see a pre-scale other than 1. W is filled with NaN before each call, so an
element the kernel no longer writes changes the digest."""
from __future__ import annotations

import argparse
import hashlib
import importlib
import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
PKG = "deep-spectral-segmentation_b200"

NORMALIZE, THRESHOLD, NO_MAX = 1, 2, 4
EDGE_N = [1, 63, 64, 65, 127, 128, 129, 196, 713, 900, 901, 1024, 3600]


def pitch(N):
    return (N + 3) // 4 * 4


# (B, N, d, flags, lambda of the colour counts or None, row pitch)
CASES = [(3, N, 384, NORMALIZE, None, pitch(N)) for N in EDGE_N] + \
        [(1, 900, d, NORMALIZE, None, 900) for d in (64, 768)] + \
        [(2, 900, 384, f, None, 900) for f in range(8) if f != NORMALIZE] + \
        [(2, 129, 384, NO_MAX, None, 132)] + \
        [(2, N, 384, NORMALIZE | THRESHOLD, 10.0, pitch(N)) for N in (129, 900)] + \
        [(2, 65, 384, NORMALIZE, None, 124), (2, 900, 384, NORMALIZE | THRESHOLD, None, 1020),
         (2, 129, 384, NORMALIZE, None, 300), (2, 713, 384, NO_MAX, None, 900)]


def _pkg(sub):
    if str(ROOT) not in sys.path:
        sys.path.insert(0, str(ROOT))
    return importlib.import_module(f"{PKG}.{sub}")


def digest(t: torch.Tensor) -> str:
    return hashlib.sha256(t.contiguous().cpu().numpy().tobytes()).hexdigest()


def key(B, N, d, flags, lam, ldw):
    return f"B{B}_N{N}_d{d}_f{flags}_c{0 if lam is None else 1}_ld{ldw}"


def inputs(B, N, d, lam, seed):
    g = torch.Generator().manual_seed(seed)
    f = torch.randn(B, N, d, generator=g) * (0.25 + 3.75 * torch.rand(B, N, 1, generator=g))
    counts = None
    if lam is not None:
        c = torch.randint(0, 6, (B, N, N), generator=g, dtype=torch.uint8)
        counts = (torch.triu(c) + torch.triu(c, 1).transpose(1, 2)).contiguous()
    return f, counts


def affinity(B, N, d, flags, lam, ldw):
    """-> (W [B, N, ldw], degree [B, N]) of dss_affinity on the case's seeded inputs"""
    _lib = _pkg("_lib")
    lib = _lib.load()
    f, counts = inputs(B, N, d, lam, seed=B * 1000003 + N * 1009 + d * 31 + flags * 7 + ldw)
    f = f.cuda()
    counts = None if counts is None else counts.cuda()
    W = torch.full((B, N, ldw), float("nan"), device="cuda")
    deg = torch.full((B, N), float("nan"), device="cuda")
    need = int(lib.dss_affinity_workspace_bytes(B, N, d))
    ws = torch.zeros(need, dtype=torch.uint8, device="cuda")
    _lib.check(lib.dss_affinity(f.data_ptr(), B, N, d, flags, _lib.ptr(counts), float(lam or 0.0), W.data_ptr(), ldw,
                                deg.data_ptr(), ws.data_ptr(), need, _lib.stream_ptr()), "dss_affinity")
    torch.cuda.synchronize()
    return W, deg


def digests() -> dict:
    torch.set_grad_enabled(False)
    out = {}
    for c in CASES:
        W, deg = affinity(*c)
        out[key(*c)] = {"W": digest(W), "degree": digest(deg)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=str(ROOT / "tests" / "golden" / "affinity_bits.json"))
    args = ap.parse_args()
    Path(args.out).parent.mkdir(parents=True, exist_ok=True)
    Path(args.out).write_text(json.dumps(digests(), indent=1, sort_keys=True) + "\n")
    print(args.out)


if __name__ == "__main__":
    main()
