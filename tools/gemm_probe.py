"""Tile-width / ring-depth sweep of the wgmma GEMM on the ViT-S shapes (tuning probe)."""
import importlib, sys
from pathlib import Path
import torch
sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
_lib = importlib.import_module("deep-spectral-segmentation_b200._lib")
lib = _lib.load()
dev = torch.device("cuda:0")
M = 256 * 901
def run(N, K, bn, st, iters=20):
    A = torch.randn(M, K, device=dev).half(); W = (torch.randn(N, K, device=dev) * 0.05).half()
    bias = torch.zeros(N, device=dev); out = torch.empty(M, N, device=dev, dtype=torch.float16)
    flush = torch.empty(64 * 1024 * 1024, device=dev)
    def call():
        _lib.check(lib.dss_debug_gemm_cfg(A.data_ptr(), W.data_ptr(), bias.data_ptr(), out.data_ptr(), M, N, K, bn, st, _lib.stream_ptr()))
    for _ in range(3): call()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        flush.zero_()
        s, e = torch.cuda.Event(True), torch.cuda.Event(True)
        s.record(); call(); e.record(); torch.cuda.synchronize(); ts.append(s.elapsed_time(e))
    ts.sort(); t = ts[len(ts)//2]
    ref = (A[:256].float() @ W.float().T)
    err = (out[:256].float() - ref).abs().max().item()
    print(f"N={N:5d} K={K:5d} bn={bn} stages={st}: {t*1e3:8.1f} us  {2*M*N*K/t/1e9:8.1f} TFLOP/s  err {err:.2e}")
for (N, K) in [(1152, 384), (1536, 384), (384, 1536), (384, 384)]:
    for bn, st in [(128, 3), (192, 4), (256, 4)]:
        if N % bn: continue
        run(N, K, bn, st)
