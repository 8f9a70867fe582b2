"""Quick device-side timing of the pipeline stages (CUDA events). Not the benchmark: see bench.py."""
import importlib
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
pkg = "deep-spectral-segmentation_b200"
vit = importlib.import_module(pkg + ".vit")
spectral = importlib.import_module(pkg + ".spectral")
synth = importlib.import_module(pkg + ".synth")
torch.set_grad_enabled(False)
dev = torch.device("cuda:0")


def timeit(fn, iters=5, warm=2):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(True), torch.cuda.Event(True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def main():
    name = sys.argv[1] if len(sys.argv) > 1 else "dino_vits16"
    H = W = int(sys.argv[2]) if len(sys.argv) > 2 else 480
    K = int(sys.argv[3]) if len(sys.argv) > 3 else 5
    model, _, P, _ = vit.get_model(name, seed=0, device=dev)
    base = synth.blobs_batch(8, H, W, 0).to(dev)
    print(f"model {name} {H}x{W} K={K} SMs={torch.cuda.get_device_properties(0).multi_processor_count}")
    for B in (1, 8, 16, 32, 64):
        imgs = base.repeat((B + 7) // 8, 1, 1, 1)[:B].contiguous()
        ms = timeit(lambda: model.forward_k(imgs))
        print(f"vit forward_k  B={B:4d}: {ms:8.3f} ms  -> {ms / B * 1e3:8.1f} us/img  {B / ms * 1e3:9.1f} img/s")
    imgs = base
    feats8 = model.forward_k(imgs)
    N = feats8.shape[1]
    for B in (8, 64, 132, 264, 528):
        feats = feats8.repeat((B + 7) // 8, 1, 1)[:B].contiguous()
        deg = torch.empty(B, N, device=dev)
        Wm = spectral.affinity(feats, degree=deg)
        ms_a = timeit(lambda: spectral.affinity(feats, out=Wm, degree=deg))
        ms_e = timeit(lambda: spectral.eigsh_laplacian(Wm, N, K, degree=deg))
        ev, vec, info, resid = spectral.eigsh_laplacian(Wm, N, K, degree=deg)
        torch.cuda.synchronize()
        print(f"spectral B={B:4d}: affinity {ms_a:8.3f} ms ({ms_a / B * 1e3:7.1f} us/img)  eigsh {ms_e:8.3f} ms "
              f"({ms_e / B * 1e3:7.1f} us/img)  steps mean {info[:, 0].float().mean().item():.1f} max {int(info[:, 0].max())} "
              f"conv {int(info[:, 1].sum())}/{B}")


if __name__ == "__main__":
    main()
