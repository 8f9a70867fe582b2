"""Images/s of the three localization methods on VOC-shaped synthetic images (375 x 500, ViT-S/16 with seeded
weights) on one GPU, next to the reference's CPU route (the oracle port: fp32 ViT on the CPU at batch 1 plus the
numpy / scipy box extraction) timed in the same run.

    python tools/localize_probe.py [--images 64] [--batch 16] [--cpu-images 4]
"""
import argparse
import importlib
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
PKG = "deep-spectral-segmentation_b200"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=64)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--cpu-images", type=int, default=4)
    a = ap.parse_args()
    torch.set_grad_enabled(False)
    loc, vit, spectral, synth = (importlib.import_module(f"{PKG}.{m}") for m in ("localize", "vit", "spectral", "synth"))
    from oracle import dino_vit, localize_ref
    dev = torch.device("cuda:0")
    ref = dino_vit.build("dino_vits16", seed=0)
    model = vit.DinoViT("dino_vits16", ref.state_dict(), device=dev)
    H, W, P = 375, 500, 16
    gh, gw = -(-H // P), -(-W // P)
    imgs = synth.blobs_batch(a.batch, H, W, seed0=0).to(dev)

    def lost():
        f, _ = model.forward_last(imgs, "k", pad=True)
        return loc.lost_boxes(f, (gh, gw), (H, W), P, 100)

    def dinoseg():
        _, at = model.forward_last(imgs, "k", pad=True, feats=False, cls_attn=True)
        return loc.dinoseg_boxes(at, (gh, gw), P, 4)

    def eigenseg():
        f, _ = model.forward_last(imgs, "k", pad=False)
        _, ev, _, _ = spectral.laplacian_eigs(f, 2, normalize=False, threshold_at_zero=True, lapnorm=True)
        return loc.eigseg_boxes(ev, 1, [(H, W)] * a.batch)

    for name, fn in (("lost", lost), ("dinoseg", dinoseg), ("eigenseg_from_features", eigenseg)):
        fn(); fn()
        torch.cuda.synchronize()
        n = max(1, a.images // a.batch)
        t0 = time.perf_counter()
        for _ in range(n):
            fn()   # each call ends in a device-to-host copy of the boxes
        dt = time.perf_counter() - t0
        print(f"gpu {name}: {n * a.batch / dt:.1f} images/s (batch {a.batch}, {n} batches)")

    # the reference's route on the CPU: fp32 ViT at batch 1, then the numpy / scipy LOST box
    cpu_imgs = synth.blobs_batch(a.cpu_images, H, W, seed0=0)
    t0 = time.perf_counter()
    for i in range(a.cpu_images):
        x = localize_ref.preprocess_pad(cpu_imgs[i], P)
        f, at = localize_ref.last_outputs(ref, x, "k")
        f = f[0].numpy()
        localize_ref.lost_box(f @ f.T, (gh, gw), (H, W), P, 100)
    dt = time.perf_counter() - t0
    print(f"cpu reference route (LOST, {torch.get_num_threads()} threads): {a.cpu_images / dt:.2f} images/s")
    print(torch.cuda.get_device_name(0))


if __name__ == "__main__":
    main()
