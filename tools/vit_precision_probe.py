"""ViT throughput and accuracy of the two precision modes (DinoViT precision='fp16' / 'fp32') on one GPU.

    python tools/vit_precision_probe.py [--out DIR] [--accuracy-images 64]

Prints (and, with --out, writes DIR/vit_precision.json): the card's name and power limit; images/s of the ViT alone (forward_k,
CUDA events after warm-up) at the benchmark's step (ViT-S/16, 264 images of 480 x 480, launched 32 at a time) and at
ViT-B/8 480 x 480; per-kernel-class times from the library's profiler (a separate, untimed pass); and, on
--accuracy-images blobs images at 480 x 480 (ViT-S/16), the K features' rel-L2 against the float64 oracle and the
sign-aligned eigenvector rel-L2 (K = 5) against the reference route (fp32 oracle ViT + scipy eigensolver)."""
from __future__ import annotations

import argparse
import copy
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import importlib  # noqa: E402

PKG = "deep-spectral-segmentation_b200"
vit = importlib.import_module(PKG + ".vit")
pipeline = importlib.import_module(PKG + ".pipeline")
synth = importlib.import_module(PKG + ".synth")
_lib = importlib.import_module(PKG + "._lib")
from oracle import dino_vit, eigs_ref  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def time_vit(model, imgs, chunk, reps):
    out = torch.empty(imgs.shape[0], (imgs.shape[1] // model.patch_size) * (imgs.shape[2] // model.patch_size),
                      model.dim, device=imgs.device)
    def run():
        for s in range(0, imgs.shape[0], chunk):
            model.forward_k(imgs[s:s + chunk], out=out[s:s + chunk])
    run()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        run()
    b.record()
    torch.cuda.synchronize()
    ms = a.elapsed_time(b) / reps
    _lib.profile(True)
    run()
    prof = _lib.profile_read()
    _lib.profile(False)
    return imgs.shape[0] / (ms / 1e3), ms, prof


def _evec_err(v, vo):
    """worst sign-aligned rel-L2 over eigenvectors 1..4 (vector 0 is the constant one)"""
    v, vo = np.asarray(v, np.float64), np.asarray(vo, np.float64)
    return float(max(np.linalg.norm(v[k] - (np.sign(np.dot(v[k], vo[k])) or 1.0) * vo[k]) / np.linalg.norm(vo[k])
                     for k in range(1, 5)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="directory for vit_precision.json")
    ap.add_argument("--accuracy-images", type=int, default=64)
    args = ap.parse_args()
    torch.set_grad_enabled(False)
    dev = torch.device("cuda:0")
    res = {"card": card(), "timing": {}, "accuracy": {}}
    print("card:", res["card"], flush=True)
    for name, n, size, chunk, reps in (("dino_vits16", 264, 480, 32, 5), ("dino_vitb8", 16, 480, 4, 3)):
        ref = dino_vit.build(name, seed=0)
        sd = ref.state_dict()
        imgs = synth.blobs_batch(n, size, size, 0).to(dev)
        for prec in ("fp16", "fp32"):
            model = vit.DinoViT(name, sd, device=dev, precision=prec)
            ips, ms, prof = time_vit(model, imgs, chunk, reps)
            key = f"{name} {size}x{size} x{n} {prec}"
            res["timing"][key] = {"images_per_s": ips, "ms_per_step": ms,
                                  "kernels_ms": {k: v[1] for k, v in prof.items()}}
            print(f"{key}: {ips:.1f} images/s ({ms:.1f} ms), kernels {res['timing'][key]['kernels_ms']}", flush=True)
            del model
            torch.cuda.empty_cache()

    n = args.accuracy_images
    ref = dino_vit.build("dino_vits16", seed=0).to(dev).eval()
    ref64 = copy.deepcopy(ref).double()
    sd = ref.state_dict()
    imgs = synth.blobs_batch(n, 480, 480, 1000)
    k_ref, vec_ref, k64 = [], [], []
    for b in range(n):
        x = dino_vit.preprocess_u8(imgs[b], 16).to(dev)
        k = ref.forward_k(x)[0]
        k_ref.append(k)
        k64.append(ref64.forward_k(x.double())[0])
        vec_ref.append(eigs_ref.extract_eig(k.cpu(), 5, rng_seed=0)[1].numpy())
    e_oracle = [((k_ref[b].double() - k64[b]).norm() / k64[b].norm()).item() for b in range(n)]
    res["accuracy"]["fp32 oracle features rel-L2 vs float64 (median, max)"] = [float(np.median(e_oracle)), max(e_oracle)]
    for prec in ("fp16", "fp32"):
        model = vit.DinoViT("dino_vits16", sd, device=dev, precision=prec)
        pipe = pipeline.SpectralPipeline("dino_vits16", K=5, device=dev, model=model, vit_batch=16)
        ev_err, f_err, over = [], [], []
        for s in range(0, n, 16):
            _, evecs, _ = pipe.run_host(imgs[s:s + 16].pin_memory())
            feats = pipe._bufs["feats"]
            for i in range(evecs.shape[0]):
                b = s + i
                f_err.append(((feats[i].double() - k64[b]).norm() / k64[b].norm()).item())
                ev_err.append(_evec_err(evecs[i].numpy(), vec_ref[b]))
                if ev_err[-1] > 1e-4:   # who is off: both routes against float64 features and a float64 eigh
                    vec64 = eigs_ref.eigh_f64(k64[b].cpu(), 6)[1][:5]
                    over.append({"image": b, "ours_vs_reference": ev_err[-1],
                                 "ours_vs_float64": _evec_err(evecs[i].numpy(), vec64),
                                 "reference_vs_float64": _evec_err(vec_ref[b], vec64)})
        res["accuracy"][prec] = {"features rel-L2 vs float64 (median, max)": [float(np.median(f_err)), max(f_err)],
                                 "eigenvector rel-L2 vs reference route (median, max)": [float(np.median(ev_err)),
                                                                                       max(ev_err)],
                                 "images over 1e-4": len(over), "over 1e-4, attributed": over[:8]}
        print(prec, res["accuracy"][prec], flush=True)
    print("oracle", res["accuracy"]["fp32 oracle features rel-L2 vs float64 (median, max)"])
    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        (Path(args.out) / "vit_precision.json").write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
