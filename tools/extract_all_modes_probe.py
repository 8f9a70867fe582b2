"""extract_all images/s in colour mode and at a finer eigenvector grid, each against the route it replaces, on one GPU.

    python tools/extract_all_modes_probe.py [--n 512] [--reps 3] [--batch 64] [--out DIR]

ViT-S/16, fp16 mode, seeded weights, K = 20, on --n synthetic JPEG files of the VOC shapes (synth.voc_shapes, blobs
images). Two comparisons, the variants alternated --reps times in one process after one warm-up call of each:

  colour:     extract_all with image_color_lambda=10, 'knn'. 'device' resizes the decoded batch on the GPU
              (resize.py); 'host' is the former route: _color_inputs re-opens every JPEG and PIL-resizes it on the
              thread that launches the batches, with the plain decoder.
  downsample: image_downsample_factor=8. 'fused' is extract_all; 'files' is extract_features followed by
              extract_eigs with the same options (the route a user had before).

Images/s is the number of images over the wall time of the whole call (model set-up included for both variants of a
comparison). Each variant's eigs files are compared with the other's (torch.equal). Prints the card's name and power
limit (nvidia-smi, read in the same run) and one JSON line (also DIR/extract_all_modes_probe.json with --out). All
files go to a temporary directory."""
from __future__ import annotations

import argparse
import importlib
import json
import shutil
import subprocess
import sys
import tempfile
import time
import types
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
PKG = "deep-spectral-segmentation_b200"
ex = importlib.import_module(PKG + ".extract")
utils = importlib.import_module(PKG + ".extract_utils")
synth = importlib.import_module(PKG + ".synth")
MODEL, K = "dino_vits16", 20


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"nvidia-smi unavailable: {e}"


def write_images(root: Path, n: int):
    from PIL import Image
    root.mkdir(parents=True)
    names = []
    for i, (H, W) in enumerate(synth.voc_shapes(n, seed=0)):
        names.append(f"im{i:05d}.jpg")
        Image.fromarray(synth.blobs_image(H, W, i).numpy()).save(root / names[-1], quality=90)
    return names


class HostColourRoute:
    """The former colour route inside extract_all: _color_inputs (PIL open + resize of every file on the launching
    thread) in place of the device resize extract_all calls for its colour images (resize.resize), and the decoder
    without the RGB-file check. That resize sees only the decoded batch: the files it stands for are those of the batch
    the decoders handed over last, which is the one extract_all is launching."""

    def __init__(self, images_root: str):
        self.root = images_root

    def __enter__(self):
        iop = ex.io_pipeline
        self.saved = ex.resize, iop.BatchAssembler, utils.ImagesDataset.load_raw_rgb_file
        root, launching = self.root, []

        class Assembler(iop.BatchAssembler):
            def __iter__(self_):
                for batch in super().__iter__():
                    launching[:] = [file[:-4] for file, _ in batch.items]
                    yield batch

        def host_resize(images_d, H_lr, W_lr, kind):
            return ex._color_inputs(root, launching, W_lr, H_lr, "rw" if kind == "u8" else "knn", images_d.device)
        ex.resize, iop.BatchAssembler = types.SimpleNamespace(resize=host_resize), Assembler
        utils.ImagesDataset.load_raw_rgb_file = utils.ImagesDataset.load_raw
        return self

    def __exit__(self, *exc):
        ex.resize, ex.io_pipeline.BatchAssembler, utils.ImagesDataset.load_raw_rgb_file = self.saved
        return False


def same_eigs(a: Path, b: Path) -> bool:
    for f in sorted(a.iterdir()):
        x, y = torch.load(f, weights_only=False), torch.load(b / f.name, weights_only=False)
        if not (torch.equal(torch.as_tensor(x["eigenvalues"]), torch.as_tensor(y["eigenvalues"]))
                and torch.equal(x["eigenvectors"], y["eigenvectors"])):
            return False
    return len(list(a.iterdir())) == len(list(b.iterdir()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=512)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    torch.set_grad_enabled(False)
    tmp = Path(tempfile.mkdtemp(prefix="dss_modes_probe_"))
    try:
        root = tmp / "images"
        names = write_images(root, a.n)
        lst = tmp / "list.txt"
        lst.write_text("\n".join(names) + "\n")
        colour = dict(image_color_lambda=10.0, which_color_matrix="knn")
        down = dict(image_downsample_factor=8)

        def run(variant, tag):
            out = tmp / tag
            t0 = time.perf_counter()
            if variant == "device":
                ex.extract_all(str(lst), str(root), MODEL, None, str(out), K=K, batch_size=a.batch, seed=0, **colour)
            elif variant == "host":
                with HostColourRoute(str(root)):
                    ex.extract_all(str(lst), str(root), MODEL, None, str(out), K=K, batch_size=a.batch, seed=0, **colour)
            elif variant == "fused":
                ex.extract_all(str(lst), str(root), MODEL, None, str(out), K=K, batch_size=a.batch, seed=0, **down)
            else:
                ex.extract_features(str(lst), str(root), MODEL, a.batch, str(tmp / f"{tag}_features"), seed=0)
                ex.extract_eigs(str(root), str(tmp / f"{tag}_features"), str(out), K=K, **down)
            torch.cuda.synchronize()
            return a.n / (time.perf_counter() - t0), out

        res = {"card": card(), "device": torch.cuda.get_device_name(0), "images": a.n, "batch_size": a.batch,
               "model": MODEL, "K": K}
        for name, pair in (("colour_knn_lambda10", ("device", "host")), ("downsample_factor8", ("fused", "files"))):
            outs = {}
            for v in pair:                                   # warm-up: module loads, weights, workspaces
                _, outs[v] = run(v, f"warm_{name}_{v}")
            rates = {v: [] for v in pair}
            for r in range(a.reps):
                for v in (pair if r % 2 == 0 else pair[::-1]):
                    rate, out = run(v, f"{name}_{v}_{r}")
                    rates[v].append(round(rate, 1))
                    shutil.rmtree(out)
            med = {v: sorted(x)[len(x) // 2] for v, x in rates.items()}
            res[name] = {"images_per_s": rates, "median": med, "ratio": round(med[pair[0]] / med[pair[1]], 3),
                         "eigs_bitwise_equal": same_eigs(outs[pair[0]], outs[pair[1]])}
        print(res["card"])
        line = json.dumps(res)
        print(line)
        if a.out:
            Path(a.out).mkdir(parents=True, exist_ok=True)
            (Path(a.out) / "extract_all_modes_probe.json").write_text(line + "\n")
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
