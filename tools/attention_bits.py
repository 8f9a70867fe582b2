"""SHA-256 digests of the fp16 attention kernel's output bytes on seeded inputs, written as the fixture that
tests/test_attention_bits_gpu.py recomputes and compares: a change to the kernel that must keep its bits is checked
against digests taken before it.

    python tools/attention_bits.py [--out tests/golden/attention_f16_bits.json]

Cases:
  - dss_op_attention_tc_f16 on seeded fp16 qkv at (B, T, heads) = (3, 901, 6), (2, 714, 6), (1, 3601, 12),
    (1, 6401, 12) and B = 2, heads = 6 at small T: every width class of an image's last key tile (1 .. 128 keys) and
    last query tiles with at most and with more than 64 rows;
  - the ragged fp16 forward (DinoViT.forward_k_ragged, ViT-S/16, seeded weights) on one batch of images whose token
    counts T mix the same classes; its K features pass through twelve ragged attention launches.
q, k and v are N(0, 1.5^2), the scale of the model's activations; every 7th query row is 6 times larger, so that its
softmax is dominated by a few keys."""
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

UNIFORM = [(3, 901, 6), (2, 714, 6), (1, 3601, 12), (1, 6401, 12)] + \
          [(2, T, 6) for T in (1, 5, 63, 64, 65, 127, 128, 129, 141, 151, 193)]
# ViT-S/16 pixel sizes: T = 2, 5, 63, 64, 65, 127, 128, 129, 141, 151, 193, 714, 901
RAGGED = [(16, 16), (32, 32), (32, 496), (112, 144), (128, 128), (144, 224), (16, 2032), (128, 256), (160, 224),
          (160, 240), (192, 256), (375, 500), (480, 480)]


def _pkg(sub):
    if str(ROOT) not in sys.path:
        sys.path.insert(0, str(ROOT))
    return importlib.import_module(f"{PKG}.{sub}")


def digest(t: torch.Tensor) -> str:
    return hashlib.sha256(t.contiguous().cpu().numpy().tobytes()).hexdigest()


def uniform_key(B, T, heads):
    return f"uniform_B{B}_T{T}_H{heads}"


def qkv(B, T, heads, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B * T, 3, heads * 64, generator=g) * 1.5
    x[::7, 0] *= 6.0
    return x.reshape(B * T, 3 * heads * 64).half()


def attention_uniform(B, T, heads):
    _lib = _pkg("_lib")
    lib = _lib.load()
    x = qkv(B, T, heads, seed=B * 100003 + T * 31 + heads).cuda()
    out = torch.empty(B * T, heads * 64, dtype=torch.float16, device="cuda")
    _lib.check(lib.dss_op_attention_tc_f16(x.data_ptr(), out.data_ptr(), B, T, heads, _lib.stream_ptr()), "attention")
    torch.cuda.synchronize()
    return out


def ragged_features():
    vit = _pkg("vit")
    model = vit.get_model("dino_vits16", seed=0, device="cuda", precision="fp16")[0]
    g = torch.Generator().manual_seed(0)
    ims = [torch.randint(0, 256, (H, W, 3), dtype=torch.uint8, generator=g).cuda() for H, W in RAGGED]
    k, _ = model.forward_k_ragged(ims)
    torch.cuda.synchronize()
    return k


def digests() -> dict:
    torch.set_grad_enabled(False)
    out = {uniform_key(*c): digest(attention_uniform(*c)) for c in UNIFORM}
    out["ragged_vits16_k"] = digest(ragged_features())
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=str(ROOT / "tests" / "golden" / "attention_f16_bits.json"))
    args = ap.parse_args()
    Path(args.out).parent.mkdir(parents=True, exist_ok=True)
    Path(args.out).write_text(json.dumps(digests(), indent=1, sort_keys=True) + "\n")
    print(args.out)


if __name__ == "__main__":
    main()
