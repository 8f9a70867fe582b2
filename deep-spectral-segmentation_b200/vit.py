"""Host side of the DINO ViT feature extractor (mirror of utils.get_model, extract/extract_utils.py:40-50).

Weights live in a plain dict of fp32 tensors with the upstream state_dict names; the device work happens in
libdss_b200 (csrc/vit.cu). ``torch.hub`` needs the network, so ``get_model`` builds the named architecture with the
upstream random-init recipe unless a checkpoint path is given."""
from __future__ import annotations

import ctypes as C
import math
from typing import Dict, List, Optional, Tuple

import torch

from . import _lib

# name -> (patch, dim, depth, heads)  (upstream hubconf: dino_vits16 / dino_vits8 / dino_vitb16 / dino_vitb8)
ARCHS = {"dino_vits16": (16, 384, 12, 6), "dino_vits8": (8, 384, 12, 6),
         "dino_vitb16": (16, 768, 12, 12), "dino_vitb8": (8, 768, 12, 12)}
MLP_RATIO = 4
LN_EPS = 1e-6
TRAIN_IMG = 224


PRECISIONS = ("fp16", "fp32")


def check_precision(precision: str) -> str:
    """'fp16' (fp16 operands, the throughput path) or 'fp32' (split-fp16 operands: the fp32 model's results)."""
    if precision not in PRECISIONS:
        raise ValueError(f"precision must be one of {PRECISIONS} (got {precision!r})")
    return precision


def arch(name: str):
    name = name.lower()
    if "dino" not in name or name not in ARCHS:
        raise ValueError(f"Cannot get model: {name}")  # extract_utils.py:48
    return ARCHS[name]


def _trunc_normal(shape, std, gen):
    t = torch.empty(shape)
    return torch.nn.init.trunc_normal_(t, std=std, generator=gen)


def random_state_dict(name: str, seed: int = 0) -> Dict[str, torch.Tensor]:
    """Upstream init recipe: trunc_normal(std=.02) for Linear/pos/cls, zero biases, LN (1,0), conv default."""
    P, d, depth, _ = arch(name)
    g = torch.Generator().manual_seed(int(seed))
    n0 = (TRAIN_IMG // P) ** 2
    sd: Dict[str, torch.Tensor] = {}
    fan_in = 3 * P * P
    bound = 1.0 / math.sqrt(fan_in)  # Conv2d default: kaiming_uniform(a=sqrt(5)) -> U(-1/sqrt(fan_in), +)
    sd["patch_embed.proj.weight"] = (torch.rand(d, 3, P, P, generator=g) * 2 - 1) * bound
    sd["patch_embed.proj.bias"] = (torch.rand(d, generator=g) * 2 - 1) * bound
    sd["cls_token"] = _trunc_normal((1, 1, d), 0.02, g)
    sd["pos_embed"] = _trunc_normal((1, n0 + 1, d), 0.02, g)
    for l in range(depth):
        p = f"blocks.{l}."
        sd[p + "norm1.weight"] = torch.ones(d); sd[p + "norm1.bias"] = torch.zeros(d)
        sd[p + "attn.qkv.weight"] = _trunc_normal((3 * d, d), 0.02, g); sd[p + "attn.qkv.bias"] = torch.zeros(3 * d)
        sd[p + "attn.proj.weight"] = _trunc_normal((d, d), 0.02, g); sd[p + "attn.proj.bias"] = torch.zeros(d)
        sd[p + "norm2.weight"] = torch.ones(d); sd[p + "norm2.bias"] = torch.zeros(d)
        sd[p + "mlp.fc1.weight"] = _trunc_normal((MLP_RATIO * d, d), 0.02, g); sd[p + "mlp.fc1.bias"] = torch.zeros(MLP_RATIO * d)
        sd[p + "mlp.fc2.weight"] = _trunc_normal((d, MLP_RATIO * d), 0.02, g); sd[p + "mlp.fc2.bias"] = torch.zeros(d)
    sd["norm.weight"] = torch.ones(d); sd["norm.bias"] = torch.zeros(d)
    return sd


def flat_param_order(name: str):
    """Deterministic parameter order used for the single NCCL broadcast of the weights."""
    _, _, depth, _ = arch(name)
    keys = ["patch_embed.proj.weight", "patch_embed.proj.bias", "cls_token", "pos_embed"]
    for l in range(depth):
        p = f"blocks.{l}."
        keys += [p + s for s in ("norm1.weight", "norm1.bias", "attn.qkv.weight", "attn.qkv.bias", "attn.proj.weight",
                                 "attn.proj.bias", "norm2.weight", "norm2.bias", "mlp.fc1.weight", "mlp.fc1.bias",
                                 "mlp.fc2.weight", "mlp.fc2.bias")]
    return keys + ["norm.weight", "norm.bias"]


class DinoViT:
    """Device handle around dss_vit_t. ``forward_k(images_u8)`` == the reference's hooked K features.

    ``precision='fp16'`` runs every ViT GEMM and the attention on fp16 operands (K features within about 3e-3 relative
    L2 of the fp32 model); ``'fp32'`` splits every operand into three fp16 values for fp32-equivalent products and
    reproduces the fp32 model, at three times the tensor-core work and weight memory."""

    def __init__(self, name: str, state_dict: Dict[str, torch.Tensor], device="cuda", precision: str = "fp16"):
        self.precision = check_precision(precision)
        self.name = name.lower()
        self.patch_size, self.dim, self.depth, self.num_heads = arch(self.name)
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise _lib.DssError("DinoViT needs a CUDA device: the hot path has no CPU implementation")
        self.lib = _lib.load()
        cfg = _lib.VitConfig(self.patch_size, self.dim, self.depth, self.num_heads, MLP_RATIO,
                             TRAIN_IMG // self.patch_size, LN_EPS)
        h = C.c_void_p()
        _lib.check(self.lib.dss_vit_create(C.byref(cfg), C.byref(h)), "dss_vit_create")
        self._h = h
        _lib.check(self.lib.dss_vit_set_precision(h, _lib.VIT_PRECISION[self.precision]), "dss_vit_set_precision")
        self._ws: Optional[torch.Tensor] = None
        self.load_state_dict(state_dict)

    def load_state_dict(self, sd: Dict[str, torch.Tensor]):
        with torch.cuda.device(self.device):
            dev = {k: sd[k].detach().to(self.device, torch.float32).contiguous() for k in flat_param_order(self.name)}
            blocks = (_lib.VitBlockWeights * self.depth)()
            names = {"ln1_w": "norm1.weight", "ln1_b": "norm1.bias", "qkv_w": "attn.qkv.weight", "qkv_b": "attn.qkv.bias",
                     "proj_w": "attn.proj.weight", "proj_b": "attn.proj.bias", "ln2_w": "norm2.weight",
                     "ln2_b": "norm2.bias", "fc1_w": "mlp.fc1.weight", "fc1_b": "mlp.fc1.bias",
                     "fc2_w": "mlp.fc2.weight", "fc2_b": "mlp.fc2.bias"}
            for l in range(self.depth):
                for f, n in names.items():
                    setattr(blocks[l], f, dev[f"blocks.{l}.{n}"].data_ptr())
            w = _lib.VitWeights(dev["patch_embed.proj.weight"].data_ptr(), dev["patch_embed.proj.bias"].data_ptr(),
                                dev["cls_token"].data_ptr(), dev["pos_embed"].data_ptr(), blocks,
                                dev["norm.weight"].data_ptr(), dev["norm.bias"].data_ptr())
            _lib.check(self.lib.dss_vit_load_weights(self._h, C.byref(w), _lib.stream_ptr(self.device)),
                       "dss_vit_load_weights")
            torch.cuda.current_stream(self.device).synchronize()

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                self.lib.dss_vit_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def _workspace(self, B, H, W) -> torch.Tensor:
        need = int(self.lib.dss_vit_workspace_bytes(self._h, B, H, W))
        if need == 0:
            raise _lib.DssError(f"image {H}x{W} is smaller than one patch")
        if self._ws is None or self._ws.numel() < need:
            self._ws = torch.empty(need, dtype=torch.uint8, device=self.device)
        return self._ws

    def _check_images(self, images_u8):
        _lib.require_cuda(images_u8, "images_u8")
        if images_u8.dtype != torch.uint8 or images_u8.dim() != 4 or images_u8.shape[-1] != 3:
            raise _lib.DssError("images_u8 must be uint8 [B, H, W, 3]")
        return images_u8.contiguous()

    @torch.no_grad()
    def forward_k(self, images_u8: torch.Tensor, which_block: int = -1, out: Optional[torch.Tensor] = None):
        """images_u8 [B,H,W,3] uint8 CUDA (RGB) -> K features [B, N, d] fp32 (extract.py:94-98)."""
        img = self._check_images(images_u8)
        B, H, W, _ = img.shape
        N = (H // self.patch_size) * (W // self.patch_size)
        with torch.cuda.device(self.device):
            ws = self._workspace(B, H, W)
            if out is None:
                out = torch.empty(B, N, self.dim, dtype=torch.float32, device=self.device)
            _lib.check(self.lib.dss_vit_forward_k(self._h, img.data_ptr(), B, H, W, which_block, out.data_ptr(),
                                                  ws.data_ptr(), ws.numel(), _lib.stream_ptr(self.device)),
                       "dss_vit_forward_k")
        return out

    @torch.no_grad()
    def forward_tokens(self, images_u8: torch.Tensor, n_blocks: int):
        """Residual stream [B, T, d] after n_blocks full blocks (parity/debug hook)."""
        img = self._check_images(images_u8)
        B, H, W, _ = img.shape
        T = (H // self.patch_size) * (W // self.patch_size) + 1
        with torch.cuda.device(self.device):
            ws = self._workspace(B, H, W)
            out = torch.empty(B, T, self.dim, dtype=torch.float32, device=self.device)
            _lib.check(self.lib.dss_vit_forward_tokens(self._h, img.data_ptr(), B, H, W, n_blocks, out.data_ptr(),
                                                       ws.data_ptr(), ws.numel(), _lib.stream_ptr(self.device)),
                       "dss_vit_forward_tokens")
        return out

    @torch.no_grad()
    def forward_cls(self, images_u8: torch.Tensor) -> torch.Tensor:
        """The model's own forward (upstream VisionTransformer.forward): all blocks, final norm, CLS token -> [B, d].
        This is what the reference calls on bounding-box crops (extract.py:537-541)."""
        img = self._check_images(images_u8)
        B, H, W, _ = img.shape
        with torch.cuda.device(self.device):
            ws = self._workspace(B, H, W)
            out = torch.empty(B, self.dim, dtype=torch.float32, device=self.device)
            _lib.check(self.lib.dss_vit_forward_cls(self._h, img.data_ptr(), B, H, W, out.data_ptr(), ws.data_ptr(),
                                                    ws.numel(), _lib.stream_ptr(self.device)), "dss_vit_forward_cls")
        return out

    __call__ = forward_cls

    @torch.no_grad()
    def forward_last(self, images_u8: torch.Tensor, which: str = "k", pad: bool = True, feats: bool = True,
                     cls_attn: bool = False):
        """Last-block outputs for object localization (object-localization/main.py:219-322). pad=True zero-pads the
        normalised image to multiples of the patch size (the grid is ceil(H/P) x ceil(W/P)); pad=False crops.
        Returns (features [B, N, d] fp32 -- the q, k or v third of the last qkv projection, CLS row dropped -- or None,
        CLS attention [B, heads, N] fp32 -- get_last_selfattention(...)[:, :, 0, 1:] -- or None)."""
        img = self._check_images(images_u8)
        B, H, W, _ = img.shape
        P = self.patch_size
        N = (-(-H // P)) * (-(-W // P)) if pad else (H // P) * (W // P)
        w = {"q": 0, "k": 1, "v": 2}.get(which)
        if w is None:
            raise ValueError(f"which must be 'q', 'k' or 'v' (got {which!r})")
        with torch.cuda.device(self.device):
            need = int(self.lib.dss_vit_forward_last_workspace_bytes(self._h, B, H, W, 1 if pad else 0))
            if need == 0:
                raise _lib.DssError(f"image {H}x{W} is smaller than one patch")
            if self._ws is None or self._ws.numel() < need:
                self._ws = torch.empty(need, dtype=torch.uint8, device=self.device)
            f = torch.empty(B, N, self.dim, dtype=torch.float32, device=self.device) if feats else None
            a = torch.empty(B, self.num_heads, N, dtype=torch.float32, device=self.device) if cls_attn else None
            _lib.check(self.lib.dss_vit_forward_last(self._h, img.data_ptr(), B, H, W, 1 if pad else 0, w, _lib.ptr(f),
                                                     _lib.ptr(a), self._ws.data_ptr(), self._ws.numel(),
                                                     _lib.stream_ptr(self.device)), "dss_vit_forward_last")
        return f, a

    def _ragged_args(self, images, dims):
        """(packed uint8 [sum H W, 3] CUDA tensor, host int32 dims [B, 2]) from a list of [H, W, 3] images or a packed
        tensor plus dims."""
        if dims is None:
            packed, dims = pack_images(images)
        else:
            packed, dims = images, torch.as_tensor(dims, dtype=torch.int32).reshape(-1, 2).contiguous()
        _lib.require_cuda(packed, "images")
        if packed.dtype != torch.uint8 or packed.shape[-1] != 3 or packed.numel() != 3 * int((dims[:, 0].long() * dims[:, 1].long()).sum()):
            raise _lib.DssError("ragged images must be uint8 RGB, packed [sum H*W, 3] as dims describes")
        return packed.contiguous(), dims

    def _ragged_workspace(self, dims: torch.Tensor, mode: int) -> torch.Tensor:
        need = int(self.lib.dss_vit_ragged_workspace_bytes(self._h, dims.data_ptr(), dims.shape[0], mode))
        if need == 0:
            # the entry point names the offending image
            _lib.check(_lib.DSS_ERR_BAD_ARG, "dss_vit_ragged_workspace_bytes")
        if self._ws is None or self._ws.numel() < need:
            self._ws = torch.empty(need, dtype=torch.uint8, device=self.device)
        return self._ws

    @torch.no_grad()
    def forward_k_ragged(self, images, dims=None, which_block: int = -1):
        """forward_k over images of different sizes in one forward. ``images``: a list of uint8 [H, W, 3] CUDA tensors,
        or a packed uint8 [sum H*W, 3] tensor with ``dims`` [B, 2] = (H, W) per image. Returns (k [sum N_b, d] fp32,
        rows): image b's features are k[rows[b][0]:rows[b][1]], the bits forward_k gives for that image alone."""
        packed, dims = self._ragged_args(images, dims)
        B, P = dims.shape[0], self.patch_size
        rows = ragged_rows(dims.tolist(), P)
        with torch.cuda.device(self.device):
            ws = self._ragged_workspace(dims, _lib.VIT_RAGGED_K)
            out = torch.empty(rows[-1][1] if rows else 0, self.dim, dtype=torch.float32, device=self.device)
            _lib.check(self.lib.dss_vit_forward_k_ragged(self._h, packed.data_ptr(), dims.data_ptr(), B, which_block,
                                                         out.data_ptr(), ws.data_ptr(), ws.numel(),
                                                         _lib.stream_ptr(self.device)), "dss_vit_forward_k_ragged")
        return out, rows

    @torch.no_grad()
    def forward_cls_ragged(self, images, dims=None):
        """forward_cls over images of different sizes in one forward (arguments as forward_k_ragged). Returns
        (cls [B, d] fp32, rows) with rows[b] = (b, b + 1)."""
        packed, dims = self._ragged_args(images, dims)
        B = dims.shape[0]
        with torch.cuda.device(self.device):
            ws = self._ragged_workspace(dims, _lib.VIT_RAGGED_CLS)
            out = torch.empty(B, self.dim, dtype=torch.float32, device=self.device)
            _lib.check(self.lib.dss_vit_forward_cls_ragged(self._h, packed.data_ptr(), dims.data_ptr(), B,
                                                           out.data_ptr(), ws.data_ptr(), ws.numel(),
                                                           _lib.stream_ptr(self.device)), "dss_vit_forward_cls_ragged")
        return out, [(b, b + 1) for b in range(B)]

    @torch.no_grad()
    def forward_last_ragged(self, images, dims=None, which: str = "k", pad: bool = True, feats: bool = True,
                            cls_attn: bool = False, n_max: Optional[int] = None):
        """forward_last over images of different sizes in one forward (images / dims as forward_k_ragged). Outputs are
        padded to n_max rows per image (default: the batch's largest N_b): (features [B, n_max, d] fp32 or None, CLS
        attention [B, heads, n_max] fp32 or None, grids) with grids[b] = (N_b, gh_b, gw_b). Image b's first N_b rows are
        the bits forward_last gives for that image alone; the rows after them are +0.0."""
        w = {"q": 0, "k": 1, "v": 2}.get(which)
        if w is None:
            raise ValueError(f"which must be 'q', 'k' or 'v' (got {which!r})")
        packed, dims = self._ragged_args(images, dims)
        B = dims.shape[0]
        grids = ragged_grids(dims.tolist(), self.patch_size, pad)
        n = max(1, *(g[0] for g in grids)) if n_max is None else int(n_max)
        with torch.cuda.device(self.device):
            ws = self._ragged_workspace(dims, _lib.VIT_RAGGED_PAD if pad else _lib.VIT_RAGGED_K)
            f = torch.empty(B, n, self.dim, dtype=torch.float32, device=self.device) if feats else None
            a = torch.empty(B, self.num_heads, n, dtype=torch.float32, device=self.device) if cls_attn else None
            _lib.check(self.lib.dss_vit_forward_last_ragged(self._h, packed.data_ptr(), dims.data_ptr(), B,
                                                            1 if pad else 0, w, _lib.ptr(f), n, _lib.ptr(a),
                                                            ws.data_ptr(), ws.numel(), _lib.stream_ptr(self.device)),
                       "dss_vit_forward_last_ragged")
        return f, a, grids

    def pos_embed(self, Hp: int, Wp: int) -> torch.Tensor:
        """The positional embedding [Hp * Wp + 1, d] fp32 the forwards add for an Hp x Wp patch grid (forward_k's
        identity rule: the stored grid for a square grid0 x grid0 grid)."""
        dims = torch.tensor([[Hp * self.patch_size, Wp * self.patch_size]], dtype=torch.int32)
        with torch.cuda.device(self.device):
            ws = self._ragged_workspace(dims, _lib.VIT_RAGGED_K)
            out = torch.empty(Hp * Wp + 1, self.dim, dtype=torch.float32, device=self.device)
            _lib.check(self.lib.dss_vit_pos_embed_ragged(self._h, dims.data_ptr(), 1, _lib.VIT_RAGGED_K, out.data_ptr(),
                                                         ws.data_ptr(), ws.numel(), _lib.stream_ptr(self.device)),
                       "dss_vit_pos_embed_ragged")
        return out


def pack_images(images) -> Tuple[torch.Tensor, torch.Tensor]:
    """A list of uint8 [H, W, 3] images -> (packed [sum H*W, 3], host int32 dims [B, 2]), images one after another:
    the input layout of the ragged forwards."""
    if len(images) == 0:
        raise _lib.DssError("a ragged batch needs at least one image")
    for im in images:
        if im.dtype != torch.uint8 or im.dim() != 3 or im.shape[-1] != 3:
            raise _lib.DssError("ragged images must be uint8 [H, W, 3]")
    dims = torch.tensor([[int(im.shape[0]), int(im.shape[1])] for im in images], dtype=torch.int32)
    return torch.cat([im.reshape(-1, 3) for im in images]), dims


def ragged_rows(dims, patch_size: int) -> List[Tuple[int, int]]:
    """Row range (start, end) of each image's features in forward_k_ragged's packed output: N_b = (H_b // P)(W_b // P)
    rows per image, image after image."""
    rows, r = [], 0
    for H, W in dims:
        n = (int(H) // patch_size) * (int(W) // patch_size)
        rows.append((r, r + n))
        r += n
    return rows


def ragged_grids(dims, patch_size: int, pad: bool) -> List[Tuple[int, int, int]]:
    """(N_b, gh_b, gw_b) of each image of forward_last_ragged: the ceil grid with pad, else the crop."""
    out = []
    for H, W in dims:
        H, W = int(H), int(W)
        gh, gw = (-(-H // patch_size), -(-W // patch_size)) if pad else (H // patch_size, W // patch_size)
        out.append((gh * gw, gh, gw))
    return out


def pos_embed_interp_host(pos_embed: torch.Tensor, grid0: int, Hp: int, Wp: int) -> torch.Tensor:
    """CPU entry point of the library's positional-embedding interpolation (no GPU needed)."""
    lib = _lib.load()
    src = pos_embed.detach().to("cpu", torch.float32).reshape(grid0 * grid0 + 1, -1).contiguous()
    out = torch.empty(Hp * Wp + 1, src.shape[1], dtype=torch.float32)
    _lib.check(lib.dss_pos_embed_interp_host(src.data_ptr(), grid0, src.shape[1], Hp, Wp, out.data_ptr()))
    return out


# upstream checkpoint file names (hubconf.py of facebookresearch/dino), looked up in the torch.hub cache
HUB_FILES = {"dino_vits16": "dino_deitsmall16_pretrain.pth", "dino_vits8": "dino_deitsmall8_pretrain.pth",
             "dino_vitb16": "dino_vitbase16_pretrain.pth", "dino_vitb8": "dino_vitbase8_pretrain.pth"}


def clean_state_dict(sd: dict) -> Dict[str, torch.Tensor]:
    """Accepts a backbone state_dict or a full DINO training checkpoint ({'teacher': ...}, 'module.' / 'backbone.'
    prefixes, projection-head entries) and returns the backbone entries under the upstream names."""
    for key in ("teacher", "state_dict", "model"):
        if isinstance(sd, dict) and key in sd and isinstance(sd[key], dict):
            sd = sd[key]
    out = {}
    for k, v in sd.items():
        for prefix in ("module.", "backbone."):
            if k.startswith(prefix):
                k = k[len(prefix):]
        if k.startswith("head."):
            continue
        out[k] = v
    return out


def find_checkpoint(name: str, checkpoint: Optional[str] = None) -> Optional[str]:
    """Explicit path > $DSS_DINO_CHECKPOINT (a file, or a directory holding {name}.pth / the upstream file name) >
    the torch.hub checkpoint cache (where torch.hub.load of the reference, extract_utils.py:42, leaves the weights)."""
    import os
    from pathlib import Path
    if checkpoint:
        return checkpoint
    cands = []
    env = os.environ.get("DSS_DINO_CHECKPOINT") or os.environ.get("DINO_CHECKPOINT")
    if env:
        e = Path(env)
        cands += [e] if e.is_file() else [e / f"{name}.pth", e / HUB_FILES[name]]
    try:
        hub = Path(torch.hub.get_dir()) / "checkpoints"
        cands.append(hub / HUB_FILES[name])
    except Exception:
        pass
    for c in cands:
        if c.is_file():
            return str(c)
    return None


def get_model(name: str, checkpoint: Optional[str] = None, seed: Optional[int] = None, device="cuda", state_dict=None,
              random_init: bool = False, precision: str = "fp16"):
    """Mirror of utils.get_model (extract_utils.py:40-50): returns (model, val_transform, patch_size, num_heads).

    ``val_transform`` is None: ToTensor + Normalize are fused into the device im2col kernel, the model takes the
    raw uint8 RGB image. The reference downloads the pretrained DINO weights through torch.hub; here they come from
    ``state_dict``, ``checkpoint``, $DSS_DINO_CHECKPOINT or the torch.hub cache (see find_checkpoint). Without any of
    them the call RAISES -- features of a randomly initialised ViT under the name 'dino_vits16' would be garbage in
    the reference's file layout -- unless the caller opts in with ``random_init=True`` or a ``seed`` (tests, benchmarks:
    the upstream init recipe), which prints a loud warning. ``precision``: see DinoViT."""
    check_precision(precision)
    name = name.lower()
    arch(name)
    if state_dict is None:
        ckpt = find_checkpoint(name, checkpoint)
        if ckpt:
            state_dict = clean_state_dict(torch.load(ckpt, map_location="cpu"))
        elif random_init or seed is not None:
            import sys
            print(f"WARNING: {name}: no pretrained checkpoint given or found -- using RANDOMLY INITIALISED weights "
                  f"(seed {seed or 0}); the features are only meaningful for tests and benchmarks", file=sys.stderr)
            state_dict = random_state_dict(name, seed or 0)
        else:
            raise _lib.DssError(
                f"{name}: pretrained DINO weights not found. The reference downloads them with torch.hub "
                f"(extract_utils.py:42), which needs the network; pass checkpoint=<{HUB_FILES[name]}>, set "
                "$DSS_DINO_CHECKPOINT, or opt into random weights with random_init=True / seed=<int> (tests only).")
    model = DinoViT(name, state_dict, device=device, precision=precision)
    return model, None, model.patch_size, model.num_heads
