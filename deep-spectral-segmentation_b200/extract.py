"""Drop-in replacements for the reference's hot-path callables (extract/extract.py):

    extract_features  (:21-116)   images -> features/{id}.pth      {'k','indices','file','id','model_name','patch_size','shape'}
    _extract_eig      (:119-244)  one features file -> eigs/{image_id}.pth  {'eigenvalues','eigenvectors'}
    extract_eigs      (:247-280)  directory of features files -> eigs files (batched on the GPU)
    extract_all                   fused: images -> both file layouts (+ optional segmentations) without the disk round-trip
    extract_single_region_segmentations / extract_multi_region_segmentations  (:283-411)  eigs -> PNG masks (GPU kernels)
    extract_bboxes        (:429-497)  segment bounding boxes after erosion / dilation (GPU kernel)
    extract_bbox_features (:500-544)  DINO CLS embedding of every bounding-box crop
    extract_bbox_clusters (:547-599)  normalise, PCA, K-means of the box features (GPU kernels)
    extract_semantic_segmentations (:602-647)  segment -> cluster lookup on every label map (host)
    extract_crf_segmentations (:650-735)  dense-CRF mean field to pixel resolution (GPU permutohedral lattices)

Same argument names, defaults, file layouts and skip-if-exists behaviour; all arithmetic runs in libdss_b200. Host I/O
(decode, pinned staging, .pth / PNG writers) is threaded, see io_pipeline.py."""
from __future__ import annotations

from collections import defaultdict
from pathlib import Path
from dataclasses import dataclass
from typing import Callable, Dict, List, Optional, Tuple

import numpy as np
import torch

from . import _lib, cluster, io_pipeline, resize, segment, spectral
from . import extract_utils as utils
from . import vit as vit_mod

torch.set_grad_enabled(False)  # extract.py:838


def _rank_world() -> Tuple[int, int]:
    """(rank, world size) of a multi-process launch (torchrun or anything else that sets RANK / WORLD_SIZE); (0, 1)
    otherwise. Images are the only parallel axis of the path (SURVEY 8e): every command below gives rank r the items
    r, r + R, r + 2R, ... of its sorted work list, on the GPU LOCAL_RANK; the ranks exchange nothing and write
    disjoint files, so `torchrun --nproc-per-node 8 extract.py extract_all ...` is the multi-GPU form of the command."""
    import os
    world = int(os.environ.get("WORLD_SIZE", "1") or 1)
    rank = int(os.environ.get("RANK", "0") or 0)
    if world < 1 or not (0 <= rank < world):
        raise ValueError(f"RANK={rank} outside WORLD_SIZE={world}")
    return rank, world


def _my_share(items: list) -> list:
    rank, world = _rank_world()
    return items if world == 1 else items[rank::world]


def _device():
    if not torch.cuda.is_available():
        raise _lib.DssError("a CUDA device is required: the hot path has no CPU implementation")
    import os
    if _rank_world()[1] > 1 and os.environ.get("LOCAL_RANK") is not None:
        torch.cuda.set_device(int(os.environ["LOCAL_RANK"]) % torch.cuda.device_count())
    return torch.device("cuda", torch.cuda.current_device())


def _feature_files(output_dir, images, rows, model_name, patch_size):
    """Writer items (io_pipeline) for the feature dicts of one batch, the dict the reference saves at extract.py:98-110:
    image j = (file, index, H, W) has the k rows rows[j] = (r0, r1) of arrays['k'], saved as [1, N, d] fp32; its shape
    is the un-cropped (1, 3, H, W)."""
    out = []
    for (file, index, H, W), (r0, r1) in zip(images, rows):
        extra = {"file": file, "id": Path(file).stem, "model_name": model_name, "patch_size": patch_size, "shape": (1, 3, H, W)}
        out.append((str(Path(output_dir) / f"{Path(file).stem}.pth"), r0, extra,
                    {"k": ("rows1", ("k", r1 - r0)), "indices": ("tensor0d", index)}))
    return out


def _feature_dict(k: torch.Tensor, index: int, file: str, model_name: str, patch_size: int, H: int, W: int) -> dict:
    """The features file the writers save for one image (k is [1, N, d] fp32 on the CPU)."""
    return io_pipeline._materialise({"k": k[0].numpy()}, *_feature_files("", [(file, index, H, W)], [(0, k.shape[1])],
                                                                          model_name, patch_size)[0][1:])


def _eigs_content(which_matrix: str, evals: torch.Tensor, evecs: Optional[torch.Tensor] = None):
    """The eigs files of a batch (extract.py:242) from descending CPU eigenvalues [B, K] (and eigenvectors [B, K, N]) ->
    (writer arrays, fields of each file's dict; io_pipeline._materialise). The reference's 'affinity' branch keeps the
    ascending numpy eigenvalues eigsh returned beside eigenvectors flipped to descending order (extract.py:171-172)."""
    affinity = which_matrix == "affinity"
    arrays = {"evals": (evals.flip(1) if affinity else evals).numpy()}
    fields = {"eigenvalues": ("np_slice" if affinity else "slice", "evals")}
    if evecs is not None:
        arrays["evecs"], fields["eigenvectors"] = evecs.numpy(), ("slice", "evecs")
    return arrays, fields


class _Batcher:
    """Groups items by a shape key. A group is handed to ``flush`` when it reaches ``batch_size``; when more than
    ``max_pending`` items are waiting in total (data sets with hundreds of distinct image sizes, e.g. VOC), the
    largest group is flushed early, so host memory stays bounded and outputs appear steadily."""

    def __init__(self, batch_size: int, flush, max_pending: Optional[int] = None):
        self.batch_size = max(1, int(batch_size))
        self.flush_fn = flush
        self.max_pending = max_pending if max_pending is not None else 8 * self.batch_size
        self.groups: Dict[object, list] = defaultdict(list)
        self.count = 0

    def _flush(self, key):
        items = self.groups.pop(key, [])
        self.count -= len(items)
        if items:
            self.flush_fn(key, items)

    def add(self, key, item):
        self.groups[key].append(item)
        self.count += 1
        if len(self.groups[key]) >= self.batch_size:
            self._flush(key)
        elif self.count > self.max_pending:
            self._flush(max(self.groups, key=lambda k: len(self.groups[k])))

    def finish(self):
        for key in list(self.groups.keys()):
            self._flush(key)


def extract_features(images_list: str, images_root: Optional[str], model_name: str, batch_size: int, output_dir: str,
                     which_block: int = -1, checkpoint: Optional[str] = None, seed: Optional[int] = None,
                     random_init: bool = False, yes: Optional[bool] = None, num_workers: Optional[int] = None,
                     num_workers_out: int = 4, writer: str = "process", precision: str = "fp16"):
    """
    Extract features from a list of images. ``precision='fp32'`` computes the ViT on split-fp16 operands and
    reproduces the fp32 model's features (see vit.DinoViT); the default 'fp16' is the faster path.

    Example:
        python extract.py extract_features \
            --images_list "./data/VOC2012/lists/images.txt" \
            --images_root "./data/VOC2012/images" \
            --output_dir "./data/VOC2012/features/dino_vits16" \
            --model_name dino_vits16 \
            --batch_size 1
    """
    vit_mod.check_precision(precision)
    utils.make_output_dir(output_dir, assume_yes=yes)
    model_name = model_name.lower()
    if not ("dino" in model_name or "mocov3" in model_name):
        raise ValueError(model_name)
    dev = _device()
    model, _, patch_size, _ = utils.get_model(model_name, checkpoint=checkpoint, seed=seed, device=dev,
                                              random_init=random_init, precision=precision)
    filenames = Path(images_list).read_text().splitlines()
    dataset = utils.ImagesDataset(filenames=filenames, images_root=images_root)
    print(f"Dataset size: {len(dataset)=}")
    # batch_size images per forward in list order, whatever their sizes: one ragged ViT forward per batch
    ring = io_pipeline.PackedRing(dev)
    batch_size = max(1, int(batch_size))

    with io_pipeline.make_writer(writer, num_workers_out) as wr:
        def flush(items):
            slot, host, dims = ring.stage([it[0] for it in items])
            k, rows = model.forward_k_ragged(ring.to_device(slot, host), dims, which_block=which_block)
            images = [(file, index, int(image.shape[0]), int(image.shape[1])) for image, file, index in items]
            wr.submit_batch({"k": k.cpu().numpy()}, _feature_files(output_dir, images, rows, model_name, patch_size))

        batch = []
        todo = []
        for i in _my_share(list(range(len(dataset)))):
            output_file = Path(output_dir) / f"{Path(dataset.filenames[i]).stem}.pth"
            if output_file.is_file():
                print(f"Skipping existing file {str(output_file)}")
            else:
                todo.append(i)
        for image, file, index in io_pipeline.ImagePrefetcher(dataset.__getitem__, todo, num_workers):
            batch.append((image, file, index))
            if len(batch) == batch_size:
                flush(batch)
                batch = []
        if batch:
            flush(batch)
    print(f"Saved features to {output_dir}")


def _load_image_lr_u8(images_root: str, image_id: str, W_lr: int, H_lr: int) -> np.ndarray:
    """extract.py:199-203: PIL open (no .convert), BILINEAR resize of the WHOLE image to (W_lr, H_lr) -> uint8 pixels."""
    from PIL import Image
    image_file = str(Path(images_root) / f"{image_id}.jpg")
    return np.array(Image.open(image_file).resize((W_lr, H_lr), Image.BILINEAR))


@dataclass(frozen=True)
class _EigOptions:
    """extract_eigs' options of the eigen stage (extract.py:119-132), checked when made: every command that runs the
    stage refuses unsupported options before any file or device work."""
    K: int
    which_matrix: str
    which_color_matrix: str
    normalize: bool
    threshold_at_zero: bool
    lapnorm: bool
    image_downsample_factor: Optional[int]
    image_color_lambda: float

    def __post_init__(self):
        if self.which_matrix == "affinity_torch":
            raise RuntimeError("which_matrix='affinity_torch' calls torch.eig, which PyTorch removed (dead in the reference)")
        if self.which_matrix not in ("laplacian", "matting_laplacian", "affinity", "affinity_svd"):
            raise ValueError(f"unknown which_matrix={self.which_matrix!r}")
        if self.colour and self.which_color_matrix not in ("knn", "rw"):
            raise ValueError(f"unknown which_color_matrix={self.which_color_matrix!r} (the reference knows 'knn' and 'rw')")
        if self.laplacian and self.image_downsample_factor is not None and int(self.image_downsample_factor) <= 0:
            raise ValueError(f"image_downsample_factor={self.image_downsample_factor} must be a positive integer")

    @property
    def laplacian(self) -> bool:
        return self.which_matrix in ("laplacian", "matting_laplacian")

    @property
    def colour(self) -> bool:
        """Colour terms in the affinity: only the Laplacian modes have them (extract.py:190-214)."""
        return self.laplacian and self.image_color_lambda > 0

    def factor(self, patch_size: int) -> int:
        """The Laplacian modes solve on the (H_pad // factor) x (W_pad // factor) grid (extract.py:175-188; factor = the
        patch size by default); the affinity modes always on the patch grid."""
        if self.image_downsample_factor is None or not self.laplacian:
            return patch_size
        return int(self.image_downsample_factor)


def _color_inputs(images_root, image_ids, W_lr, H_lr, which_color_matrix, dev):
    """Low-resolution colour images of a batch on the device: fp32 /255 for 'knn', the uint8 pixels for 'rw'."""
    lr = np.stack([_load_image_lr_u8(images_root, i, W_lr, H_lr) for i in image_ids]).reshape(len(image_ids), H_lr * W_lr, 3)
    if which_color_matrix == "rw":
        return torch.from_numpy(np.ascontiguousarray(lr)).to(dev)
    return torch.from_numpy((lr / 255.0).astype(np.float32)).to(dev)


def _eigen_stage(feats: torch.Tensor, grid: Tuple[int, int], patch_size: int, opts: _EigOptions,
                 colour: Callable[[int, int], torch.Tensor]):
    """extract.py:148-240 for device features [B, Hp*Wp, d] fp32 of one patch grid (Hp, Wp) -> (solve, (H_lr, W_lr)):
    ``solve(sel, max_steps)`` enqueues the eigensolve of batch rows ``sel`` (None: all) -> device (eigenvalues [B, K],
    eigenvectors [B, K, H_lr * W_lr], info), as _solve_with_retry / _retry_bad_rows call it. Affinity modes solve on the
    patch grid; Laplacian modes on opts.factor's grid, features normalised, then up-sampled (extract.py:179-188), with
    ``colour(H_lr, W_lr)`` the low-resolution image of the colour terms. Nothing here waits for the device."""
    Hp, Wp = grid
    if not opts.laplacian:
        def solve(sel, max_steps):
            f = feats if sel is None else feats[sel]
            return spectral.affinity_eigs(f, opts.K, opts.which_matrix, opts.normalize, opts.threshold_at_zero,
                                          max_steps=max_steps)
        return solve, grid
    factor = opts.factor(patch_size)
    lr_size = (Hp * patch_size // factor, Wp * patch_size // factor)
    normalize = opts.normalize
    if lr_size != grid:
        if normalize:
            feats, normalize = spectral.normalize_rows(feats), False
        feats = spectral.upsample_bilinear(feats, Hp, Wp, *lr_size)
    rgb_lr = colour(*lr_size) if opts.colour else None

    def solve(sel, max_steps):
        f = feats if sel is None else feats[sel]
        rgb = rgb_lr if (sel is None or rgb_lr is None) else rgb_lr[sel]
        return spectral.laplacian_eigs(f, opts.K, normalize, opts.threshold_at_zero, opts.lapnorm, rgb, lr_size,
                                       opts.image_color_lambda, max_steps=max_steps,
                                       which_color_matrix=opts.which_color_matrix)[:3]
    return solve, lr_size


def _warn_eigs(which_matrix: str, info: torch.Tensor, failed: List[str]):
    """A solved and retried batch's warnings: images without a file; an 'affinity' eigenvalue eigsh('LM') would pick."""
    if failed:
        print(f"Warning: eigensolver did not converge for {failed}; no file is written for them")
    if which_matrix == "affinity" and bool((info[:, 2] != 0).any()):
        print("Warning: a negative eigenvalue exceeds the K-th largest in magnitude; eigsh(which='LM') would pick it")


def _bad_rows(evals: torch.Tensor, evecs: torch.Tensor, info: torch.Tensor) -> List[int]:
    """Rows of a batch (CPU tensors) whose solve did not reach the tolerance or came back non-finite. Three tensor
    operations per batch: a per-image Python loop here cost more main-thread time than launching the kernels did."""
    ok = (info[:, 1] != 0) & torch.isfinite(evecs).flatten(1).all(1) & torch.isfinite(evals).flatten(1).all(1)
    return (~ok).nonzero().flatten().tolist()


def _retry_bad_rows(solve, evals: torch.Tensor, evecs: torch.Tensor, info: torch.Tensor, N: int) -> List[int]:
    """Second half of the solve of a batch whose default-budget results (CPU tensors) are given: re-solves the rows whose
    Lanczos run did not reach its tolerance or came back non-finite through ``solve(rows, max_steps)`` with the largest
    Krylov space the solver fits -- N - 1 steps up to N = 3816, fewer above (spectral.max_steps; 1602 at N = 6400) --
    and writes the converged ones into evals / evecs / info. Where that budget is no larger than the default (N <= 321,
    or N >= 7893) a retry would only repeat the first run, so nothing is re-solved. The reference's own safety net is
    a second eigsh call (which='SM', extract.py:226-234). Returns the rows that still failed."""
    bad = _bad_rows(evals, evecs, info)
    if not bad:
        return []
    steps = spectral.max_steps(N)
    if steps <= spectral.DEFAULT_MAX_STEPS:
        return bad
    failed = []
    ev2, vec2, info2 = (t.cpu() for t in solve(bad, steps))
    for j, i in enumerate(bad):
        ok = int(info2[j, 1]) == 1 and bool(torch.isfinite(vec2[j]).all() and torch.isfinite(ev2[j]).all())
        if ok:
            evals[i], evecs[i], info[i] = ev2[j], vec2[j], info2[j]
        else:
            failed.append(i)
    return failed


def _solve_with_retry(solve, n_images: int, N: int):
    """Runs ``solve(sel, max_steps)`` (sel = None for the whole batch, else a list of batch rows) with the default
    budget, then _retry_bad_rows. Returns (eigenvalues, eigenvectors, info, failed rows) on the CPU."""
    evals, evecs, info = (t.cpu() for t in solve(None, 0))
    failed = _retry_bad_rows(solve, evals, evecs, info, N)
    return evals, evecs, info, failed


def _eigs_for_group(data_dicts: List[dict], opts: _EigOptions, images_root, which_features, dev
                    ) -> Tuple[torch.Tensor, torch.Tensor, List[int]]:
    """One GPU batch: feature dicts whose patch grids have the same size -> (eigenvalues [B,K], eigenvectors [B,K,N],
    rows whose solve failed even after the retry) on the CPU. The colour images are read from the image files."""
    feats = torch.stack([d[which_features].squeeze() for d in data_dicts]).to(torch.float32)
    feats = feats.pin_memory().to(dev, non_blocking=True)
    P, H_patch, W_patch = utils.get_image_sizes(data_dicts[0])[4:7]
    image_ids = [d["file"][:-4] for d in data_dicts]
    solve, (H_lr, W_lr) = _eigen_stage(
        feats, (H_patch, W_patch), P, opts,
        lambda h, w: _color_inputs(images_root, image_ids, w, h, opts.which_color_matrix, dev))
    evals, evecs, info, failed = _solve_with_retry(solve, len(data_dicts), H_lr * W_lr)
    _warn_eigs(opts.which_matrix, info, [data_dicts[i]["id"] for i in failed])
    return evals, evecs, failed


def _extract_eig(inp: Tuple[int, str], K: int, images_root: str, output_dir: str, which_matrix: str = "laplacian",
                 which_features: str = "k", normalize: bool = True, lapnorm: bool = True,
                 which_color_matrix: str = "knn", threshold_at_zero: bool = True,
                 image_downsample_factor: Optional[int] = None, image_color_lambda: float = 10):
    """Single-image worker with the reference's signature (extract.py:119-132); writes {output_dir}/{image_id}.pth."""
    opts = _EigOptions(K=K, which_matrix=which_matrix, which_color_matrix=which_color_matrix, normalize=normalize,
                       threshold_at_zero=threshold_at_zero, lapnorm=lapnorm,
                       image_downsample_factor=image_downsample_factor, image_color_lambda=image_color_lambda)
    index, features_file = inp
    data_dict = torch.load(features_file, map_location="cpu")
    image_id = data_dict["file"][:-4]
    output_file = Path(output_dir) / f"{image_id}.pth"
    if output_file.is_file():
        print(f"Skipping existing file {str(output_file)}")
        return
    evals, evecs, failed = _eigs_for_group([data_dict], opts, images_root, which_features, _device())
    if failed:
        raise _lib.DssError(f"eigensolver did not converge for {image_id}")
    arrays, fields = _eigs_content(which_matrix, evals, evecs)
    output_file.parent.mkdir(parents=True, exist_ok=True)
    torch.save(io_pipeline._materialise(arrays, 0, {}, fields), str(output_file))


def extract_eigs(images_root: str, features_dir: str, output_dir: str, which_matrix: str = "laplacian",
                 which_color_matrix: str = "knn", which_features: str = "k", normalize: bool = True,
                 threshold_at_zero: bool = True, lapnorm: bool = True, K: int = 20,
                 image_downsample_factor: Optional[int] = None, image_color_lambda: float = 0.0,
                 multiprocessing: int = 0, batch_size: int = 128, yes: Optional[bool] = None,
                 num_workers: Optional[int] = None, num_workers_out: int = 4, writer: str = "process"):
    """
    Extracts eigenvalues from features.

    Example:
        python extract.py extract_eigs \
            --images_root "./data/VOC2012/images" \
            --features_dir "./data/VOC2012/features/dino_vits16" \
            --which_matrix "laplacian" \
            --output_dir "./data/VOC2012/eigs/laplacian" \
            --K 5
    """
    opts = _EigOptions(K=K, which_matrix=which_matrix, which_color_matrix=which_color_matrix, normalize=normalize,
                       threshold_at_zero=threshold_at_zero, lapnorm=lapnorm,
                       image_downsample_factor=image_downsample_factor, image_color_lambda=image_color_lambda)
    utils.make_output_dir(output_dir, assume_yes=yes)
    kwargs = dict(K=K, which_matrix=which_matrix, which_features=which_features, which_color_matrix=which_color_matrix,
                  normalize=normalize, threshold_at_zero=threshold_at_zero, images_root=images_root,
                  output_dir=output_dir, image_downsample_factor=image_downsample_factor,
                  image_color_lambda=image_color_lambda, lapnorm=lapnorm)
    print(kwargs)
    if multiprocessing:
        print(f"Note: multiprocessing={multiprocessing} is ignored: images are batched inside the GPU kernels "
              f"({batch_size} per launch) instead of forked CPU workers")
    dev = _device()
    inputs = _my_share(list(enumerate(sorted(Path(features_dir).iterdir()))))
    import time
    start = time.time()
    all_failed: List[str] = []

    with io_pipeline.make_writer(writer, num_workers_out) as wr:
        def flush(key, dds):
            evals, evecs, failed = _eigs_for_group(dds, opts, images_root, which_features, dev)
            all_failed.extend(dds[j]["id"] for j in failed)
            arrays, fields = _eigs_content(which_matrix, evals, evecs)
            wr.submit_batch(arrays, [(str(Path(output_dir) / f"{d['file'][:-4]}.pth"), j, {}, fields)
                                     for j, d in enumerate(dds) if j not in failed])

        batcher = _Batcher(batch_size, flush)
        load = lambda i: torch.load(str(inputs[i][1]), map_location="cpu")   # noqa: E731  (file reads overlap on threads)
        for data_dict in io_pipeline.ImagePrefetcher(load, range(len(inputs)), num_workers):
            image_id = data_dict["file"][:-4]
            if (Path(output_dir) / f"{image_id}.pth").is_file():
                print(f"Skipping existing file {str(Path(output_dir) / (image_id + '.pth'))}")
                continue
            batcher.add((tuple(data_dict[which_features].shape[-2:]), tuple(data_dict["shape"])), data_dict)
        batcher.finish()
    print(f"Finished in {time.time() - start:.1f}s")
    if all_failed:
        raise _lib.DssError(f"eigensolver did not converge for {len(all_failed)} image(s): {all_failed[:8]} -- their files "
                            "were not written (all other outputs were)")


# ---------------------------------------------------------------------------------------------------------------
# Segmentations (SURVEY 8f rank 1): device kernels on batches of eigenvector files
def _png_writer_pool(num_threads: int):
    from concurrent.futures import ThreadPoolExecutor
    return ThreadPoolExecutor(max(1, num_threads), thread_name_prefix="dss-png")


def _save_png(arr_u8: np.ndarray, path: str):
    from PIL import Image
    Image.fromarray(arr_u8, mode="L").save(path)


def _paired_dicts(inputs, output_dir, num_workers):
    """Loads (features, eigs) file pairs on threads, skipping pairs whose PNG exists (extract.py:300-304)."""
    def load(i):
        _, (feature_path, eigs_path) = inputs[i]
        data_dict = torch.load(str(feature_path), map_location="cpu")
        data_dict.update(torch.load(str(eigs_path), map_location="cpu", weights_only=False))
        return data_dict
    for data_dict in io_pipeline.ImagePrefetcher(load, range(len(inputs)), num_workers):
        output_file = str(Path(output_dir) / f"{Path(data_dict['id'])}.png")
        if Path(output_file).is_file():
            print(f"Skipping existing file {str(output_file)}")
            continue
        yield data_dict, output_file


def extract_single_region_segmentations(features_dir: str, eigs_dir: str, output_dir: str, threshold: float = 0.0,
                                        multiprocessing: int = 0, yes: Optional[bool] = None, batch_size: int = 256,
                                        num_workers: Optional[int] = None):
    """
    Thresholds the Fiedler-like eigenvector of every image into a patch-grid mask (reference
    extract/extract.py:364-411), same command / file contract; the threshold runs on the GPU for a batch of images.

    Example:
    python extract.py extract_single_region_segmentations \
        --features_dir "./data/VOC2012/features/dino_vits16" \
        --eigs_dir "./data/VOC2012/eigs/laplacian" \
        --output_dir "./data/VOC2012/single_region_segmentation/patches" \
    """
    utils.make_output_dir(output_dir, assume_yes=yes)
    inputs = _my_share(utils.get_paired_input_files(features_dir, eigs_dir))
    dev = _device()
    with _png_writer_pool(4) as pool:
        def flush(key, items):
            evecs = torch.stack([torch.as_tensor(d["eigenvectors"]) for d, _ in items]).to(dev)
            masks = segment.threshold_masks(evecs, threshold, which=1).cpu().numpy()
            for j, (d, output_file) in enumerate(items):
                _, _, _, _, _, H_patch, W_patch, _, _ = utils.get_image_sizes(d)
                pool.submit(_save_png, masks[j].reshape(H_patch, W_patch).copy(), output_file)

        batcher = _Batcher(batch_size, flush)
        for d, output_file in _paired_dicts(inputs, output_dir, num_workers):
            batcher.add(tuple(torch.as_tensor(d["eigenvectors"]).shape), (d, output_file))
        batcher.finish()


def extract_multi_region_segmentations(features_dir: str, eigs_dir: str, output_dir: str, adaptive: bool = False,
                                       non_adaptive_num_segments: int = 4, infer_bg_index: bool = True,
                                       kmeans_baseline: bool = False, num_eigenvectors: int = 1_000_000,
                                       multiprocessing: int = 0, random_state: Optional[int] = None,
                                       yes: Optional[bool] = None, batch_size: int = 256,
                                       num_workers: Optional[int] = None):
    """
    K-means on the non-constant eigenvectors (or on the raw features, ``kmeans_baseline``) of every image -> label map
    on the patch grid, background label swapped to 0 (reference extract/extract.py:283-376), same command / file
    contract. The clustering is the batched device K-means of csrc/segment.cu (k-means++ / Lloyd with scikit-learn's
    stopping rules); the reference's KMeans is unseeded, so label NUMBERS differ from run to run there and only the
    partition is comparable. ``random_state`` seeds the device generator (default 0: reproducible).

    Example:
    python extract.py extract_multi_region_segmentations \
        --features_dir "./data/VOC2012/features/dino_vits16" \
        --eigs_dir "./data/VOC2012/eigs/laplacian" \
        --output_dir "./data/VOC2012/multi_region_segmentation/fixed" \
    """
    utils.make_output_dir(output_dir, assume_yes=yes)
    inputs = _my_share(utils.get_paired_input_files(features_dir, eigs_dir))
    dev = _device()
    seed = 0 if random_state is None else int(random_state)
    with _png_writer_pool(4) as pool:
        def flush(key, items):
            dicts = [d for d, _ in items]
            ks = [segment.adaptive_num_clusters(torch.as_tensor(d["eigenvalues"]).numpy()) if adaptive
                  else non_adaptive_num_segments for d in dicts]
            _, _, _, _, _, H_patch, W_patch, _, _ = utils.get_image_sizes(dicts[0])
            if kmeans_baseline:
                pts = torch.stack([d["k"].squeeze() for d in dicts]).to(dev)
                n_pts, layout = pts.shape[1], "features"
            else:
                pts = torch.stack([torch.as_tensor(d["eigenvectors"])[1:1 + num_eigenvectors] for d in dicts]).to(dev)
                n_pts, layout = pts.shape[2], "eigenvectors"
            if n_pts == H_patch * W_patch:     # extract.py:328-333
                grid = (H_patch, W_patch)
            elif n_pts == H_patch * W_patch * 4:
                grid = (H_patch * 2, W_patch * 2)
            else:
                raise ValueError(f"{n_pts} labels do not fit a {H_patch} x {W_patch} patch grid")
            labels, _, _ = segment.kmeans_labels(pts, ks, grid, infer_bg_index, layout, seed,
                                                 image_keys=[int(d["indices"]) for d in dicts])
            labels = labels.cpu().numpy()
            for j, (_, output_file) in enumerate(items):
                pool.submit(_save_png, labels[j].reshape(grid).copy(), output_file)

        batcher = _Batcher(batch_size, flush)
        for d, output_file in _paired_dicts(inputs, output_dir, num_workers):
            key = (tuple(torch.as_tensor(d["eigenvectors"]).shape), tuple(d["k"].shape), tuple(d["shape"]))
            batcher.add(key, (d, output_file))
        batcher.finish()


# ---------------------------------------------------------------------------------------------------------------
def extract_bbox_features(images_root: str, bbox_file: str, model_name: str, output_file: str,
                          checkpoint: Optional[str] = None, seed: Optional[int] = None, random_init: bool = False,
                          batch_size: int = 64, precision: str = "fp16"):
    """
    DINO CLS embedding of every bounding-box crop (reference extract/extract.py:500-544), same command / file
    contract: each dict of ``bbox_file`` gains 'features' [n_boxes, d] fp32. ``batch_size`` crops per ViT forward in
    (image, box) order, whatever their sizes (one ragged forward per batch).
    ``precision``: ViT arithmetic, as in extract_features.

    Example:
        python extract.py extract_bbox_features \
            --model_name dino_vits16 \
            --images_root "./data/VOC2012/images" \
            --bbox_file "./data/VOC2012/multi_region_bboxes/fixed/bboxes_e2_d5.pth" \
            --output_file "./data/VOC2012/multi_region_bboxes/fixed/bbox_features_e2_d5.pth" \
    """
    from PIL import Image
    vit_mod.check_precision(precision)
    bbox_list = torch.load(bbox_file, weights_only=False)
    total_num_boxes = sum(len(d["bboxes"]) for d in bbox_list)
    print(f"Loaded bounding box list. There are {total_num_boxes} total bounding boxes.")
    dev = _device()
    model, _, patch_size, _ = utils.get_model(model_name.lower(), checkpoint=checkpoint, seed=seed, device=dev,
                                              random_init=random_init, precision=precision)
    feats: Dict[Tuple[int, int], torch.Tensor] = {}   # (image row, box row) -> [d]

    def flush(items):
        packed, dims = vit_mod.pack_images([it[0] for it in items])
        cls, _ = model.forward_cls_ragged(packed.to(dev), dims)
        cls = cls.cpu()
        for j, (_, where) in enumerate(items):
            feats[where] = cls[j].clone()

    batch_size = max(1, int(batch_size))
    batch = []
    for bi, bbox_dict in enumerate(bbox_list):
        image_filename = str(Path(images_root) / f"{bbox_dict['id']}.jpg")
        image = torch.from_numpy(np.ascontiguousarray(np.asarray(Image.open(image_filename).convert("RGB"))))
        for ji, (xmin, ymin, xmax, ymax) in enumerate(bbox_dict["bboxes_original_resolution"]):
            crop = image[ymin:ymax, xmin:xmax].contiguous()          # image[:, :, ymin:ymax, xmin:xmax] at :539
            if crop.shape[0] < patch_size or crop.shape[1] < patch_size:
                raise ValueError(f"{bbox_dict['id']}: box {(xmin, ymin, xmax, ymax)} is smaller than one patch")
            batch.append((crop, (bi, ji)))
            if len(batch) == batch_size:
                flush(batch)
                batch = []
    if batch:
        flush(batch)
    for bi, bbox_dict in enumerate(bbox_list):
        bbox_dict["features"] = torch.stack([feats[(bi, ji)] for ji in range(len(bbox_dict["bboxes"]))], dim=0)
    torch.save(bbox_list, output_file)
    print(f"Saved features to {output_file}")


def _read_label_map(path) -> np.ndarray:
    """np.array(Image.open(path)) as uint8 (a mode '1' PNG reads as bool)."""
    from PIL import Image
    segmap = np.array(Image.open(str(path)))
    if segmap.dtype == bool:
        segmap = segmap.astype(np.uint8)
    if segmap.dtype != np.uint8 or segmap.ndim != 2:
        raise ValueError(f"{path}: expected a single-channel 8-bit label map, got {segmap.dtype} {segmap.shape}")
    return segmap


def _bbox_dict(image_id, P: int, boxes: np.ndarray, present: np.ndarray, skip_bg_index: bool) -> dict:
    """The dict _extract_bbox returns (extract.py:447-468): python int segment indices, numpy int64 coordinates."""
    out = {"bboxes": [], "bboxes_original_resolution": [], "segment_indices": [], "id": image_id,
           "format": "(xmin, ymin, xmax, ymax)"}
    for v in np.flatnonzero(present).tolist():
        if skip_bg_index and v == 0:
            continue
        bbox = [np.int64(c) for c in boxes[v]]
        out["segment_indices"].append(v)
        out["bboxes"].append(bbox)
        out["bboxes_original_resolution"].append([c * P for c in bbox])
    return out


def extract_bboxes(features_dir: str, segmentations_dir: str, output_file: str, num_erode: int = 2, num_dilate: int = 3,
                   skip_bg_index: bool = True, downsample_factor: Optional[int] = None, batch_size: int = 1024,
                   num_workers: Optional[int] = None):
    """
    Bounding box of every segment of the multi-region segmentations after erosion and dilation (reference
    extract/extract.py:429-497), same command / file contract: one list of dicts {'bboxes', 'bboxes_original_resolution',
    'segment_indices', 'id', 'format'} saved to ``output_file``. The morphology and the boxes run on the GPU for batches
    of label maps of equal size (csrc/cluster.cu); files are read on threads.

    Example:
    python extract.py extract_bboxes \
        --features_dir "./data/VOC2012/features/dino_vits16" \
        --segmentations_dir "./data/VOC2012/multi_region_segmentation/fixed" \
        --num_erode 2 --num_dilate 5 \
        --output_file "./data/VOC2012/multi_region_bboxes/fixed/bboxes_e2_d5.pth" \
    """
    utils.make_output_dir(str(Path(output_file).parent), check_if_empty=False)
    inputs = utils.get_paired_input_files(features_dir, segmentations_dir)
    dev = _device()
    outputs: List[Optional[dict]] = [None] * len(inputs)

    def load(i):
        _, (feature_path, segmentation_path) = inputs[i]
        data_dict = torch.load(str(feature_path), map_location="cpu")
        P = utils.get_image_sizes(data_dict, downsample_factor)[4]
        return i, data_dict["id"], P, _read_label_map(segmentation_path)

    def flush(key, items):
        maps = torch.from_numpy(np.stack([it[3] for it in items])).to(dev)
        boxes, present = cluster.segment_bboxes(maps, num_erode, num_dilate)
        boxes, present = boxes.cpu().numpy(), present.cpu().numpy()
        for j, (i, image_id, P, _) in enumerate(items):
            outputs[i] = _bbox_dict(image_id, P, boxes[j], present[j], skip_bg_index)

    batcher = _Batcher(batch_size, flush)
    for item in io_pipeline.ImagePrefetcher(load, range(len(inputs)), num_workers):
        batcher.add(item[3].shape, item)
    batcher.finish()
    torch.save(outputs, output_file)
    print("Done")


def extract_bbox_clusters(bbox_features_file: str, output_file: str, num_clusters: int = 20, seed: int = 0,
                          pca_dim: Optional[int] = 0, max_iter: int = 300, tol: float = 1e-4):
    """
    Clusters the CLS features of all boxes (reference extract/extract.py:547-599), same command / file contract: every
    dict loses 'features' and gains 'clusters' (numpy int32, its slice of the labels). Runs on the GPU: row L2
    normalisation, PCA by the covariance-eigh route (as scikit-learn's PCA does when there are many more rows than
    columns), and K-means over the whole data set.

    Deliberate deviations, both on the device's side of an ill-defined comparison:
      - The reference runs MiniBatchKMeans(batch_size=4096, max_iter=5000, random_state=seed), a stochastic
        approximation of the K-means objective whose label numbers are not reproducible across its own seeds. This
        runs full-batch K-means (k-means++ seeding, Lloyd iterations, scikit-learn KMeans' stopping rules ``max_iter``
        and ``tol``) seeded by ``seed``: the same objective, reproducible to the bit. Cluster ids compare up to
        relabelling, which is what the Hungarian-matched evaluation uses.
      - An all-zero feature row normalises to zeros here; the reference divides by its zero norm and gets NaN.

    Example:
        python extract.py extract_bbox_clusters \
            --bbox_features_file "./data/VOC2012/multi_region_bboxes/fixed/bbox_features_e2_d5.pth" \
            --pca_dim 32 --num_clusters 21 --seed 0 \
            --output_file "./data/VOC2012/multi_region_bboxes/fixed/bbox_clusters_e2_d5_pca_32.pth" \
    """
    bbox_list = torch.load(bbox_features_file, weights_only=False)
    total_num_boxes = sum(len(d["bboxes"]) for d in bbox_list)
    print(f"Loaded bounding box list. There are {total_num_boxes} total bounding boxes with features.")
    dev = _device()
    print("Stacking and normalizing features")
    feats = torch.cat([torch.as_tensor(d["features"]).to(torch.float32).reshape(-1, d["features"].shape[-1])
                       for d in bbox_list], dim=0)
    feats = spectral.normalize_rows(feats.to(dev))
    if pca_dim:
        print(f"Computing PCA with dimension {pca_dim}")
        feats = cluster.pca(feats, int(pca_dim))
    print(f"Computing K-Means clustering with {num_clusters} clusters")
    labels, _, info, _ = cluster.kmeans(feats, int(num_clusters), seed=seed, max_iter=max_iter, tol=tol)
    clusters = labels.cpu().numpy()
    _indices, _counts = np.unique(clusters, return_counts=True)
    print(f"Cluster indices: {_indices.tolist()}")
    print(f"Cluster counts: {_counts.tolist()}")
    idx = 0
    for bbox_dict in bbox_list:
        num_bboxes = len(bbox_dict["bboxes"])
        del bbox_dict["features"]
        bbox_dict["clusters"] = clusters[idx: idx + num_bboxes]
        idx = idx + num_bboxes
    torch.save(bbox_list, output_file)
    print(f"Saved features to {output_file}")


def semantic_map(segmap: np.ndarray, segment_indices, clusters) -> np.ndarray:
    """extract.py:630-642 on one label map: a {0, 255} map becomes {0, 1}; each segment index maps to its cluster and 0
    to 0 (so cluster 0 shares the background's value, as in the reference). The reference drops into pdb on a length
    mismatch, asserts that 0 is not a segment index and raises KeyError on a label without an entry: ValueError here."""
    segmap = np.array(segmap, dtype=np.uint8)
    if set(np.unique(segmap).tolist()).issubset({0, 255}):
        segmap[segmap == 255] = 1
    clusters = np.asarray(clusters).reshape(-1).tolist()
    if len(segment_indices) != len(clusters):
        raise ValueError(f"{len(segment_indices)} segment indices but {len(clusters)} clusters")
    lut = np.zeros(256, dtype=np.int64)
    known = np.zeros(256, dtype=bool)
    for s, c in zip(segment_indices, clusters):
        if int(s) == 0:
            raise ValueError("segment index 0 is the background and cannot carry a cluster")
        lut[int(s)], known[int(s)] = c, True
    known[0] = True
    missing = sorted(set(np.unique(segmap).tolist()) - set(np.flatnonzero(known).tolist()))
    if missing:
        raise ValueError(f"labels {missing} of the segmentation have no cluster")
    return lut[segmap].astype(np.uint8)


def extract_semantic_segmentations(segmentations_dir: str, bbox_clusters_file: str, output_dir: str,
                                   yes: Optional[bool] = None, num_workers: int = 4):
    """
    Pseudo-label maps: every segment of the multi-region segmentation takes the cluster of its box (reference
    extract/extract.py:602-647), same command / file contract ({output_dir}/{id}.png, 8-bit 'L'). A 256-entry lookup
    per image: PNG decode and encode dominate, so it runs on the host on the PNG writer threads.

    Example:
        python extract.py extract_semantic_segmentations \
            --segmentations_dir "./data/VOC2012/multi_region_segmentation/fixed" \
            --bbox_clusters_file "./data/VOC2012/multi_region_bboxes/fixed/bbox_clusters_e2_d5_pca_32.pth" \
            --output_dir "./data/VOC2012/semantic_segmentations/patches/fixed/segmaps_e2_d5_pca_32" \
    """
    bbox_list = torch.load(bbox_clusters_file, weights_only=False)
    total_num_boxes = sum(len(d["bboxes"]) for d in bbox_list)
    print(f"Loaded bounding box list. There are {total_num_boxes} total bounding boxes with features and clusters.")
    utils.make_output_dir(output_dir, assume_yes=yes)

    def one(bbox_dict):
        image_id = bbox_dict["id"]
        segmap = _read_label_map(Path(segmentations_dir) / f"{image_id}.png")
        try:
            out = semantic_map(segmap, bbox_dict["segment_indices"], bbox_dict["clusters"])
        except ValueError as e:
            raise ValueError(f"{image_id}: {e}") from None
        _save_png(out, str(Path(output_dir) / f"{image_id}.png"))

    with _png_writer_pool(num_workers) as pool:
        for f in [pool.submit(one, d) for d in bbox_list]:
            f.result()
    print(f"Saved features to {output_dir}")


def extract_crf_segmentations(images_list: str, images_root: str, segmentations_dir: str, output_dir: str,
                              num_classes: int = 21, downsample_factor: int = 16, multiprocessing: int = 0,
                              w1=10, alpha=80, beta=13, w2=3, gamma=3, it=5.0, unary_eps: float = 1e-5,
                              yes: Optional[bool] = None, batch_size: int = 16, num_workers: Optional[int] = None):
    """
    Refines patch-resolution segmentations to pixel resolution with a dense CRF (reference extract/extract.py:650-735),
    same command / file contract: {output_dir}/{id}.png, 8-bit 'L', the size of {images_root}/{id}.jpg; existing outputs
    are skipped. The reference calls SimpleCRF on the CPU; here mean field runs on the GPU on permutohedral lattices
    (csrc/crf.cu) for ragged batches of ``batch_size`` images of any sizes. Images (PIL, as the reference) and label maps
    are read on threads, PNGs written on threads. ``multiprocessing`` is accepted and unused.

    Parameters as the reference: w1 / alpha / beta the bilateral weight and its spatial / colour standard deviations,
    w2 / gamma the spatial kernel, ``it`` mean-field iterations (cast with int()). ``unary_eps`` clips the one-hot
    probabilities before the log (densecrf's unary_from_softmax default); at 0 every other label would cost +inf and
    the CRF would return its input. The device workspace is about 2.5 KB per pixel at 21 classes (a batch of 16 VOC
    images: 7.5 GB).

    Example:
        python extract.py extract_crf_segmentations \
            --images_list "./data/VOC2012/lists/images.txt" \
            --images_root "./data/VOC2012/images" \
            --segmentations_dir "./data/VOC2012/semantic_segmentations/patches/fixed/segmaps_e2_d5_pca_32" \
            --output_dir "./data/VOC2012/semantic_segmentations/crf/fixed/segmaps_e2_d5_pca_32" \
    """
    from PIL import Image
    from . import crf
    utils.make_output_dir(output_dir, assume_yes=yes)
    inputs = _my_share(utils.get_paired_input_files(images_list, segmentations_dir))
    print(f"Found {len(inputs)} images and segmaps")
    dev = _device()
    P, num_classes = int(downsample_factor), int(num_classes)
    todo = []
    for _, (image_file, segmap_path) in inputs:
        image_id = Path(image_file).stem
        output_file = str(Path(output_dir) / f"{image_id}.png")
        if Path(output_file).is_file():
            print(f"Skipping existing file {output_file}")
            continue
        todo.append((image_id, segmap_path, output_file))

    def load(i):
        image_id, segmap_path, output_file = todo[i]
        image = np.array(Image.open(str(Path(images_root) / f"{image_id}.jpg")).convert("RGB"))
        segmap = crf.prepare_segmap(_read_label_map(segmap_path), image.shape[0], image.shape[1], P, num_classes,
                                    str(segmap_path))
        return image, segmap, output_file

    with _png_writer_pool(4) as pool:
        futures, batch = [], []

        def flush():
            labels, _, _ = crf.dense_crf([b[0] for b in batch], [b[1] for b in batch], num_classes, P, w1=w1,
                                         alpha=alpha, beta=beta, w2=w2, gamma=gamma, it=int(it), unary_eps=unary_eps,
                                         device=dev)
            host = torch.cat([lab.reshape(-1) for lab in labels]).cpu().numpy()
            o = 0
            for lab, (_, _, output_file) in zip(labels, batch):
                h, w = lab.shape
                futures.append(pool.submit(_save_png, host[o:o + h * w].reshape(h, w), output_file))
                o += h * w
            batch.clear()

        for item in io_pipeline.ImagePrefetcher(load, range(len(todo)), num_workers):
            batch.append(item)
            if len(batch) >= max(1, int(batch_size)):
                flush()
        if batch:
            flush()
        for f in futures:
            f.result()
    print(f"Saved CRF segmentations to {output_dir}")


# ---------------------------------------------------------------------------------------------------------------
def _extract_all_options(model_name, opts: _EigOptions, single_region: bool, multi_region: bool):
    """extract_all's own refusals, before any device work. The segmentation commands read eigenvectors on the patch grid
    (single region), or on it and the grid twice as fine (multi region); other grids are refused."""
    patch_size = vit_mod.arch(model_name)[0]
    factor = opts.factor(patch_size)
    if single_region and factor != patch_size:
        raise ValueError(f"single_region_dir: with image_downsample_factor={factor} the eigenvectors have "
                         f"(H // {factor}) x (W // {factor}) entries, which the single-region segmentation cannot "
                         f"reshape to the {patch_size}-pixel patch grid")
    if multi_region and 2 * factor != patch_size and factor != patch_size:
        raise ValueError(f"multi_region_dir: with image_downsample_factor={factor} the eigenvectors have "
                         f"(H // {factor}) x (W // {factor}) entries; the multi-region segmentation labels only the "
                         f"{patch_size}-pixel patch grid or the grid twice as fine (factor {patch_size // 2})")


def extract_all(images_list: str, images_root: Optional[str], model_name: str, features_dir: Optional[str],
                eigs_dir: str, K: int = 20, batch_size: int = 64, which_block: int = -1, normalize: bool = True,
                threshold_at_zero: bool = True, lapnorm: bool = True, image_color_lambda: float = 0.0,
                which_color_matrix: str = "knn", checkpoint: Optional[str] = None, seed: Optional[int] = None,
                random_init: bool = False, yes: Optional[bool] = None, single_region_dir: Optional[str] = None,
                multi_region_dir: Optional[str] = None, non_adaptive_num_segments: int = 4, adaptive: bool = False,
                infer_bg_index: bool = True, threshold: float = 0.0, num_workers: Optional[int] = None,
                num_workers_out: int = 4, writer: str = "process", precision: str = "fp16",
                which_matrix: str = "laplacian", image_downsample_factor: Optional[int] = None):
    """Fused extract_features + extract_eigs (+ the two segmentation commands): features and eigenvectors never leave
    the GPU between the stages. Writes the eigs files and, if the directories are given, the features files and the
    single- / multi-region segmentation PNGs, all in the reference's layouts. Decoding, pinned staging and the file
    writers run on threads (io_pipeline.py). ``precision``: ViT arithmetic, as in extract_features.

    ``which_matrix``, ``image_downsample_factor``, ``image_color_lambda`` and ``which_color_matrix`` are extract_eigs'
    options with its defaults, and every file equals what extract_features followed by extract_eigs writes. The colour
    image is the decoded image already on the device, resized by Pillow's bilinear rule on the GPU (resize.py), so no
    file is read twice; files that are not 3-channel RGB images are refused by name in colour mode. With a Laplacian
    grid other than the patch grid (image_downsample_factor other than the patch size), ``single_region_dir`` is
    refused, as extract_single_region_segmentations cannot reshape such eigenvectors; ``multi_region_dir`` is accepted
    only at half the patch size, whose 2x finer grid extract_multi_region_segmentations also labels."""
    vit_mod.check_precision(precision)
    model_name = model_name.lower()
    opts = _EigOptions(K=K, which_matrix=which_matrix, which_color_matrix=which_color_matrix, normalize=normalize,
                       threshold_at_zero=threshold_at_zero, lapnorm=lapnorm,
                       image_downsample_factor=image_downsample_factor, image_color_lambda=image_color_lambda)
    _extract_all_options(model_name, opts, bool(single_region_dir), bool(multi_region_dir))
    for dname in (features_dir, eigs_dir, single_region_dir, multi_region_dir):
        if dname:
            utils.make_output_dir(dname, assume_yes=yes)
    wr = io_pipeline.make_writer(writer, num_workers_out)   # first: writer processes import torch while the model is set up
    dev = _device()
    model, _, patch_size, _ = utils.get_model(model_name, checkpoint=checkpoint, seed=seed, device=dev,
                                              random_init=random_init, precision=precision)
    filenames = Path(images_list).read_text().splitlines()
    dataset = utils.ImagesDataset(filenames=filenames, images_root=images_root)
    all_failed: List[str] = []
    decode_threads: dict = {}
    import time
    t_start = time.perf_counter()   # model set-up (weights, packing) is done: what follows is the per-image pipeline

    tm = {"decode_wait": 0.0, "pinned_alloc": 0.0, "launch": 0.0, "wait_gpu": 0.0, "submit": 0.0}
    in_flight: List[dict] = []       # batches whose kernels / read-back copies are still running (software pipeline)
    with wr, _png_writer_pool(2) as png_pool:
        def finish(h):
            """Second half of a batch: wait for its read-back, retry stragglers, hand everything to the writers."""
            ta = time.perf_counter()
            h["event"].synchronize()
            assembler.release(h["batch"])     # its host->device copy is long done: the decode threads may refill it
            tb = time.perf_counter()
            items, H, W, Hp, Wp, grid = h["items"], h["H"], h["W"], h["Hp"], h["Wp"], h["grid"]
            evals, evecs, info = h["evals"], h["evecs"], h["info"]
            # rare: the largest Krylov space that fits for the images that did not reach the tolerance
            failed = _retry_bad_rows(h["solve"], evals, evecs, info, grid[0] * grid[1])
            failed_files = [items[j][1] for j in failed]
            all_failed.extend(failed_files)
            _warn_eigs(which_matrix, info, failed_files)
            if features_dir:
                k = h["k"].numpy()
                N = k.shape[1]
                wr.submit_batch({"k": k.reshape(-1, k.shape[2])}, [it_ for j, it_ in enumerate(_feature_files(
                    features_dir, [(file, index, H, W) for _, file, index in items],
                    [(j * N, (j + 1) * N) for j in range(len(items))], model_name, patch_size)) if j not in failed])
            arrays, fields = _eigs_content(which_matrix, evals, evecs)
            wr.submit_batch(arrays, [(str(Path(eigs_dir) / f"{file[:-4]}.pth"), j, {}, fields)
                                     for j, (_, file, _) in enumerate(items) if j not in failed])
            for j, (_, file, index) in enumerate(items):
                if j in failed:
                    continue
                if h["masks"] is not None:
                    png_pool.submit(_save_png, h["masks"][j].numpy().reshape(Hp, Wp).copy(),
                                    str(Path(single_region_dir) / f"{Path(file).stem}.png"))
                if h["labels"] is not None:
                    png_pool.submit(_save_png, h["labels"][j].numpy().reshape(grid).copy(),
                                    str(Path(multi_region_dir) / f"{Path(file).stem}.png"))
            tm["wait_gpu"] += tb - ta
            tm["submit"] += time.perf_counter() - tb

        def flush(batch):
            """First half of a batch: start the H2D copy of the page-locked batch the decode threads filled, enqueue every
            kernel and the read-back copies; then finish the PREVIOUS batch while this one runs."""
            H, W = batch.key
            tb = time.perf_counter()
            items = [(None, file, index) for file, index in batch.items]
            host = batch.host[:len(items)]
            images_d = host.to(dev, non_blocking=True)
            k = model.forward_k(images_d, which_block=which_block)
            Hp, Wp = H // patch_size, W // patch_size
            # the colour images: the decoded batch already on the device, resized by Pillow's bilinear rule (resize.py)
            solve, (H_lr, W_lr) = _eigen_stage(
                k, (Hp, Wp), patch_size, opts,
                lambda h, w: resize.resize(images_d, h, w, "u8" if which_color_matrix == "rw" else "f32"))
            evals_d, evecs_d, info_d = solve(None, 0)
            masks_d = labels_d = None
            if single_region_dir:
                masks_d = segment.threshold_masks(evecs_d, threshold, which=1)
            if multi_region_dir:
                if adaptive:   # the per-image cluster count comes from the eigenvalues (host arithmetic on K numbers)
                    saved, _ = _eigs_content(which_matrix, evals_d.cpu())   # what the eigs file holds
                    ks = [segment.adaptive_num_clusters(e) for e in saved["evals"]]
                else:
                    ks = [non_adaptive_num_segments] * len(items)
                labels_d = segment.kmeans_labels(evecs_d[:, 1:], ks, (H_lr, W_lr), infer_bg_index,
                                                 image_keys=[it[2] for it in items])[0]

            def to_host(t):
                if t is None:
                    return None
                h_ = torch.empty(t.shape, dtype=t.dtype, pin_memory=True)
                h_.copy_(t, non_blocking=True)
                return h_
            h = {"items": items, "H": H, "W": W, "Hp": Hp, "Wp": Wp, "grid": (H_lr, W_lr), "solve": solve, "evals": to_host(evals_d),
                 "evecs": to_host(evecs_d), "info": to_host(info_d), "masks": to_host(masks_d), "labels": to_host(labels_d),
                 "k": to_host(k) if features_dir else None, "keep": (k, evals_d, evecs_d, info_d, masks_d, labels_d),
                 "batch": batch}
            ev = torch.cuda.Event()
            ev.record(torch.cuda.current_stream(dev))
            h["event"] = ev
            tm["launch"] += time.perf_counter() - tb
            in_flight.append(h)
            while len(in_flight) > 1:
                finish(in_flight.pop(0))

        todo = []
        for i in _my_share(list(range(len(dataset)))):
            file = dataset.filenames[i]
            if (Path(eigs_dir) / f"{file[:-4]}.pth").is_file():
                print(f"Skipping existing file {str(Path(eigs_dir) / (file[:-4] + '.pth'))}")
            else:
                todo.append(i)
        # The decode threads group the images by shape and write them straight into page-locked batches
        # (io_pipeline.BatchAssembler); this thread only sees completed batches.
        if dataset.transform is None:
            load = dataset.load_raw_rgb_file if opts.colour else dataset.load_raw
        else:
            def load(i):
                image, file, index = dataset[i]
                return image.numpy(), False, file, index
        assembler = io_pipeline.BatchAssembler(load, todo, max(1, int(batch_size)), num_workers)
        it = iter(assembler)
        while True:
            ta = time.perf_counter()
            batch = next(it, None)
            tm["decode_wait"] += time.perf_counter() - ta
            if batch is None:
                break
            flush(batch)
        tm["pinned_alloc"] = assembler.alloc_seconds
        decode_threads = {k_: round(v_, 3) for k_, v_ in assembler.worker_seconds.items()}
        decode_threads["threads"] = len(assembler.threads)
        if assembler.trace is not None:
            decode_threads["trace"] = [(round(t_ - t_start, 4), ev_, d_) for t_, ev_, d_ in sorted(assembler.trace)]
        while in_flight:
            finish(in_flight.pop(0))
    seconds = time.perf_counter() - t_start
    print(f"Saved eigs to {eigs_dir} ({len(todo)} images in {seconds:.2f}s after model set-up: "
          f"{len(todo) / max(seconds, 1e-9):.0f} images/s incl. decode and file writes; main thread: "
          + ", ".join(f"{k_} {v_:.2f}s" for k_, v_ in tm.items()) + ")")
    if all_failed:
        raise _lib.DssError(f"eigensolver did not converge for {len(all_failed)} image(s): {all_failed[:8]}")
    return {"images": len(todo), "seconds": seconds, "images_per_s": len(todo) / max(seconds, 1e-9),
            "decode_thread_seconds_summed": decode_threads,
            "main_thread_seconds": {"waiting_for_decoders": tm["decode_wait"],
                                    "pinned_alloc_in_decoders": tm["pinned_alloc"], "kernel_launches": tm["launch"],
                                    "waiting_for_gpu": tm["wait_gpu"], "writer_submit": tm["submit"], "total": seconds}}
