#!/usr/bin/env python
"""Drop-in command line for the deep-spectral hot path (same commands and flags as the reference's extract/extract.py):

    python extract.py extract_features --images_list ... --images_root ... --output_dir ... --model_name dino_vits16 --batch_size 1
    python extract.py extract_eigs --images_root ... --features_dir ... --which_matrix laplacian --output_dir ... --K 5
    python extract.py extract_all --images_list ... --images_root ... --model_name dino_vits16 --eigs_dir ... --K 5

Multi-GPU: launch the same command under torchrun (one process per GPU); every rank takes a strided share of the sorted
work list and writes its own files, nothing is exchanged:

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 extract.py extract_all ...
"""
import importlib
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
_pkg = "deep-spectral-segmentation_b200"
_extract = importlib.import_module(_pkg + ".extract")
_cli = importlib.import_module(_pkg + ".cli")

if __name__ == "__main__":
    _cli.Fire(dict(
        extract_features=_extract.extract_features,
        extract_eigs=_extract.extract_eigs,
        extract_single_region_segmentations=_extract.extract_single_region_segmentations,
        extract_multi_region_segmentations=_extract.extract_multi_region_segmentations,
        extract_bboxes=_extract.extract_bboxes,
        extract_bbox_features=_extract.extract_bbox_features,
        extract_bbox_clusters=_extract.extract_bbox_clusters,
        extract_semantic_segmentations=_extract.extract_semantic_segmentations,
        extract_all=_extract.extract_all,
    ))
