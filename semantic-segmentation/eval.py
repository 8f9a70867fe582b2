#!/usr/bin/env python
"""Drop-in command line for the semantic-segmentation evaluation (the reference's semantic-segmentation/eval.py), with
the counts on the GPU. Hydra-style overrides of the keys the reference reads:

    python semantic-segmentation/eval.py segments_dir=<dir>/semantic_segmentations/patches/laplacian_dino_vits16/crf \
        data.val_kwargs.root=<VOC root> [data.num_classes=20] [n_clusters=27]

Single process, one GPU. See DESIGN.md section 5 for the differences from the reference.
"""
import importlib
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
_segeval = importlib.import_module("deep-spectral-segmentation_b200.segeval")

if __name__ == "__main__":
    _segeval.semantic_main(sys.argv[1:])
