#!/usr/bin/env python
"""Drop-in command line for the object-segmentation evaluation (the reference's object-segmentation/main.py), with the
counts on the GPU. Hydra-style overrides:

    python object-segmentation/main.py data_root=<dir> predictions.root=<dir> predictions.run=<run> \
        [predictions.downsample=16|null] [predictions.CUB=<dir>] [datasets=CUB,ECSSD]

Single process, one GPU. See DESIGN.md section 5 for the differences from the reference.
"""
import importlib
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
_segeval = importlib.import_module("deep-spectral-segmentation_b200.segeval")

if __name__ == "__main__":
    _segeval.object_main(sys.argv[1:])
