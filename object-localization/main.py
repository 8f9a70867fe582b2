#!/usr/bin/env python
"""Drop-in command line for object localization (same flags and output files as the reference's
object-localization/main.py), on the GPU:

    python object-localization/main.py --eigenseg --precomputed_eigs_dir <dir>/laplacian_... --dataset VOC07 --set trainval
    python object-localization/main.py --arch vit_small --patch_size 16 --which_features k          # LOST
    python object-localization/main.py --dinoseg --dinoseg_head 4                                   # DINO-seg

Single process, one GPU. See DESIGN.md section 5 for the differences from the reference.
"""
import importlib
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
_localize = importlib.import_module("deep-spectral-segmentation_b200.localize")

if __name__ == "__main__":
    _localize.main(sys.argv[1:])
