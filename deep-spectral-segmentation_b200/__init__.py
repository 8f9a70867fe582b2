"""deep-spectral-segmentation_b200: H100-native implementation of the deep-spectral hot path
(extract_features -> extract_eigs of lukemelas/deep-spectral-segmentation, extract/extract.py:21-280).

All device work is hand-written sm_90a CUDA reached through the C-ABI library ``libdss_b200.so``
(include/dss_b200.h); this package is the thin Python host side that mirrors the reference's callables.
The directory name contains a hyphen, so import it with
``importlib.import_module("deep-spectral-segmentation_b200")`` (tests/conftest.py does this as ``dss``).
"""
__version__ = "0.1.0"
