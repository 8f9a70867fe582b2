import importlib
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100: run with -m gpu)")
    # the CPU oracles (fp64 eigh, fp32 ViT) run on torch's intra-op pool: size it by the CPUs this container may use
    # (a host may show many more hardware threads than the container's CPU quota; spinning threads get it throttled)
    try:
        import torch
        n = importlib.import_module("deep-spectral-segmentation_b200.io_pipeline").available_cpus()
        if torch.get_num_threads() > n:
            torch.set_num_threads(n)
    except Exception:  # noqa: BLE001  (never let a sizing hint break test collection)
        pass


@pytest.fixture(scope="session")
def dss():
    """The product package (its directory name has a hyphen, so it is imported by string)."""
    return importlib.import_module("deep-spectral-segmentation_b200")


def load_pkg(sub: str = ""):
    name = "deep-spectral-segmentation_b200" + (("." + sub) if sub else "")
    return importlib.import_module(name)


@pytest.fixture(scope="session")
def cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.set_grad_enabled(False)
    # the fp32 oracle runs on the GPU in several tests: keep it true fp32 (no TF32 in matmuls / cuDNN convolutions)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    return torch.device("cuda:0")
