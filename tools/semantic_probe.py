"""Times the semantic-segmentation stages on the GPU (CUDA events, warmed up) next to the reference's host path.

    python tools/semantic_probe.py [--out DIR]

  extract_bbox_clusters : M = 160k box features, d = 384, pca_dim = 32, k = 21 -- device normalise + PCA + K-means,
                          against scikit-learn PCA + MiniBatchKMeans(batch_size=4096, max_iter=5000) on the host cores
  extract_bboxes        : 10k synthetic 30 x 30 label maps, num_erode 2, num_dilate 3 (kernel only)
Prints one JSON line with the card name and power limit; --out also writes it to DIR/semantic_probe.json."""
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import importlib  # noqa: E402

cluster = importlib.import_module("deep-spectral-segmentation_b200.cluster")
spectral = importlib.import_module("deep-spectral-segmentation_b200.spectral")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    torch.set_grad_enabled(False)
    dev = torch.device("cuda:0")
    g = np.random.default_rng(0)
    M, d, p, k = 160_000, 384, 32, 21
    centres = g.normal(size=(k, d)).astype(np.float32)
    X = (centres[g.integers(0, k, size=M)] + 1.5 * g.normal(size=(M, d))).astype(np.float32)
    Xd = torch.from_numpy(X).to(dev)
    out = {"card": card()}

    def clusters():
        f = spectral.normalize_rows(Xd)
        f = cluster.pca(f, p)
        return cluster.kmeans(f, k, seed=0)

    res = clusters()
    out["clusters_device_ms"] = timed(clusters, 3)
    out["kmeans_iterations"] = int(res[2][0])
    out["kmeans_converged"] = int(res[2][1])

    from sklearn.cluster import MiniBatchKMeans
    from sklearn.decomposition import PCA
    t0 = time.perf_counter()
    Xn = X / np.linalg.norm(X, axis=-1, keepdims=True)
    Y = PCA(p).fit_transform(Xn)
    MiniBatchKMeans(n_clusters=k, batch_size=4096, max_iter=5000, random_state=0).fit_predict(Y)
    out["clusters_host_sklearn_ms"] = (time.perf_counter() - t0) * 1e3

    maps = torch.from_numpy(g.integers(0, 6, size=(10_000, 30, 30)).astype(np.uint8))
    maps = torch.nn.functional.max_pool2d(maps.float()[:, None], 5, 1, 2)[:, 0].to(torch.uint8).to(dev)   # blobs
    out["bboxes_10k_30x30_ms"] = timed(lambda: cluster.segment_bboxes(maps, 2, 3), 5)
    line = json.dumps(out)
    print(line)
    if "--out" in sys.argv:
        o = Path(sys.argv[sys.argv.index("--out") + 1])
        o.mkdir(parents=True, exist_ok=True)
        (o / "semantic_probe.json").write_text(line + "\n")


if __name__ == "__main__":
    main()
