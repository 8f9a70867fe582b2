"""-m gpu: affinity + eigensolver of libdss_b200 against the oracle (oracle/eigs_ref.py = the reference's scipy
path) and a float64 dense ground truth, on identical fp32 features.

Tolerance (BASELINE.json north_star): eigenvectors within 1e-4 relative L2 after sign alignment. The reference's
own float32 ARPACK path is only accurate to ~3e-6..2e-4 against float64 on these inputs (see tools/lanczos_proto.py),
so the CUDA result is held to 1e-4 against the float64 truth always, and to max(1e-4, 2x the oracle's own error)
against the oracle."""
import numpy as np
import pytest
import torch

from conftest import load_pkg

pytestmark = pytest.mark.gpu


def _rel_err(a, b, D=None):
    """per-vector sign-aligned relative L2 error of a against b, both (K, N) numpy"""
    out = []
    for k in range(a.shape[0]):
        w = b[k] * D if D is not None else b[k]
        s = np.sign(np.dot(a[k], w)) or 1.0
        out.append(np.linalg.norm(a[k] - s * b[k]) / np.linalg.norm(b[k]))
    return np.array(out)


def _check_case(cuda, feats, K, normalize=True, lapnorm=True, threshold=True):
    from oracle import eigs_ref
    spectral = load_pkg("spectral")
    f = feats[None].to(cuda)
    evals, evecs, info, resid = spectral.laplacian_eigs(f, K, normalize, threshold, lapnorm)
    torch.cuda.synchronize()
    ev, vec = evals[0].cpu().numpy(), evecs[0].cpu().numpy()
    n_steps, conv = int(info[0, 0]), int(info[0, 1])
    ev_o, vec_o = eigs_ref.extract_eig(feats, K, normalize=normalize, lapnorm=lapnorm, threshold_at_zero=threshold,
                                       rng_seed=0)
    ev_o, vec_o = ev_o.numpy(), vec_o.numpy()
    ev64, vec64 = eigs_ref.eigh_f64(feats, K, normalize=normalize, lapnorm=lapnorm, threshold_at_zero=threshold)
    e_truth = _rel_err(vec, vec64)
    e_oracle = _rel_err(vec, vec_o)
    e_oracle_truth = _rel_err(vec_o, vec64)
    print(f"N={feats.shape[0]} K={K} lapnorm={lapnorm}: steps={n_steps} conv={conv} "
          f"cuda-vs-f64 {e_truth.max():.2e}  cuda-vs-oracle {e_oracle.max():.2e}  oracle-vs-f64 {e_oracle_truth.max():.2e} "
          f"|dlam| {np.abs(ev - ev_o).max():.2e}")
    assert conv == 1
    assert np.all(np.isfinite(vec)) and np.all(np.isfinite(ev))
    assert np.all(np.diff(ev) >= -1e-6), ev                      # ascending
    assert np.abs(ev - ev64).max() <= 1e-5 * max(1.0, np.abs(ev64).max())
    assert np.abs(ev - ev_o).max() <= 2e-5 * max(1.0, np.abs(ev64).max())
    assert e_truth.max() <= 1e-4, e_truth
    assert np.all(e_oracle <= np.maximum(1e-4, 2 * e_oracle_truth + 1e-6)), (e_oracle, e_oracle_truth)
    # sign rule (extract.py:237-240): at most half of the entries positive unless all are
    for k in range(K):
        m = float((vec[k] > 0).mean())
        assert not (0.5 < m < 1.0), (k, m)
    return ev, vec


@pytest.mark.parametrize("N,d,seed", [(196, 384, 0), (900, 384, 0), (900, 384, 1), (713, 384, 2), (400, 768, 3)])
def test_laplacian_eigs_structured(cuda, N, d, seed):
    synth = load_pkg("synth")
    _check_case(cuda, synth.structured_features(N, d, 6, seed), K=5)


def test_laplacian_eigs_K15(cuda):
    synth = load_pkg("synth")
    _check_case(cuda, synth.structured_features(900, 384, 6, 3), K=15)


def test_laplacian_eigs_unnormalised_laplacian(cuda):
    synth = load_pkg("synth")
    _check_case(cuda, synth.structured_features(400, 384, 4, 5), K=4, lapnorm=False)


def test_laplacian_eigs_no_threshold_no_normalize(cuda):
    synth = load_pkg("synth")
    f = synth.structured_features(300, 384, 6, 9)
    f = f - f.min() + 0.1  # keep affinities positive without thresholding
    _check_case(cuda, f, K=5, normalize=False, threshold=False)


def test_d_orthonormal_and_constant_first_vector(cuda):
    from oracle import eigs_ref
    synth = load_pkg("synth")
    feats = synth.structured_features(500, 384, 6, 4)
    ev, vec = _check_case(cuda, feats, K=6)
    W, D = eigs_ref.affinity_matrices(feats)
    d = np.diag(D).astype(np.float64)
    G = (vec.astype(np.float64) * d[None]) @ vec.astype(np.float64).T
    assert np.abs(G - np.eye(6)).max() <= 1e-5                     # V^T D V = I
    assert abs(ev[0]) <= 1e-6
    assert np.ptp(vec[0]) <= 1e-7 * abs(vec[0]).max() + 1e-12      # v0 constant


def test_affinity_matches_reference_arithmetic(cuda):
    from oracle import eigs_ref
    spectral = load_pkg("spectral")
    synth = load_pkg("synth")
    for N, d in [(196, 384), (713, 384), (130, 768)]:
        feats = synth.structured_features(N, d, 6, N)
        W = spectral.affinity(feats[None].to(cuda))[0].cpu().numpy()
        W_ref, _ = eigs_ref.affinity_matrices(feats)
        assert W.shape == (N, spectral.pitch(N))
        # the wgmma fp32 accumulation over K = 3d: measured 5e-6 (d = 384, H100 at 400 W) against float64, where the
        # fp32 product is off by 0.5e-6..1.6e-6 (DESIGN.md section 3)
        assert np.abs(W[:, :N] - W_ref).max() <= 1e-5
        assert np.all(W[:, N:] == 0)
        assert W[:, :N].max() <= 1.0 + 1e-6 and W.min() >= 0.0


def test_batch_of_images_independent(cuda):
    spectral = load_pkg("spectral")
    synth = load_pkg("synth")
    B = 40
    feats = torch.stack([synth.structured_features(196, 384, 6, s) for s in range(B)]).to(cuda)
    ev, vec, info, _ = spectral.laplacian_eigs(feats, 5)
    ev1, vec1, _, _ = spectral.laplacian_eigs(feats[7:8], 5)
    torch.cuda.synchronize()
    assert int(info[:, 1].min()) == 1
    assert torch.equal(vec[7], vec1[0]) and torch.equal(ev[7], ev1[0])   # deterministic, no cross-image coupling


def test_known_answer_two_cliques(cuda):
    """Two weakly coupled blocks: lambda_1 small, eigenvector 1 is (D-weighted) piecewise constant with opposite signs."""
    spectral = load_pkg("spectral")
    N = 64
    W = torch.full((N, N), 1e-3)
    W[:32, :32] = 1.0
    W[32:, 32:] = 1.0
    Wd = W[None].contiguous().to(cuda)
    ev, vec, info, _ = spectral.eigsh_laplacian(Wd, N, 3)
    torch.cuda.synchronize()
    W64 = W.double().numpy()
    import scipy.linalg
    d = W64.sum(1)
    vals = scipy.linalg.eigh(np.diag(d) - W64, np.diag(d), eigvals_only=True)[:3]
    assert np.abs(ev[0].cpu().numpy() - vals).max() <= 1e-5
    v1 = vec[0, 1].cpu().numpy()
    assert np.ptp(np.sign(v1[:32])) == 0 and np.ptp(np.sign(v1[32:])) == 0 and np.sign(v1[0]) != np.sign(v1[-1])
