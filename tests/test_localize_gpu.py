"""GPU suite for object localization: the three box kernels against the oracle restatement and the reference's
fixtures (exact), the CLS-attention kernel, the zero-padded / q / v ViT outputs against the fp32 oracle, and the
command end to end."""
import pickle
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from conftest import ROOT, load_pkg
from oracle import dino_vit, localize_ref
from oracle.make_localize_golden import build_tree

pytestmark = pytest.mark.gpu
GOLD = ROOT / "tests" / "golden"


def _unpack(flat, offs, i, shape=None):
    a = flat[offs[i]:offs[i + 1]]
    return a.reshape(shape) if shape is not None else a


def test_eigseg_kernel_matches_fixtures(cuda):
    loc = load_pkg("localize")
    z = np.load(GOLD / "ref_loc_eigseg.npz")
    for i in range(len(z["H"])):
        v = torch.from_numpy(_unpack(z["v"], z["offs"], i)).to(cuda)
        boxes, status = loc.eigseg_boxes(v[None, None], 0, [(int(z["H"][i]), int(z["W"][i]))])
        if z["err"][i]:
            assert status[0] == 1
        else:
            assert status[0] == 0 and np.array_equal(boxes[0], z["boxes"][i]), i


@pytest.mark.parametrize("P", [8, 16])
def test_eigseg_kernel_random_masks_batched(cuda, P):
    """Densities 0.05 - 0.95 around both percolation thresholds, grids 1x1 .. 128x128; a batch of images of different
    sizes with the same cell count gives the same boxes as each image alone."""
    loc = load_pkg("localize")
    rng = np.random.default_rng(P)
    grids = [(1, 1), (1, 7), (5, 1), (3, 3), (17, 23), (64, 64), (100, 128), (128, 128), (128, 1), (37, 91)]
    for gh, gw in grids:
        dens = np.linspace(0.05, 0.95, 10)
        V = np.stack([np.where(rng.random(gh * gw) < d, 1.0, -1.0) for d in dens]).astype(np.float32)
        # sizes with the same cell count on the P grid: not multiples of P
        sizes = [(gh * P + int(rng.integers(0, P)), gw * P + int(rng.integers(0, P))) for _ in dens]
        boxes, status = loc.eigseg_boxes(torch.from_numpy(V)[:, None].to(cuda), 0, sizes)
        assert (status == 0).all()
        for j in range(len(dens)):
            want = localize_ref.eigseg_box(V[j], *sizes[j])
            assert np.array_equal(boxes[j], want), (gh, gw, dens[j])
            alone, _ = loc.eigseg_boxes(torch.from_numpy(V[j:j + 1])[:, None].to(cuda), 0, [sizes[j]])
            assert np.array_equal(alone[0], boxes[j])


def test_lost_kernel_matches_fixtures(cuda):
    loc = load_pkg("localize")
    z = np.load(GOLD / "ref_loc_lost.npz")
    for i in range(len(z["gh"])):
        f = torch.from_numpy(_unpack(z["feats"], z["offs"], i, (-1, int(z["d"][i])))).to(cuda)
        boxes, seeds, status = loc.lost_boxes(f[None], (int(z["gh"][i]), int(z["gw"][i])), (int(z["H"][i]), int(z["W"][i])),
                                              int(z["P"][i]), int(z["k"][i]))
        assert seeds[0] == z["seeds"][i], i
        if z["err"][i]:
            assert status[0] == 2
        else:
            assert status[0] == 0 and np.array_equal(boxes[0], z["boxes"][i]), i


def test_lost_kernel_real_valued_features(cuda):
    """Real-valued features: exact against the oracle given the same A (the affinity kernel's F F^T), so no sign of an
    A_ij near 0 can differ between the two."""
    loc = load_pkg("localize")
    spectral = load_pkg("spectral")
    rng = np.random.default_rng(7)
    for gh, gw, d in [(24, 32, 64), (20, 20, 384), (47, 63, 64)]:
        f = torch.from_numpy(rng.normal(0, 1, (6, gh * gw, d)).astype(np.float32)).to(cuda)
        size = (gh * 16 - 5, gw * 16 - 3)
        boxes, seeds, status = loc.lost_boxes(f, (gh, gw), size, 16, 100)
        A = spectral.affinity(f, normalize=False, threshold_at_zero=False, scale_by_max=False)[:, :, :gh * gw].cpu().numpy()
        for b in range(6):
            want, seed = localize_ref.lost_box(A[b], (gh, gw), size, 16, 100)
            assert status[b] == 0 and seeds[b] == seed and np.array_equal(boxes[b], want)


def test_dinoseg_kernel_matches_fixtures_and_random_maps(cuda):
    loc = load_pkg("localize")
    z = np.load(GOLD / "ref_loc_dinoseg.npz")
    for i in range(len(z["gh"])):
        a = torch.from_numpy(_unpack(z["attn"], z["offs"], i, (int(z["heads"][i]), -1))).to(cuda)
        boxes, status = loc.dinoseg_boxes(a[None], (int(z["gh"][i]), int(z["gw"][i])), int(z["P"][i]), int(z["head"][i]))
        if z["err"][i]:
            assert status[0] == 3
        else:
            assert status[0] == 0 and np.array_equal(boxes[0], z["boxes"][i]), i
    rng = np.random.default_rng(3)
    checked = 0
    for gh, gw in [(24, 32), (63, 63), (128, 128), (3, 5)]:
        s = rng.normal(0, 2, (4, 6, gh * gw))
        a = (np.exp(s) / np.exp(s).sum(-1, keepdims=True)).astype(np.float32)
        boxes, status = loc.dinoseg_boxes(torch.from_numpy(a).to(cuda), (gh, gw), 16, 4)
        for b in range(4):
            row = a[b, 4]
            # the kernel normalises by the exactly rounded sum; torch's float sum may differ by an ulp and keep other cells
            k64 = localize_ref.dinoseg_kept(row, "fp64")
            assert status[b] == 0 and np.array_equal(boxes[b], localize_ref.dinoseg_select(k64, (gh, gw), 16)[0])
            if np.array_equal(k64, localize_ref.dinoseg_kept(row)):
                assert np.array_equal(boxes[b], localize_ref.dinoseg_box(row, (gh, gw), 16))
                checked += 1
    assert checked >= 12


def test_cls_attention_kernel(cuda):
    """Against the float64 softmax of the same fp16 qkv, logits of standard deviation 1. (At a logit spread of 4 the
    fp32 rounding of the scores alone reaches 1.3e-6 relative.)"""
    _lib = load_pkg("_lib")
    g = torch.Generator(device=cuda).manual_seed(197)   # its own stream: the draw must not depend on earlier tests
    for B, T, heads in [(2, 197, 6), (3, 1025, 12), (1, 2, 6)]:
        qkv = torch.randn(B, T, 3 * heads * 64, generator=g, device=cuda).half()   # q . k / 8 has standard deviation 1
        out = torch.empty(B, heads, T - 1, device=cuda)
        _lib.check(_lib.load().dss_op_cls_attention(qkv.data_ptr(), B, T, heads, out.data_ptr(), _lib.stream_ptr(cuda)))
        want = localize_ref.cls_attention_from_qkv(qkv.cpu(), heads)
        err = out.cpu().double() - want
        rel = (err.norm(dim=-1) / want.norm(dim=-1)).max().item()          # per (image, head) row
        assert rel <= 1e-6, rel
        # per element, from the kernel's roundings (1e-6 of the row's max is not a bound: some draws exceed it)
        _, bound = localize_ref.cls_attention_bound(qkv, heads)
        assert (err.abs() <= bound).all(), float((err.abs() / bound).max())


@pytest.mark.parametrize("name", ["dino_vits16", "dino_vits8"])
def test_pad_mode_vit_outputs_match_oracle(cuda, name):
    vit = load_pkg("vit")
    synth = load_pkg("synth")
    ref = dino_vit.build(name, seed=1).to(cuda)
    model = vit.DinoViT(name, ref.state_dict(), device=cuda)
    P = model.patch_size
    for H, W in [(375, 500), (333, 500), (500, 500)]:
        img = synth.blobs_batch(1, H, W, seed0=H).to(cuda)
        x = localize_ref.preprocess_pad(img[0].cpu(), P).to(cuda)
        for which in ("q", "k", "v"):
            f, a = model.forward_last(img, which, pad=True, cls_attn=(which == "k"))
            wf, wa = localize_ref.last_outputs(ref, x, which)
            assert f.shape == wf.shape
            rel = float((f - wf).norm() / wf.norm())
            assert rel <= 3e-3, (H, W, which, rel)
            if a is not None:
                rel_a = float((a - wa).norm() / wa.norm())
                assert rel_a <= 3e-3, (H, W, rel_a)
        # crop mode: the K features are the bits dss_vit_forward_k writes
        fk, _ = model.forward_last(img, "k", pad=False)
        assert torch.equal(fk, model.forward_k(img))


def _run_main(tmp_path, argv):
    cmd = [sys.executable, str(ROOT / "object-localization" / "main.py")] + argv
    return subprocess.run(cmd, cwd=tmp_path, capture_output=True, text=True, check=True)


@pytest.mark.parametrize("tag", ["hard", "nohard"])
def test_main_eigenseg_precomputed_matches_reference(cuda, tmp_path, tag):
    z = np.load(GOLD / "ref_loc_main.npz")
    K = z["eig_K"]
    eigs = [_unpack(z["eigs"], z["eig_offs"], i, (int(K[i]), -1)) for i in range(len(K))]
    _, edir = build_tree(tmp_path, list(z["ids"]), list(z["xml"]), [tuple(s) for s in z["sizes"]], eigs)
    extra = ["--no_hard"] if tag == "nohard" else []
    r = _run_main(tmp_path, ["--eigenseg", "--precomputed_eigs_dir", str(edir), "--output_dir", "outputs"] + extra)
    folder = tmp_path / "outputs" / ("VOC07_trainval" + ("-nohards" if extra else "")) / "LOST-vit_small16_k"
    assert (folder / "results.txt").read_bytes() == z[f"{tag}_results"].tobytes()
    assert "corloc:" in r.stdout
    preds = pickle.loads((folder / "preds.pkl").read_bytes())
    gt = pickle.loads((folder / "gt.pkl").read_bytes())
    names = list(z[f"{tag}_names"])
    assert list(preds) == names and list(gt) == names
    for i, n in enumerate(names):
        assert preds[n].dtype == np.int64 and np.array_equal(preds[n], z[f"{tag}_preds"][i])
        g = _unpack(z[f"{tag}_gt"], z[f"{tag}_gt_offs"], i, (-1, 4))
        assert gt[n].dtype == np.int64 and np.array_equal(gt[n], g)


def test_methods_from_images_match_oracle_postprocessing(cuda):
    """LOST, DINO-seg and eigenseg from features on blobs images with seeded weights: the boxes equal the oracle's
    post-processing of the GPU's own features / attention; the share of boxes with IoU >= 0.5 against the full fp32
    oracle pipeline is measured and printed."""
    loc = load_pkg("localize")
    vit = load_pkg("vit")
    spectral = load_pkg("spectral")
    synth = load_pkg("synth")
    ref = dino_vit.build("dino_vits16", seed=2).to(cuda)
    model = vit.DinoViT("dino_vits16", ref.state_dict(), device=cuda)
    H, W, P, B = 333, 500, 16, 4
    gh, gw = -(-H // P), -(-W // P)
    img = synth.blobs_batch(B, H, W, seed0=11).to(cuda)
    f, a = model.forward_last(img, "k", pad=True, cls_attn=True)
    A = spectral.affinity(f, normalize=False, threshold_at_zero=False, scale_by_max=False)
    lb, _, ls = loc.lost_boxes(f, (gh, gw), (H, W), P, 100)
    db, ds = loc.dinoseg_boxes(a, (gh, gw), P, 4)
    fc, _ = model.forward_last(img, "k", pad=False)
    _, ev, _, _ = spectral.laplacian_eigs(fc, 2, normalize=False, threshold_at_zero=True, lapnorm=True)
    eb, es = loc.eigseg_boxes(ev, 1, [(H, W)] * B)
    An, an, evn = A.cpu().numpy()[:, :, :gh * gw], a.cpu().numpy(), ev.cpu().numpy()
    agree = []
    for b in range(B):
        assert ls[b] == 0 and np.array_equal(lb[b], localize_ref.lost_box(An[b], (gh, gw), (H, W), P, 100)[0])
        assert ds[b] == 0 and np.array_equal(db[b], localize_ref.dinoseg_box(an[b, 4], (gh, gw), P))
        assert es[b] == 0 and np.array_equal(eb[b], localize_ref.eigseg_box(evn[b, 1], H, W))
        x = localize_ref.preprocess_pad(img[b].cpu(), P).to(cuda)
        wf, wa = localize_ref.last_outputs(ref, x, "k")
        wf = wf[0].cpu().numpy()
        ob, _ = localize_ref.lost_box(wf @ wf.T, (gh, gw), (H, W), P, 100)
        od = localize_ref.dinoseg_box(wa[0, 4].cpu().numpy(), (gh, gw), P)
        for got, want in ((lb[b], ob), (db[b], od)):
            agree.append(float(loc.bbox_iou(torch.from_numpy(got), torch.from_numpy(want[None]))[0]) >= 0.5)
    print(f"boxes with IoU >= 0.5 against the full fp32 oracle pipeline: {sum(agree)}/{len(agree)}")
    assert all(agree)   # measured on an H100: 8 of 8 (LOST and DINO-seg, 4 images)
