"""CPU suite for object localization: the oracle restatements reproduce the reference's own outputs (fixtures written by
oracle/make_localize_golden.py), the VOC reader equals torchvision's VOCDetection + the reference's extract_gt_VOC, the
host CorLoc IoU is the reference's float32 arithmetic at the 0.5 boundary, and the new C entry points reject bad
arguments before any device work."""
import ctypes as C
from pathlib import Path

import numpy as np
import pytest
import scipy.ndimage
import torch

from conftest import ROOT, load_pkg
from oracle import localize_ref
from oracle.make_localize_golden import build_tree

GOLD = ROOT / "tests" / "golden"


def _unpack(flat, offs, i, shape=None):
    a = flat[offs[i]:offs[i + 1]]
    return a.reshape(shape) if shape is not None else a


def test_eigseg_restatement_reproduces_reference():
    z = np.load(GOLD / "ref_loc_eigseg.npz")
    for i in range(len(z["H"])):
        v, H, W = _unpack(z["v"], z["offs"], i), int(z["H"][i]), int(z["W"][i])
        if z["err"][i]:
            with pytest.raises(ValueError):
                localize_ref.eigseg_box(v, H, W)
        else:
            assert np.array_equal(localize_ref.eigseg_box(v, H, W), z["boxes"][i]), i


def test_lost_restatement_reproduces_reference():
    z = np.load(GOLD / "ref_loc_lost.npz")
    assert z["err"].any()
    for i in range(len(z["gh"])):
        f = _unpack(z["feats"], z["offs"], i, (-1, int(z["d"][i])))
        args = ((int(z["gh"][i]), int(z["gw"][i])), (int(z["H"][i]), int(z["W"][i])), int(z["P"][i]), int(z["k"][i]))
        if z["err"][i]:
            with pytest.raises(ValueError, match="background"):
                localize_ref.lost_box(f @ f.T, *args)
        else:
            box, seed = localize_ref.lost_box(f @ f.T, *args)
            assert np.array_equal(box, z["boxes"][i]) and seed == z["seeds"][i], i


def test_dinoseg_restatement_reproduces_reference():
    z = np.load(GOLD / "ref_loc_dinoseg.npz")
    assert z["err"].any()
    for i in range(len(z["gh"])):
        a = _unpack(z["attn"], z["offs"], i, (int(z["heads"][i]), -1))
        grid, P, head = (int(z["gh"][i]), int(z["gw"][i])), int(z["P"][i]), int(z["head"][i])
        if z["err"][i]:
            with pytest.raises(ValueError):
                localize_ref.dinoseg_box(a[head], grid, P)
        else:
            assert np.array_equal(localize_ref.dinoseg_box(a[head], grid, P), z["boxes"][i]), i


GRIDS = [(1, 1), (1, 16384), (16384, 1), (2, 8192), (63, 63), (127, 129), (128, 128)]


def test_cc_patterns_have_the_designed_components():
    """The edge-case masks the GPU tests feed all three kernels: counted with scipy under both connectivities."""
    def count(m, conn8):
        return scipy.ndimage.label(m, structure=localize_ref.EIGHT if conn8 else None)[1]

    for gh, gw in GRIDS:
        p = localize_ref.cc_patterns(gh, gw)
        N = gh * gw
        assert p["all"].all() and not p["none"].any()
        assert 2 * p["half"].sum() == 2 * (N // 2) and p["half_plus_one"].sum() == N // 2 + 1
        if N > 1:
            assert count(p["checkerboard"], True) == 1 or min(gh, gw) == 1
            assert count(p["checkerboard"], False) == p["checkerboard"].sum()
        if min(gh, gw) >= 3:
            assert count(p["row_ends"], True) == p["row_ends"].sum()       # no wrap between the two ends of a row
            assert count(p["row_wrap"], False) == p["row_wrap"].sum()      # nor from one row's end to the next's start
            assert count(p["u"], False) == 1 and count(p["serpentine"], False) == 1
            lab, n = scipy.ndimage.label(p["twin"])
            assert n == 2 and (lab == 1).sum() == (lab == 2).sum()
    assert localize_ref.cc_patterns(128, 128)["dots"].sum() == 4096
    assert scipy.ndimage.label(localize_ref.cc_patterns(128, 128)["twin_then_small"])[1] == 3


def test_dyadic_rows_give_designed_masks_under_torch():
    """Every dyadic row the GPU tests use: exact in fp32 under torch's own CPU sort / sum / cumsum (dyadic_exact), and
    the reference's ops keep exactly the designed cells, with either normalising sum. The last non-kept cell's
    cumulative mass is fl32(0.4) = 0x3ECCCCCD itself, and torch compares with it in fp32 (it is not kept)."""
    assert np.float32(localize_ref.THRESHOLD_UNITS * localize_ref.DYADIC_UNIT).view(np.uint32) == 0x3ECCCCCD
    assert np.float32(1 - 0.6).view(np.uint32) == 0x3ECCCCCD
    assert not (torch.tensor([np.float32(0.4)]) > (1 - 0.6)).item()
    used = zeros = 0
    for gh, gw in GRIDS + [(14, 14), (8, 12)]:
        for name, m in localize_ref.cc_patterns(gh, gw).items():
            try:
                u = localize_ref.dyadic_row(m)
            except ValueError:
                continue
            row = (u * localize_ref.DYADIC_UNIT).astype(np.float32)
            srt = np.sort(u)
            assert np.cumsum(srt)[(~m).sum() - 1] == localize_ref.THRESHOLD_UNITS
            zeros += int((u == 0).sum())
            for total in ("torch", "fp64"):
                assert np.array_equal(localize_ref.dinoseg_kept(row, total), m.ravel()), (gh, gw, name, total)
            used += 1
    assert used >= 60 and zeros >= 100000                              # runs of exact zeros (underflowed softmax)
    # equal values straddling the threshold: the smaller index is the last one not kept
    m = np.zeros((8, 12), bool)
    m[3:6, 4:8] = True
    m[7, 11] = True
    u = localize_ref.dyadic_row(m, tie_cell=2 * 12 + 4)
    assert u[2 * 12 + 4] == u[3 * 12 + 4]
    assert np.array_equal(localize_ref.dinoseg_kept((u * localize_ref.DYADIC_UNIT).astype(np.float32)), m.ravel())


def test_lost_expand_in_chunks_and_sum_decidability():
    """lost_expand reading A in row chunks gives lost_box's seed and M; where torch's CPU sum (the reference's
    torch.sum(A[similars, :], dim=0)) and the sequential fp32 sum have different signs, sum_decided calls the cell
    undecidable."""
    rng = np.random.default_rng(5)
    f = rng.normal(0, 1, (24 * 32, 64)).astype(np.float32)
    A = f @ f.T
    for k in (1, 33, 100, A.shape[0]):
        seed, sim, M = localize_ref.lost_expand(lambda idx: A[idx], A.shape[0], k, chunk=100)
        box, s2 = localize_ref.lost_box(A, (24, 32), (24 * 16, 32 * 16), 16, k)
        assert seed == s2 and np.array_equal(localize_ref.detect_box(M, seed, (24, 32), (384, 512), 16)[0], box)
        m64, decided = localize_ref.sum_decided(A[sim])
        mt = torch.sum(torch.from_numpy(A[sim]), dim=0).numpy()
        assert not ((M > 0) != (mt > 0))[decided].any()
        assert ((M > 0) == (m64 > 0))[decided].all()
    # integer rows: every order is exact, every nonzero cell is decided
    a = rng.integers(-3, 4, (40, 50)).astype(np.float32)
    m64, decided = localize_ref.sum_decided(a)
    assert np.array_equal(decided, m64 != 0)


def _tree(tmp_path):
    z = np.load(GOLD / "ref_loc_main.npz")
    K = z["eig_K"]
    eigs = [_unpack(z["eigs"], z["eig_offs"], i, (int(K[i]), -1)) for i in range(len(K))]
    root, edir = build_tree(Path(tmp_path), list(z["ids"]), list(z["xml"]), [tuple(s) for s in z["sizes"]], eigs)
    return z, root, edir


@pytest.mark.parametrize("no_hard", [False, True])
def test_voc_reader_equals_vocdetection(tmp_path, no_hard):
    import torchvision
    loc = load_pkg("localize")
    z, root, _ = _tree(tmp_path)
    ds = torchvision.datasets.VOCDetection(str(root), year="2007", image_set="trainval", download=False)
    voc = loc.voc_root(str(root), "2007")
    ids = loc.read_voc_list(voc, "trainval")
    assert len(ids) == len(ds)
    for i, iid in enumerate(ids):
        target = ds.parse_voc_xml(__import__("xml.etree.ElementTree").etree.ElementTree.parse(ds.targets[i]).getroot())
        ann = loc.parse_voc_xml(voc / "Annotations" / f"{iid}.xml")
        assert ann["filename"] == target["annotation"]["filename"]
        mine, _ = loc.extract_gt_voc(ann, remove_hards=no_hard)
        want = localize_ref.extract_gt_voc(target, remove_hards=no_hard)
        assert mine.dtype == want.dtype and np.array_equal(mine, want)
        assert loc.jpeg_size(ds.images[i]) == tuple(int(s) for s in z["sizes"][i])


def test_host_iou_is_reference_float32_at_half():
    loc = load_pkg("localize")
    z = np.load(GOLD / "ref_loc_iou.npz")
    for p, g, want in zip(z["pred"], z["gt"], z["iou"]):
        got = loc.bbox_iou(torch.from_numpy(p), torch.from_numpy(g[None]))
        assert got.dtype == torch.float32 and got.numpy()[0].view(np.uint32) == want.view(np.uint32)
        assert loc.corloc_hit(p, g[None]) == bool(want >= 0.5)
    # the fixtures include decisions that float64 arithmetic would flip (IoU just below 0.5 there, 0.5 in float32)
    f64 = np.array([localize_ref.iou_float64(p, g)[0] for p, g in zip(z["pred"], z["gt"])])
    assert ((f64 < 0.5) & (z["iou"] >= 0.5)).any()


def test_unsupported_modes_are_rejected_up_front():
    loc = load_pkg("localize")
    for argv, what in [(["--arch", "resnet50"], "CNN"), (["--arch", "vit_tiny"], "192"), (["--visualize", "pred"], "visualize"),
                       (["--dataset", "COCO20k"], "COCO20k"), (["--patch_size", "14"], "patch size"),
                       (["--eigenseg"], "infer")]:
        with pytest.raises(ValueError, match=what):
            loc.check_supported(loc.parse_args(argv))
    a = loc.parse_args(["--dinoseg", "--arch", "vit_base", "--patch_size", "8", "--dinoseg_head", "2"])
    assert loc.experiment_name(a) == "vit_base-8_dinoseg-head2"
    assert loc.experiment_name(loc.parse_args(["--which_features", "q"])) == "LOST-vit_small16_q"
    assert loc.ARCH_MAP[("vit_small", 8)] == "dino_vits8"


def test_localization_entry_points_reject_bad_arguments_before_any_device_work():
    _lib = load_pkg("_lib")
    lib = _lib.load()
    n0 = lib.dss_kernel_launch_count()
    buf = torch.zeros(1 << 16, dtype=torch.uint8)
    p = (buf.data_ptr() + 255) // 256 * 256
    dims = (C.c_int * 4)(64, 64, 64, 64)
    ws = 1 << 15
    assert lib.dss_eigseg_boxes(None, 1, 2, 64, 1, dims, p, p, p, ws, None) == -1            # null evecs
    assert lib.dss_eigseg_boxes(p, 1, 2, 64, 2, dims, p, p, p, ws, None) == -1               # row >= K
    assert lib.dss_eigseg_boxes(p, 1, 2, 129 * 128, 1, dims, p, p, p, ws, None) == -4        # > 128 x 128 cells
    assert lib.dss_eigseg_boxes(p, 2, 2, 64, 1, dims, p, p, p, 8, None) == -3                # workspace too small
    assert lib.dss_lost_boxes(None, 1, 16, 16, 4, 4, 64, 64, 16, 100, p, None, p, p, ws, None) == -1
    assert lib.dss_lost_boxes(p, 1, 16, 16, 4, 5, 64, 64, 16, 100, p, None, p, p, ws, None) == -1   # grid != N
    assert lib.dss_lost_boxes(p, 1, 16, 16, 4, 4, 64, 64, 16, 0, p, None, p, p, ws, None) == -1     # k_patches 0
    assert lib.dss_lost_boxes(p, 1, 129 * 128, 129 * 128, 129, 128, 64, 64, 16, 100, p, None, p, p, ws, None) == -4
    assert lib.dss_dinoseg_boxes(p, 1, 6, 16, 6, 4, 4, 16, p, p, None) == -1                # head >= heads
    assert lib.dss_dinoseg_boxes(p, 1, 6, 16, -1, 4, 4, 16, p, p, None) == -1
    assert lib.dss_dinoseg_boxes(None, 1, 6, 16, 0, 4, 4, 16, p, p, None) == -1
    assert lib.dss_dinoseg_boxes(p, 1, 6, 129 * 128, 0, 129, 128, 16, p, p, None) == -4
    assert lib.dss_op_cls_attention(None, 1, 5, 6, p, None) == -1
    assert lib.dss_op_cls_attention(p, 1, 1, 6, p, None) == -1                              # T < 2
    assert lib.dss_op_im2col_pad_f16(p, p, 1, 20, 20, 12, None) == -1                       # P not a multiple of 8
    cfg = _lib.VitConfig(16, 384, 12, 6, 4, 14, 1e-6)
    h = C.c_void_p()
    assert lib.dss_vit_create(C.byref(cfg), C.byref(h)) == 0
    assert lib.dss_vit_forward_last_workspace_bytes(h, 1, 20, 20, 1) > lib.dss_vit_forward_last_workspace_bytes(h, 1, 20, 20, 0)
    assert lib.dss_vit_forward_last_workspace_bytes(h, 1, 8, 8, 0) == 0                     # crop: smaller than a patch
    assert lib.dss_vit_forward_last(h, p, 1, 224, 224, 1, 3, p, None, p, ws, None) == -1    # which not q / k / v
    assert lib.dss_vit_forward_last(h, p, 1, 224, 224, 1, 1, None, None, p, ws, None) == -1 # no output
    assert lib.dss_vit_forward_last(h, p, 1, 224, 224, 1, 1, p, None, p, ws, None) == -1    # weights not loaded
    lib.dss_vit_destroy(h)
    assert lib.dss_kernel_launch_count() == n0


def test_command_shim_and_module_import():
    src = (ROOT / "object-localization" / "main.py").read_text()
    assert "localize" in src
    loc = load_pkg("localize")
    assert loc.SEGMENT_INDEX == {"matting": 1, "laplacian": 1, "affinity": 0}
