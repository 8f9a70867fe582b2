"""CPU suite for the semantic-segmentation stages: the box oracle against the reference's stored outputs, the host-side
semantic maps against the reference's stored PNGs, and argument checks of the new C entry points."""
import ast

import numpy as np
import pytest
import torch
from PIL import Image

from conftest import ROOT, load_pkg

GOLDEN = ROOT / "tests" / "golden"


def _golden(name):
    return np.load(GOLDEN / name, allow_pickle=False)


def _maps(z):
    return {k[4:]: z[k] for k in z.files if k.startswith("map_")}


def test_bbox_oracle_matches_reference_outputs():
    from oracle import bbox_ref
    z = _golden("ref_bboxes.npz")
    cases = ast.literal_eval(str(z["cases"]))
    for ci, (ne, nd, skip, ds) in enumerate(cases):
        for name, m in _maps(z).items():
            P = 16 if ds is None else ds
            out = bbox_ref.extract_bbox(m, name, P, ne, nd, skip)
            rows = np.array([[s, *b, *o] for s, b, o in zip(out["segment_indices"], out["bboxes"],
                                                           out["bboxes_original_resolution"])], np.int64).reshape(-1, 9)
            assert np.array_equal(rows, z[f"case{ci}_{name}"]), (ci, name)
            types = (type(out["segment_indices"][0]).__name__, type(out["bboxes"][0][0]).__name__,
                     type(out["bboxes_original_resolution"][0][0]).__name__, out["format"])
            assert repr(types) == str(z[f"types_case{ci}_{name}"])


def test_bbox_dict_has_the_reference_element_types():
    """The host assembly of the kernel's boxes (extract._bbox_dict) against the reference's stored types and values."""
    ex = load_pkg("extract")
    z = _golden("ref_bboxes.npz")
    cases = ast.literal_eval(str(z["cases"]))
    ci = 0
    ne, nd, skip, ds = cases[ci]
    for name in _maps(z):
        want = z[f"case{ci}_{name}"]
        boxes = np.zeros((256, 4), np.int32)
        present = np.zeros(256, bool)
        for row in want:
            boxes[row[0]] = row[1:5]
            present[row[0]] = True
        present[0] = True      # the background is present and skipped
        d = ex._bbox_dict(name, 16, boxes, present, skip)
        got = np.array([[s, *b, *o] for s, b, o in zip(d["segment_indices"], d["bboxes"], d["bboxes_original_resolution"])],
                       np.int64).reshape(-1, 9)
        assert np.array_equal(got, want)
        types = (type(d["segment_indices"][0]).__name__, type(d["bboxes"][0][0]).__name__,
                 type(d["bboxes_original_resolution"][0][0]).__name__, d["format"])
        assert repr(types) == str(z[f"types_case{ci}_{name}"])
        assert set(d) == {"bboxes", "bboxes_original_resolution", "segment_indices", "id", "format"}


def _write_semantic_inputs(tmp_path, z):
    sdir = tmp_path / "segs"
    sdir.mkdir()
    bbox_list = []
    for name, m in _maps(z).items():
        Image.fromarray(m).save(sdir / f"{name}.png")
        bbox_list.append({"id": name, "bboxes": [[0, 0, 1, 1]] * len(z[f"segment_indices_{name}"]),
                          "segment_indices": z[f"segment_indices_{name}"].tolist(), "clusters": z[f"clusters_{name}"]})
    return sdir, bbox_list


def test_semantic_segmentations_match_reference_pngs(tmp_path):
    ex = load_pkg("extract")
    z = _golden("ref_semantic_segmaps.npz")
    sdir, bbox_list = _write_semantic_inputs(tmp_path, z)
    torch.save(bbox_list, tmp_path / "clusters.pth")
    ex.extract_semantic_segmentations(str(sdir), str(tmp_path / "clusters.pth"), str(tmp_path / "out"), yes=True)
    for name in _maps(z):
        img = Image.open(tmp_path / "out" / f"{name}.png")
        assert img.mode == "L"
        got = np.array(img)
        assert got.dtype == np.uint8 and np.array_equal(got, z[f"semantic_{name}"]), name
    assert set(np.unique(z["map_binary"]).tolist()) == {0, 255}     # the binary case is covered


def test_semantic_map_rejects_inconsistent_inputs():
    ex = load_pkg("extract")
    m = np.array([[0, 1], [2, 2]], np.uint8)
    assert np.array_equal(ex.semantic_map(m, [1, 2], np.array([5, 0], np.int32)), [[0, 5], [0, 0]])
    with pytest.raises(ValueError, match="segment indices"):
        ex.semantic_map(m, [1, 2], np.array([5], np.int32))
    with pytest.raises(ValueError, match="no cluster"):
        ex.semantic_map(m, [1], np.array([5], np.int32))
    with pytest.raises(ValueError, match="background"):
        ex.semantic_map(m, [0, 1, 2], np.array([1, 2, 3], np.int32))


def test_new_entry_points_reject_bad_arguments_before_any_device_work():
    _lib = load_pkg("_lib")
    lib = _lib.load()
    n0 = lib.dss_kernel_launch_count()
    buf = torch.zeros(1 << 16, dtype=torch.uint8)
    p = (buf.data_ptr() + 255) // 256 * 256
    BAD, UNSUP = -1, -4
    # boxes
    assert lib.dss_segment_bboxes(None, 1, 8, 8, 2, 3, p, p, None) == BAD
    assert lib.dss_segment_bboxes(p, 0, 8, 8, 2, 3, p, p, None) == BAD
    assert lib.dss_segment_bboxes(p, 1, 8, 0, 2, 3, p, p, None) == BAD
    assert lib.dss_segment_bboxes(p, 1, 8, 8, -1, 3, p, p, None) == BAD
    assert lib.dss_segment_bboxes(p, 1, 129, 129, 2, 3, p, p, None) == UNSUP        # grid larger than 128 x 128
    # covariance / projection
    assert lib.dss_covariance(None, 10, 4, p, p, 4, p, 1 << 15, None) == BAD
    assert lib.dss_covariance(p, 1, 4, p, p, 4, p, 1 << 15, None) == BAD               # one row
    assert lib.dss_covariance(p, 10, 8, p, p, 4, p, 1 << 15, None) == BAD              # ldc < d
    assert lib.dss_covariance(p, 10, 4, p, p, 4, p + 8, 1 << 15, None) == BAD          # misaligned workspace
    assert lib.dss_covariance(p, 10, 4, p, p, 4, p, 16, None) == -3                    # workspace too small
    assert lib.dss_covariance(p, 10, 2048, p, p, 2048, p, 1 << 15, None) == UNSUP
    assert lib.dss_pca_project(p, 10, 8, p, p, 0, p, None) == BAD
    assert lib.dss_pca_project(p, 10, 8, None, p, 4, p, None) == BAD
    assert lib.dss_pca_project(p, 10, 128, p, p, 65, p, None) == UNSUP
    # k-means
    ws = 1 << 15
    assert lib.dss_kmeans(None, 100, 8, 4, 0, 300, 1e-4, p, p, p, None, p, ws, None) == BAD
    assert lib.dss_kmeans(p, 0, 8, 4, 0, 300, 1e-4, p, p, p, None, p, ws, None) == BAD
    assert lib.dss_kmeans(p, 100, 8, 0, 0, 300, 1e-4, p, p, p, None, p, ws, None) == BAD
    assert lib.dss_kmeans(p, 3, 8, 4, 0, 300, 1e-4, p, p, p, None, p, ws, None) == BAD       # k > M
    assert lib.dss_kmeans(p, 100, 8, 4, 0, 300, 1e-4, p, p, p, None, p + 8, ws, None) == BAD
    assert lib.dss_kmeans(p, 1000, 769, 4, 0, 300, 1e-4, p, p, p, None, p, ws, None) == UNSUP
    assert lib.dss_kmeans(p, 1000, 768, 65, 0, 300, 1e-4, p, p, p, None, p, ws, None) == UNSUP
    assert lib.dss_kmeans(p, 1000, 65, 256, 0, 300, 1e-4, p, p, p, None, p, ws, None) == UNSUP
    assert lib.dss_kmeans(p, 1000, 64, 257, 0, 300, 1e-4, p, p, p, None, p, ws, None) == UNSUP
    assert lib.dss_kmeans(p, 100000, 32, 21, 0, 300, 1e-4, p, p, p, None, p, 16, None) == -3  # workspace too small
    assert lib.dss_kmeans_workspace_bytes(1000, 768, 65) == 0
    assert lib.dss_kmeans_workspace_bytes(1000, 768, 64) > 0 and lib.dss_kmeans_workspace_bytes(1000, 64, 256) > 0
    assert lib.dss_covariance_workspace_bytes(1000, 384) > 0
    assert lib.dss_kernel_launch_count() == n0


def test_pca_dim_above_the_eigensolver_limit_is_rejected():
    _lib = load_pkg("_lib")
    cluster = load_pkg("cluster")
    with pytest.raises(_lib.DssError, match="at most 64"):
        cluster.pca_components(torch.zeros(1, 1), 384, 65)
