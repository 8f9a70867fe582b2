"""CPU: the pieces of the semantic-segmentation stages that need no GPU -- the library's positional-embedding
interpolation against the upstream restatement at the grids box crops produce, the upstream identity rule that decides
from pixel sizes, PCA's acceptance rule, and the hand-built label maps of the box oracle."""
import numpy as np
import pytest
import torch

from conftest import load_pkg


# 1 x 1, 1 x n, n x 1, 196 patches as 7 x 28 / 28 x 7, grid0 +- 1 and the stored grid; ViT-B/8 (grid0 28) 1 x 80 / 80 x 1
@pytest.mark.parametrize("name,Hp,Wp", [
    ("dino_vits16", 1, 1), ("dino_vits16", 1, 25), ("dino_vits16", 25, 1), ("dino_vits16", 7, 28),
    ("dino_vits16", 28, 7), ("dino_vits16", 13, 13), ("dino_vits16", 15, 15), ("dino_vits16", 13, 15),
    ("dino_vits16", 14, 14), ("dino_vits16", 2, 98), ("dino_vitb8", 1, 80), ("dino_vitb8", 80, 1),
    ("dino_vitb8", 27, 27), ("dino_vitb8", 29, 29), ("dino_vitb8", 28, 28), ("dino_vitb8", 1, 1)])
def test_pos_embed_interpolation_at_box_crop_grids(name, Hp, Wp):
    from oracle import dino_vit
    vit = load_pkg("vit")
    ref = dino_vit.build(name, seed=Hp * 100 + Wp)
    P = ref.cfg.patch
    want = ref.interpolate_pos_encoding(Hp * Wp, Hp * P, Wp * P)[0]
    got = vit.pos_embed_interp_host(ref.pos_embed, ref.cfg.grid0, Hp, Wp)
    assert got.shape == want.shape
    if Hp == Wp == ref.cfg.grid0:
        assert torch.equal(got, want)
    else:
        assert (got - want).abs().max().item() <= 2e-6


@pytest.mark.parametrize("name,H,W", [("dino_vits16", 224, 232), ("dino_vits16", 239, 224), ("dino_vitb8", 224, 231)])
def test_upstream_resamples_a_stored_size_grid_from_non_square_pixels(name, H, W):
    """The rule the library follows for uncropped inputs: a grid0 x grid0 patch grid from an H != W input is resampled
    with scale (grid0 + 0.1) / grid0 -- not the identity -- and keeps its grid0 x grid0 size."""
    from oracle import dino_vit
    ref = dino_vit.build(name, seed=1)
    g, P = ref.cfg.grid0, ref.cfg.patch
    assert H // P == g and W // P == g
    pos = ref.interpolate_pos_encoding(g * g, H, W)
    assert pos.shape == ref.pos_embed.shape
    assert torch.equal(pos[0, 0], ref.pos_embed[0, 0])
    assert (pos[0, 1:] - ref.pos_embed[0, 1:]).abs().max().item() > 1e-4
    assert ref.interpolate_pos_encoding(g * g, H, H) is ref.pos_embed


@pytest.mark.parametrize("M,p", [(31, 32), (1, 1), (10, 64), (0, 1)])
def test_pca_refuses_more_components_than_rows(M, p):
    """scikit-learn's rule: pca_dim <= min(M, d), and at least two rows for a covariance with ddof 1. Checked before
    anything touches a device."""
    cluster = load_pkg("cluster")
    with pytest.raises(ValueError, match="rows"):
        cluster.pca(torch.ones(M, 384), p)


def test_edge_maps_hold_what_they_promise():
    from oracle import bbox_ref
    for H, W in [(1, 16384), (16384, 1), (2, 8192), (127, 129), (128, 128)]:
        maps = bbox_ref.edge_maps(H, W)
        assert all(m.shape == (H, W) and m.dtype == np.uint8 for m in maps.values())
        assert len(np.unique(maps["all_values"])) == 256
        assert np.unique(maps["zeros"]).tolist() == [0] and np.unique(maps["ones255"]).tolist() == [255]
        assert np.unique(maps["checker"]).tolist() == [0, 255]
        assert len(np.unique(maps["squares"])) > 5
    sq = bbox_ref.edge_maps(64, 64)["squares"]
    for s, v in ((1, 11), (3, 12), (5, 13), (9, 15)):          # side 2t - 1 empties at erosion step t: kept from t - 1
        m = sq == v
        assert m.sum() == s * s
        assert bbox_ref.erode_or_dilate_mask(m, r=(s - 1) // 2, erode=True).sum() == 1
        assert bbox_ref.erode_or_dilate_mask(m, r=(s + 1) // 2 + 3, erode=True).sum() == 1
