"""CPU: validation of the ViT precision choice (DinoViT, get_model, the extract commands, the localization CLI and
dss_vit_set_precision). Everything here is refused before any device work, so no GPU is needed."""
import ctypes as C

import pytest

from conftest import load_pkg


@pytest.mark.parametrize("bad", ["fp64", "FP32", "bf16", "", None, 32])
def test_dinovit_and_get_model_reject_unknown_precision(bad):
    vit = load_pkg("vit")
    with pytest.raises(ValueError, match="precision"):
        vit.DinoViT("dino_vits16", {}, device="cuda", precision=bad)
    with pytest.raises(ValueError, match="precision"):
        vit.get_model("dino_vits16", seed=0, device="cuda", precision=bad)


def test_extract_commands_reject_unknown_precision(tmp_path):
    ex = load_pkg("extract")
    (tmp_path / "list.txt").write_text("a.png\n")
    with pytest.raises(ValueError, match="precision"):
        ex.extract_features(str(tmp_path / "list.txt"), str(tmp_path), "dino_vits16", 1, str(tmp_path / "f"), seed=0,
                            precision="fp64")
    with pytest.raises(ValueError, match="precision"):
        ex.extract_all(str(tmp_path / "list.txt"), str(tmp_path), "dino_vits16", None, str(tmp_path / "e"), seed=0,
                       precision="half")
    with pytest.raises(ValueError, match="precision"):
        ex.extract_bbox_features(str(tmp_path), str(tmp_path / "boxes.pth"), "dino_vits16", str(tmp_path / "o.pth"),
                                 seed=0, precision="tf32")
    assert not (tmp_path / "f").exists()


def test_cli_flag_reaches_extract_commands():
    cli = load_pkg("cli")
    ex = load_pkg("extract")
    _, kw = cli.parse_args(ex.extract_features, ["--precision", "fp32"])
    assert kw == {"precision": "fp32"}
    _, kw = cli.parse_args(ex.extract_all, ["--precision=fp16"])
    assert kw == {"precision": "fp16"}


def test_localization_precision_flag():
    loc = load_pkg("localize")
    assert loc.parse_args([]).precision == "fp16"
    assert loc.parse_args(["--precision", "fp32"]).precision == "fp32"
    with pytest.raises(SystemExit):
        loc.parse_args(["--precision", "fp64"])


def test_set_precision_on_the_handle():
    L = load_pkg("_lib")
    vit = load_pkg("vit")
    lib = L.load()
    P, d, depth, heads = vit.arch("dino_vits16")
    cfg = L.VitConfig(P, d, depth, heads, vit.MLP_RATIO, vit.TRAIN_IMG // P, vit.LN_EPS)
    h = C.c_void_p()
    assert lib.dss_vit_create(C.byref(cfg), C.byref(h)) == 0
    try:
        fp16_ws = lib.dss_vit_workspace_bytes(h, 2, 480, 480)
        for bad in (-1, 2, 7):
            assert lib.dss_vit_set_precision(h, bad) == -1
            assert b"precision must be" in lib.dss_last_error()
        assert lib.dss_vit_set_precision(None, 1) == -1
        assert lib.dss_vit_workspace_bytes(h, 2, 480, 480) == fp16_ws
        assert lib.dss_vit_set_precision(h, L.VIT_PRECISION["fp32"]) == 0
        fp32_ws = lib.dss_vit_workspace_bytes(h, 2, 480, 480)
        assert fp32_ws > fp16_ws
        assert lib.dss_vit_forward_last_workspace_bytes(h, 2, 479, 479, 1) == fp32_ws
        assert lib.dss_vit_set_precision(h, L.VIT_PRECISION["fp16"]) == 0
        assert lib.dss_vit_workspace_bytes(h, 2, 480, 480) == fp16_ws
    finally:
        lib.dss_vit_destroy(h)
    assert lib.dss_version() >= 2
