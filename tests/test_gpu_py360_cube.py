"""GPU: pf_c2e_py360 / pf_e2c_py360 (py360convert.c2e / e2c, external/py360convert/c2e.py:6-64, e2c.py:6-40) on every
golden case and at the stitcher's real size, against the numpy oracle (which the golden's digests pin bit for bit to the
executed reference), and the
`python -m panfusion_b200.stitch_mp3d` CLI end to end on synthetic skybox JPEGs.

Gates (device float32 trig is the float64 function rounded, numpy's float32 kernels are within about an ulp of that,
so a coordinate can move by an ulp): c2e float64 mean |d| <= 1e-4 and max |d| <= 5e-2, its uint8 truncation one level
apart on < 1e-3 of the values; e2c uint8 one level apart on < 1e-3, fp32 max |d| <= 5e-2; `nearest` identical but for
< 1e-4 of the values (ties)."""
import numpy as np
import pytest
import torch

import _py360_cube_oracle as oc
from panfusion_b200 import py360

pytestmark = pytest.mark.gpu


def _c2e_gate(got, ref, mode, tag, what):
    assert got.dtype == np.float64 and got.shape == ref.shape, what
    d = np.abs(got - ref)
    if mode == "nearest":
        assert (d > 0).mean() < 1e-4, (what, (d > 0).mean())
        return
    assert d.mean() <= 1e-4 and d.max() <= 5e-2, (what, d.mean(), d.max())
    if tag == "u8":
        t = np.abs(got.astype(np.uint8).astype(int) - ref.astype(np.uint8).astype(int))
        assert t.max() <= 1 and (t > 0).mean() < 1e-3, (what, t.max(), (t > 0).mean())
    print(f"{what}: mean |d| {d.mean():.2e} max |d| {d.max():.2e}")


def _e2c_gate(got, ref, mode, tag, what):
    assert got.dtype == ref.dtype and got.shape == ref.shape, what
    d = np.abs(got.astype(np.float64) - ref.astype(np.float64))
    if mode == "nearest":
        assert (d > 0).mean() < 1e-4, (what, (d > 0).mean())
    elif tag == "u8":
        assert d.max() <= 1 and (d > 0).mean() < 1e-3, (what, d.max(), (d > 0).mean())
    else:
        assert d.max() <= 5e-2, (what, d.max())
    print(f"{what}: max |d| {d.max():.2e}, {(d > 0).mean():.2e} of values differ")


def test_c2e_e2c_vs_reference_cases(cuda_device):
    """Every golden case, against the restatement on the same seeded input (pinned bit for bit to the executed
    reference by the golden's digests in test_py360_cube.py)."""
    for k, (fw, (h, w), mode, tag, C, fmt) in enumerate(oc.C2E_CASES):
        cube = oc.c2e_input(k)
        got = py360.c2e(cube, h, w, mode=mode, cube_format=fmt)                      # numpy in -> numpy out
        assert isinstance(got, np.ndarray)
        _c2e_gate(got, oc.c2e(oc.as_horizon(cube, fmt), h, w, mode), mode, tag, f"c2e case {k}")
    for k, (fw, _, mode, tag, C, fmt) in enumerate(oc.E2C_CASES):
        im = oc.e2c_input(k)
        got = py360.e2c(im, face_w=fw, mode=mode, cube_format=fmt)
        _e2c_gate(oc.as_horizon(got, fmt), oc.e2c(im, fw, mode), mode, tag, f"e2c case {k}")


def _photo_like(shape, seed):
    """Smooth seeded uint8 content with a little grain: gradients of a few levels per pixel, like a photograph."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:shape[0], 0:shape[1]].astype(np.float64)
    ch = [np.sin(xx * a + yy * b + p) * 90 + 128 for a, b, p in rng.random((shape[2], 3)) * [0.02, 0.02, 6.0]]
    return np.clip(np.stack(ch, -1) + rng.normal(0, 2, shape), 0, 255).astype(np.uint8)


def test_c2e_e2c_vs_oracle_at_stitcher_size(cuda_device):
    """Six 1024^2 uint8 faces -> 1024 x 2048 (the Matterport3D stitcher), and back to 256^2 faces (e2c's default).
    A face coordinate that differs by one float32 ulp (about 6e-5 pixel at face_w 1024) moves a bilinear value by
    that fraction of the local gradient, so the mean gate is applied to photograph-like faces; white-noise faces, the
    worst case (gradients up to 255 levels per pixel), are held to the max |d| gate (e2c: one level)."""
    cube = _photo_like((1024, 6 * 1024, 3), 7)
    for mode in ("bilinear", "nearest"):
        got = py360.c2e(cube, 1024, 2048, mode=mode, cube_format="horizon")
        _c2e_gate(got, oc.c2e(cube, 1024, 2048, mode), mode, "u8", f"c2e 1024^2 -> 1024x2048 {mode}")
    noise = oc.seeded((1024, 6 * 1024, 3), "u8", 7)
    d = np.abs(py360.c2e(noise, 1024, 2048, cube_format="horizon") - oc.c2e(noise, 1024, 2048))
    print(f"c2e 1024^2 white noise: mean |d| {d.mean():.2e} max |d| {d.max():.2e}")
    assert d.max() <= 5e-2, d.max()
    pano = _photo_like((1024, 2048, 3), 8)
    for mode in ("bilinear", "nearest"):
        got = py360.e2c(pano, 256, mode=mode, cube_format="horizon")
        _e2c_gate(got, oc.e2c(pano, 256, mode), mode, "u8", f"e2c 1024x2048 -> 256^2 {mode}")
    noise = oc.seeded((1024, 2048, 3), "u8", 8)
    d = np.abs(py360.e2c(noise, 256, cube_format="horizon").astype(int) - oc.e2c(noise, 256).astype(int))
    print(f"e2c 1024x2048 white noise: {(d > 0).mean():.2e} of values one level apart")
    assert d.max() <= 1, d.max()


def test_repeatable_and_numpy_matches_cuda_tensor(cuda_device):
    cube = oc.seeded((64, 384, 3), "u8", 9)
    pano = oc.seeded((96, 200, 3), "f32", 10)
    t, tp = torch.from_numpy(cube).to(cuda_device), torch.from_numpy(pano).to(cuda_device)
    for mode in ("bilinear", "nearest"):
        a = py360.c2e(t, 96, 200, mode=mode, cube_format="horizon")
        assert a.is_cuda and a.dtype == torch.float64 and a.shape == (96, 200, 3)
        for _ in range(3):
            assert torch.equal(py360.c2e(t, 96, 200, mode=mode, cube_format="horizon"), a)
        assert np.array_equal(py360.c2e(cube, 96, 200, mode=mode, cube_format="horizon"), a.cpu().numpy())
        b = py360.e2c(tp, 40, mode=mode, cube_format="dice")                          # CUDA in -> CUDA out, any layout
        assert b.is_cuda and b.dtype == torch.float32 and b.shape == (120, 160, 3)
        for _ in range(3):
            assert torch.equal(py360.e2c(tp, 40, mode=mode, cube_format="dice"), b)
        assert np.array_equal(py360.e2c(pano, 40, mode=mode, cube_format="dice"), b.cpu().numpy())
        d = py360.e2c(tp, 40, mode=mode, cube_format="dict")
        assert all(torch.equal(d[k], v) for k, v in py360.cube_h2dict(py360.cube_dice2h(b)).items())
    # a 2-D-per-face list of CUDA tensors goes through the same kernel
    faces = py360.cube_h2list(t)
    assert torch.equal(py360.c2e(faces, 96, 200, cube_format="list"), py360.c2e(t, 96, 200, cube_format="horizon"))


def _orient_like_from_mp3d_skybox(imgs):
    """utils/pano.py:127-139 restated: skybox0..5 = U L F R B D; R, B mirrored; U flipped up-down, rotated; D rotated."""
    U, L, F, R, B, D = imgs
    return np.concatenate([F, R[:, ::-1], B[:, ::-1], L, np.rot90(U[::-1], 1), np.rot90(D, 1)], 1)


def test_stitch_mp3d_cli_matches_oracle_pipeline(cuda_device, tmp_path):
    from PIL import Image
    from panfusion_b200 import stitch_mp3d
    rng = np.random.default_rng(11)
    yy, xx = np.mgrid[0:256, 0:256]
    views = {"sceneA": ["v0", "v1"], "sceneB": ["w0"]}
    for scene, vs in views.items():
        d = tmp_path / scene / "matterport_skybox_images"
        d.mkdir(parents=True)
        for v in vs:
            for i in range(6):
                a, b, c = rng.random(3) * 0.2
                img = np.stack([np.sin(a * xx + i) * 100 + 128, np.cos(b * yy) * 100 + 128, (xx * c + yy) % 256], -1)
                Image.fromarray(img.astype(np.uint8)).save(d / f"{v}_skybox{i}_sami.jpg", quality=90)
    assert stitch_mp3d.main(["--mp3d_skybox_path", str(tmp_path), "--processes", "3"]) == 0
    for scene, vs in views.items():
        for v in vs:
            assert (tmp_path / scene / "matterport_stitched_images" / f"{v}.png").exists()
    # one view against the oracle pipeline on the same decoded faces; the single-view form writes the same file
    png = tmp_path / "sceneA" / "matterport_stitched_images" / "v1.png"
    got = np.array(Image.open(png))
    png.unlink()
    assert stitch_mp3d.main(["--mp3d_skybox_path", str(tmp_path), "--scene", "sceneA", "--view", "v1",
                             "--processes", "0"]) == 0
    assert np.array_equal(np.array(Image.open(png)), got)
    faces = [np.array(Image.open(p)) for p in stitch_mp3d.skybox_paths(str(tmp_path), "sceneA", "v1")]
    cube = _orient_like_from_mp3d_skybox(faces)
    assert np.array_equal(stitch_mp3d.skybox_cube(faces), cube)
    ref = oc.c2e(cube, 1024, 2048).astype(np.uint8)
    assert got.shape == (1024, 2048, 3) and got.dtype == np.uint8
    t = np.abs(got.astype(int) - ref.astype(int))
    assert t.max() <= 1 and (t > 0).mean() < 1e-3, (t.max(), (t > 0).mean())
