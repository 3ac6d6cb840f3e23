"""Cubemap conversions on the GPU, measured in one run:

    python scripts/cube_micro.py [--views 16] [--workers 16] [--out result.json]

  * pf_c2e_py360: six 1024^2 uint8 RGB faces -> 1024 x 2048 float64 (the Matterport3D stitcher's shape) and
    pf_e2c_py360: 1024 x 2048 uint8 RGB -> 6 x 512^2 faces. Kernel time from CUDA events around 50 back-to-back C-ABI
    launches; the share of HBM bandwidth is (bytes read once + bytes written) / time over 3.35 TB/s (H100 SXM data
    sheet).
  * `python -m panfusion_b200.stitch_mp3d` on a temporary tree of `--views` synthetic skyboxes (1024^2 JPEG faces):
    panoramas per second end to end (decode, GPU c2e, uint8, PNG), against the 1.01 s per panorama that the
    reference's CPU c2e alone takes on one core (numpy 2.3.5, scipy 1.18.1, same shape).
The card's name and power limit are read in the same run and printed with the numbers."""
import argparse
import json
import subprocess
import sys
import tempfile
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from panfusion_b200 import _lib, py360, stitch_mp3d  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
REF_CPU_C2E_S = 1.01


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def time_launches(fn, n=50):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n * 1e-3


def kernels(dev):
    lib, Cv, st = _lib.lib(), _lib.C.c_void_p, _lib.C.c_void_p(_lib.stream_ptr())
    fw, h, w, C = 1024, 1024, 2048, 3
    cube = torch.randint(0, 256, (fw, 6 * fw, C), dtype=torch.uint8, device=dev)
    eq = torch.empty((h, w, C), dtype=torch.float64, device=dev)
    ceil, border = py360._c2e_tables(h, w, fw, dev)
    res = {}
    for mode, name in ((0, "bilinear"), (1, "nearest")):
        t = time_launches(lambda: _lib.check(lib.pf_c2e_py360(Cv(cube.data_ptr()), Cv(eq.data_ptr()), 1, fw, C, h, w,
                                                               Cv(ceil.data_ptr()), Cv(border.data_ptr()), mode, st)))
        nbytes = cube.numel() + eq.numel() * 8
        res[f"c2e_{name}"] = dict(shape="6x1024^2x3 u8 -> 1024x2048x3 f64", us=t * 1e6, bytes=nbytes,
                                  hbm_share=nbytes / t / HBM_BYTES_PER_S)
    pano = torch.randint(0, 256, (h, w, C), dtype=torch.uint8, device=dev)
    fo = 512
    out = torch.empty((fo, 6 * fo, C), dtype=torch.uint8, device=dev)
    for mode, name in ((0, "bilinear"), (1, "nearest")):
        t = time_launches(lambda: _lib.check(lib.pf_e2c_py360(Cv(pano.data_ptr()), Cv(out.data_ptr()), 1, h, w, C, fo,
                                                               mode, st)))
        nbytes = pano.numel() + out.numel()
        res[f"e2c_{name}"] = dict(shape="1024x2048x3 u8 -> 6x512^2x3 u8", us=t * 1e6, bytes=nbytes,
                                  hbm_share=nbytes / t / HBM_BYTES_PER_S)
    return res


def stitcher(views, workers):
    from PIL import Image
    rng = np.random.default_rng(0)
    yy, xx = np.mgrid[0:1024, 0:1024]
    with tempfile.TemporaryDirectory() as root:
        d = Path(root) / "scene0" / "matterport_skybox_images"
        d.mkdir(parents=True)
        for i in range(6):  # smooth synthetic faces, so JPEG / PNG sizes are those of photographs rather than noise
            a, b = rng.random(2) * 0.05
            img = np.stack([np.sin(a * xx + i) * 100 + 128, np.cos(b * yy) * 100 + 128, (xx + yy * i) % 256], -1)
            Image.fromarray(img.astype(np.uint8)).save(d / f"tmpl_skybox{i}_sami.jpg", quality=90)
        for v in range(views):
            for i in range(6):
                (d / f"v{v:03d}_skybox{i}_sami.jpg").write_bytes((d / f"tmpl_skybox{i}_sami.jpg").read_bytes())
        args = ["--mp3d_skybox_path", root, "--scene", "scene0", "--view", "tmpl", "--processes", str(workers)]
        stitch_mp3d.main(args)  # warm-up: module load, tables
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        stitch_mp3d.main(["--mp3d_skybox_path", root, "--processes", str(workers)])
        dt = time.perf_counter() - t0
    n = views + 1  # the scan also finds the template view
    return dict(panoramas=n, seconds=dt, panoramas_per_s=n / dt, workers=workers,
                speedup_vs_ref_cpu_c2e_alone=(n / dt) * REF_CPU_C2E_S)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=16)
    ap.add_argument("--workers", type=int, default=16)
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "cube_micro measures the GPU kernels: no CUDA device"
    dev = torch.device("cuda:0")
    res = dict(card=card(), kernels=kernels(dev), stitcher=stitcher(a.views, a.workers))
    print(json.dumps(res, indent=1))
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
