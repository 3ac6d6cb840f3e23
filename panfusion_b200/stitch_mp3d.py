"""Stitch Matterport3D skyboxes into 1024 x 2048 equirectangular PNGs on the GPU: `scripts.stitch_mp3d` of the reference
(its README's first data step) with the same flags and output path.

    python -m panfusion_b200.stitch_mp3d [--mp3d_skybox_path data/Matterport3D/mp3d_skybox] [--scene S --view V]
                                         [--processes 16]

For each view, the six `<view>_skybox{0..5}_sami.jpg` faces are oriented like `Cubemap.from_mp3d_skybox`
(utils/pano.py:127-139), stitched with `py360.c2e` (pf_c2e_py360) and truncated to uint8 like `Equirectangular.save`
(utils/pano.py:154-156) before `<scene>/matterport_stitched_images/<view>.png` is written. JPEG decoding and PNG
encoding run on `--processes` host worker threads (Pillow releases the GIL while it codes), ahead of and behind the GPU.
"""
from __future__ import annotations

import argparse
import glob
import os
from collections import deque
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch
from PIL import Image

from . import py360

SKYBOX_KEYS = ("U", "L", "F", "R", "B", "D")  # face of skybox0 .. skybox5


def skybox_paths(root, scene, view):
    return [os.path.join(root, scene, "matterport_skybox_images", f"{view}_skybox{i}_sami.jpg") for i in range(6)]


def output_path(root, scene, view):
    return os.path.join(root, scene, "matterport_stitched_images", f"{view}.png")


def skybox_cube(faces) -> np.ndarray:
    """Six decoded skybox images (skybox0 .. skybox5) -> horizon cube [fw, 6 fw, C] (from_mp3d_skybox's orientation:
    R and B mirrored left-right, U flipped upside down then rotated by 90 degrees, D rotated by 90 degrees)."""
    f = dict(zip(SKYBOX_KEYS, faces))
    f["R"], f["B"] = np.flip(f["R"], 1), np.flip(f["B"], 1)
    f["U"] = np.rot90(np.flip(f["U"], 0), 1)
    f["D"] = np.rot90(f["D"], 1)
    return np.ascontiguousarray(py360.cube_dict2h(f))


def load_cube(root, scene, view) -> np.ndarray:
    return skybox_cube([np.array(Image.open(p)) for p in skybox_paths(root, scene, view)])


def stitch(cube_h: np.ndarray, h: int = 1024, w: int = 2048) -> np.ndarray:
    """Horizon cube -> uint8 equirect [h, w, C]: c2e on the GPU, then the float64 result truncated on the GPU."""
    x = torch.from_numpy(cube_h).cuda()
    return py360.c2e(x, h, w, "bilinear", cube_format="horizon").to(torch.uint8).cpu().numpy()


def save_png(img: np.ndarray, path: str) -> None:
    os.makedirs(os.path.dirname(path), exist_ok=True)
    Image.fromarray(img).save(path)


def list_views(args):
    """(scene, view) pairs: the one given, or every view with skybox images under every scene directory."""
    if args.scene is not None and args.view is not None:
        return [(args.scene, args.view)]
    jobs = []
    for scene in sorted(os.listdir(args.mp3d_skybox_path)):
        if not os.path.isdir(os.path.join(args.mp3d_skybox_path, scene)):
            continue
        jpgs = glob.glob(os.path.join(args.mp3d_skybox_path, scene, "matterport_skybox_images", "*.jpg"))
        jobs += [(scene, v) for v in sorted({os.path.basename(p).split("_")[0] for p in jpgs})]
    return jobs


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description="Stitch Matterport3D Skybox")
    ap.add_argument("--mp3d_skybox_path", type=str, default="data/Matterport3D/mp3d_skybox",
                    help="Matterport3D mp3d_skybox path")
    ap.add_argument("--processes", type=int, default=16, help="host workers for JPEG decoding and PNG encoding")
    ap.add_argument("--scene", default=None, type=str, help="scene id")
    ap.add_argument("--view", default=None, type=str, help="view id")
    return ap.parse_args(argv)


def main(argv=None) -> int:
    args = parse_args(argv)
    root = args.mp3d_skybox_path
    jobs = list_views(args)
    workers = max(1, args.processes)
    with ThreadPoolExecutor(workers) as pool:
        loads = deque(pool.submit(load_cube, root, s, v) for s, v in jobs[:workers])
        saves = []
        for k, (scene, view) in enumerate(jobs):
            cube = loads.popleft().result()
            if k + workers < len(jobs):
                loads.append(pool.submit(load_cube, root, *jobs[k + workers]))
            saves.append(pool.submit(save_png, stitch(cube), output_path(root, scene, view)))
        for f in saves:
            f.result()
    print(f"stitched {len(jobs)} panoramas")
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
