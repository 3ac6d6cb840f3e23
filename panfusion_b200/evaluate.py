"""EvalPanoGen (models/pano/EvalPanoGen.py:18-190): the paper's evaluation table on the sm_90a kernels.

Per panorama it fills 17 metrics over six image sets: the panorama, its roll by W/2 (`rot_`), `num_eval_crops` random
90-degree crops (`crop_`), as many crops on the seam (`seam_`), 8 horizon crops (`mv_`), all at 299x299, and the
generated views against 8 ground-truth crops at the views' size (`pers_`). All crops of a batch come out of one
pf_eval_crops launch as uint8 (the conversion the metrics apply to the reference's fp32 crops, so no fp32 crop is
materialised), and every distinct image goes through the shared InceptionV3 once: its pool3 feeds the FID state and its
logits the IS state (the reference runs each generated set through the network twice). The layout metric is not
computed.

    python -m panfusion_b200.evaluate --results DIR --data DIR [--pano-height 512] [--num-eval-crops 20] [--seed S]
                                      [--out metrics.json]

reads the reference's predict / test layout (`<scene>_<view>/pano.png`, `{0..7}.png`, `prompt.txt` under the results,
`<scene>/matterport_stitched_images/<view>.png` and `<scene>/blip3/<view>_<deg>.txt` under the data) and prints and
writes the metrics.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import sys
from pathlib import Path

import numpy as np
import torch
from torch import nn

from . import _lib, geometry
from .clip_score import CLIPEncoder, CLIPScore
from .faed import FAEDEncoder, FrechetAutoEncoderDistance, load_encoder_state
from .inception import WEIGHTS, FrechetInceptionDistance, InceptionScore, InceptionV3

CROP = 299
FOV = 90.0
MV_VIEWS = 8
CHUNK = 128  # images per Inception forward: bounds the activations (~2.7 MB per 299^2 image at the widest layer)


# ---- host side: cameras and crop bookkeeping ------------------------------------------------------------------------

def random_sample_camera(n: int, rng=np.random) -> tuple[np.ndarray, np.ndarray]:
    """utils/pano.py random_sample_camera: n normal draws of xyz from `rng` (the legacy RandomState API; np.random
    itself by default), normalised, -> (theta, phi) in radians."""
    xyz = rng.normal(size=(n, 3))
    xyz = xyz / (np.linalg.norm(xyz, axis=-1, keepdims=True) + 1e-9)
    return np.arctan2(xyz[:, 0], xyz[:, 1]), np.arcsin(xyz[:, 2].clip(-1, 1))


def horizon_sample_camera(n: int) -> tuple[np.ndarray, np.ndarray]:
    theta = np.linspace(0, 2 * np.pi, n, endpoint=False)
    return theta, np.zeros_like(theta)


def _deg32(theta, phi) -> list[tuple[float, float]]:
    """np.rad2deg, then .float(): the fp32 angles e2p receives, as Python floats."""
    t = torch.from_numpy(np.rad2deg(theta)).float().tolist()
    p = torch.from_numpy(np.rad2deg(phi)).float().tolist()
    return list(zip(t, p))


def draw_cameras(batch_size: int, num_eval_crops: int, rng=np.random) -> dict[str, list]:
    """The cameras of one test_step, in degrees (fp32 values): per panorama a random_sample_camera draw for `crop`, then
    one for `seam` with theta set to 180; `mv` is the 8 horizon cameras shared by every panorama. The draws are per
    panorama, so a batch of B draws what B steps of one panorama draw (the reference draws once per batch, which is
    the same at its batch size of 1)."""
    crop, seam = [], []
    for _ in range(batch_size):
        crop.append(_deg32(*random_sample_camera(num_eval_crops, rng)))
        seam.append([(180.0, p) for _, p in _deg32(*random_sample_camera(num_eval_crops, rng))])
    return {"crop": crop, "seam": seam, "mv": _deg32(*horizon_sample_camera(MV_VIEWS))}


def camera_records(angles: list[tuple[float, float]], h: int, w: int, device) -> torch.Tensor:
    """e2p camera records (PF_CAM_DOUBLES each) of 90-degree cameras at (theta, phi) degrees for h x w crops."""
    recs = [geometry._camera_record("e2p", FOV, t, p, h, w) for t, p in angles]
    return torch.tensor(recs, dtype=torch.float64).to(device)


def slot_counts(batch_size: int, num_eval_crops: int, views: int | None, prompts: bool) -> dict[str, tuple]:
    """Images per metric and side after one test_step: {FID key: (real, fake), IS / CS / FAED key: n or (real, fake)}.
    `views`: images_pred per panorama (None when absent)."""
    B, K = batch_size, num_eval_crops
    out = {"FID": (B, B), "IS": B, "CS": B, "FAED": (B, B), "rot_FID": (B, B), "rot_IS": B, "rot_CS": B,
           "crop_FID": (B * K, B * K), "crop_IS": B * K, "seam_FID": (B * K, B * K), "seam_IS": B * K,
           "mv_FID": (B * MV_VIEWS, B * MV_VIEWS), "mv_IS": B * MV_VIEWS}
    if prompts:
        out["mv_CS"] = B * MV_VIEWS
    if views is not None:
        if views == MV_VIEWS:
            out["pers_FID"], out["pers_IS"] = (B * views, B * views), B * views
        if prompts:
            out["pers_CS"] = B * views
    return out


# ---- kernels --------------------------------------------------------------------------------------------------------

def eval_crops(panos: torch.Tensor, cams: torch.Tensor, crops_per_pano: int, hw: tuple[int, int],
               normalize: bool) -> torch.Tensor:
    """pf_eval_crops: uint8 panoramas [P, 3, H, W] (CUDA) and N camera records -> uint8 crops [N, 3, h, w], crop n from
    panorama n // crops_per_pano. normalize: the crop of `pano.float() / 255` as the metrics convert it to uint8;
    otherwise `e2p(pano.float()).to(torch.uint8)`."""
    _lib.require_cuda(panos, cams)
    if panos.dtype != torch.uint8 or panos.dim() != 4 or panos.shape[1] != 3:
        raise ValueError(f"expected uint8 panoramas [P, 3, H, W], got {panos.dtype} {tuple(panos.shape)}")
    if cams.dtype != torch.float64 or cams.dim() != 2 or cams.shape[1] != _lib.PF_CAM_DOUBLES:
        raise ValueError("expected float64 camera records [N, 20]")
    panos, cams = panos.contiguous(), cams.contiguous()
    P, _, H, W = panos.shape
    N, (h, w) = cams.shape[0], (int(hw[0]), int(hw[1]))
    out = torch.empty(N, 3, h, w, dtype=torch.uint8, device=panos.device)
    with torch.cuda.device(panos.device):
        _lib.check(_lib.lib().pf_eval_crops(C.c_void_p(panos.data_ptr()), P, H, W, crops_per_pano, N, h, w,
                                            C.c_void_p(cams.data_ptr()), int(normalize), C.c_void_p(out.data_ptr()),
                                            C.c_void_p(_lib.stream_ptr())))
    return out


def resize_area2(imgs: torch.Tensor, hw: tuple[int, int]) -> torch.Tensor:
    """cv2.resize(INTER_AREA) of uint8 [B, C, H, W] (CUDA) to hw, for an exact factor of 2 (or the same size);
    anything else raises NotImplementedError (pf_resize_area2_u8)."""
    _lib.require_cuda(imgs)
    if imgs.dtype != torch.uint8 or imgs.dim() != 4:
        raise ValueError(f"expected uint8 images [B, C, H, W], got {imgs.dtype} {tuple(imgs.shape)}")
    imgs = imgs.contiguous()
    B, Cc, H, W = imgs.shape
    out = torch.empty(B, Cc, int(hw[0]), int(hw[1]), dtype=torch.uint8, device=imgs.device)
    with torch.cuda.device(imgs.device):
        _lib.check(_lib.lib().pf_resize_area2_u8(C.c_void_p(imgs.data_ptr()), B, Cc, H, W, out.shape[2], out.shape[3],
                                                 C.c_void_p(out.data_ptr()), C.c_void_p(_lib.stream_ptr())))
    return out


# ---- the evaluation -------------------------------------------------------------------------------------------------

def _panos(x: torch.Tensor, name: str) -> torch.Tensor:
    if x.dtype != torch.uint8 or x.dim() != 5 or x.shape[1] != 1 or x.shape[2] != 3:
        raise ValueError(f"batch['{name}'] must be uint8 [B, 1, 3, H, W], got {x.dtype} {tuple(x.shape)}")
    return x[:, 0].contiguous()


class EvalPanoGen(nn.Module):
    """models/pano/EvalPanoGen.py's metrics and test_step / on_test_end, without the layout metric. Built on the CPU
    (or `device`); `.to(device)` moves every network and state.

    inception: an InceptionV3, a torch-fidelity state dict, or None for the weights file WEIGHTS; one network serves
    all eight Inception metrics. clip: a CLIPEncoder or a local CLIP directory, shared by the four CLIP scores
    (tokenizer as CLIPScore takes it). faed: a FAEDEncoder, an encoder state dict or the FAED checkpoint's path."""

    def __init__(self, num_eval_crops: int = 20, pano_height: int = 512, inception=None,
                 clip="openai/clip-vit-base-patch16", faed="weights/faed.ckpt", tokenizer=None,
                 device: torch.device | str | None = None):
        super().__init__()
        if not isinstance(num_eval_crops, int) or num_eval_crops < 1:
            raise ValueError(f"num_eval_crops must be a positive int, got {num_eval_crops!r}")
        self.num_eval_crops, self.pano_height = num_eval_crops, pano_height
        net = inception if isinstance(inception, InceptionV3) else InceptionV3(WEIGHTS if inception is None else inception)
        enc = clip if isinstance(clip, CLIPEncoder) else CLIPEncoder(clip)
        if not isinstance(faed, FAEDEncoder):
            faed = FAEDEncoder(load_encoder_state(faed) if isinstance(faed, (str, Path)) else faed)
        fid = lambda: FrechetInceptionDistance(inception=net)  # noqa: E731
        iscore = lambda: InceptionScore(inception=net)  # noqa: E731
        cs = lambda: CLIPScore(clip=enc, tokenizer=tokenizer)  # noqa: E731
        # the reference's order: on_test_end computes in it, and each IS compute draws a randperm
        self.eval_metrics = nn.ModuleDict({
            "FID": fid(), "IS": iscore(), "CS": cs(), "rot_FID": fid(), "rot_IS": iscore(), "rot_CS": cs(),
            "crop_FID": fid(), "crop_IS": iscore(), "seam_FID": fid(), "seam_IS": iscore(), "mv_FID": fid(),
            "mv_IS": iscore(), "mv_CS": cs(), "pers_FID": fid(), "pers_IS": iscore(), "pers_CS": cs(),
            "FAED": FrechetAutoEncoderDistance(pano_height, encoder=faed)})
        self.eval_metrics.requires_grad_(False)
        self.inception = net
        self.inception_forwards = 0  # images through the network since construction
        if device is not None:
            self.to(device)

    def reset(self) -> None:
        for m in self.eval_metrics.values():
            m.reset()

    def _features(self, imgs: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
        parts = [self.inception(imgs[i:i + CHUNK]) for i in range(0, imgs.shape[0], CHUNK)]
        self.inception_forwards += imgs.shape[0]
        return torch.cat([p for p, _ in parts]), torch.cat([l for _, l in parts])

    def _fid_is(self, prefix: str, pool3, logits, real_rows, fake_rows) -> None:
        """One panorama's share of `prefix`FID (real then fake) and `prefix`IS (the fake rows)."""
        self.eval_metrics[f"{prefix}FID"].update_features(pool3[real_rows], real=True)
        self.eval_metrics[f"{prefix}FID"].update_features(pool3[fake_rows], real=False)
        self.eval_metrics[f"{prefix}IS"].update_logits(logits[fake_rows])

    @torch.no_grad()
    def test_step(self, batch: dict, rng=np.random) -> dict[str, list]:
        """EvalPanoGen.test_step (EvalPanoGen.py:62-172) on `batch` with the reference's keys: uint8 `pano` and
        `pano_pred` [B, 1, 3, H, W], `pano_prompt` (B strings), optional `prompt` (8 sequences over the batch, as
        collated) and `images_pred` uint8 [B, m, 3, h, w]. The metrics are updated panorama by panorama, so a batch of B
        gives what B steps of one panorama give. -> the cameras drawn (draw_cameras)."""
        dev = self.eval_metrics["FID"].real_features_sum.device
        gt, gen = _panos(batch["pano"], "pano").to(dev), _panos(batch["pano_pred"], "pano_pred").to(dev)
        if gt.shape != gen.shape:
            raise ValueError(f"pano {tuple(gt.shape)} and pano_pred {tuple(gen.shape)} differ in shape")
        B, _, H, W = gt.shape
        K, M = self.num_eval_crops, MV_VIEWS
        pano_prompt = list(batch["pano_prompt"])
        pers_prompt = [p for per_pano in zip(*batch["prompt"]) for p in per_pano] if "prompt" in batch else None
        cams = draw_cameras(B, K, rng)

        # the panoramas and their roll by W/2: one forward of [gt, gen, gt_rot, gen_rot]
        rot_gt, rot_gen = torch.roll(gt, W // 2, 3), torch.roll(gen, W // 2, 3)
        pool3, logits = self._features(torch.cat([gt, gen, rot_gt, rot_gen]))
        # the 299^2 crops of every panorama, gt then gen: per panorama crop (K), seam (K), mv (8) cameras
        per = 2 * K + M
        angles = [a for b in range(B) for a in cams["crop"][b] + cams["seam"][b] + cams["mv"]]
        recs = camera_records(angles, CROP, CROP, dev)
        crops = eval_crops(torch.cat([gt, gen]), torch.cat([recs, recs]), per, (CROP, CROP), normalize=True)
        cpool3, clogits = self._features(crops)

        images_pred = None
        if "images_pred" in batch:
            ip = batch["images_pred"]
            images_pred = ip.reshape(-1, *ip.shape[2:]).to(dev).contiguous()
            if images_pred.dtype != torch.uint8 or images_pred.shape[1] != 3:
                raise ValueError(f"batch['images_pred'] must be uint8 [B, m, 3, h, w], got {ip.dtype} {tuple(ip.shape)}")
        pers = images_pred is not None and images_pred.shape[0] == B * M
        if pers:
            h, w = images_pred.shape[-2:]
            pers_gt = eval_crops(gt, camera_records(cams["mv"] * B, h, w, dev), M, (h, w), normalize=False)
            ppool3, plogits = self._features(torch.cat([pers_gt, images_pred]))

        m = self.eval_metrics
        for b in range(B):
            one = slice(b, b + 1)
            self._fid_is("", pool3, logits, [b], [B + b])
            m["CS"].update(gen[one], pano_prompt[b:b + 1])
            m["FAED"].update(gt[one], real=True)
            m["FAED"].update(gen[one], real=False)
            self._fid_is("rot_", pool3, logits, [2 * B + b], [3 * B + b])
            m["rot_CS"].update(rot_gen[one], pano_prompt[b:b + 1])
            for prefix, off, n in (("crop_", 0, K), ("seam_", K, K), ("mv_", 2 * K, M)):
                rows = torch.arange(n, device=dev) + b * per + off
                self._fid_is(prefix, cpool3, clogits, rows, rows + B * per)
            if pers_prompt is not None:
                mv = torch.arange(M, device=dev) + (B + b) * per + 2 * K
                m["mv_CS"].update(crops[mv], pers_prompt[b * M:(b + 1) * M])
            if pers:
                rows = torch.arange(M, device=dev) + b * M
                self._fid_is("pers_", ppool3, plogits, rows, rows + B * M)
        if images_pred is not None and pers_prompt is not None and images_pred.shape[0] == len(pers_prompt):
            v = images_pred.shape[0] // B
            for b in range(B):
                m["pers_CS"].update(images_pred[b * v:(b + 1) * v], pers_prompt[b * v:(b + 1) * v])
        return cams

    def compute(self) -> dict[str, float]:
        """on_test_end: {key: value} and {key}_std for the IS keys, over the metrics that were updated, computed in
        the reference's order (each IS draws torch.randperm from the global CPU generator)."""
        out = {}
        for key, metric in self.eval_metrics.items():
            if not metric._update_called:
                continue
            if key.endswith("IS"):
                mean, std = metric.compute()
                out[key], out[f"{key}_std"] = float(mean), float(std)
            else:
                out[key] = float(metric.compute())
        return out


# ---- command line ---------------------------------------------------------------------------------------------------

def _load_rgb(path: Path) -> np.ndarray:
    """Equirectangular.from_file / Image.open(...).convert('RGB') as the reference loads them: uint8 [H, W, 3]."""
    from PIL import Image
    img = Image.open(path)
    if img.mode != "RGB":
        img = img.convert("RGB")
    return np.array(img)


def _chw(a: np.ndarray, dev) -> torch.Tensor:
    return torch.from_numpy(a).to(dev).permute(2, 0, 1).contiguous()


def _first_line(path: Path) -> str:
    with open(path) as f:
        return f.readlines()[0]  # load_prompt keeps the line's newline


def load_result(result_dir: Path, data_dir: Path, pano_height: int, pers_resolution: int, dev) -> dict:
    """One `<scene>_<view>` result as the test dataloader gives it (dataset/PanoDataset.py:128-213), batch size 1."""
    scene, view = result_dir.name.split("_", 1)
    H, W = pano_height, 2 * pano_height
    gt = _chw(_load_rgb(data_dir / scene / "matterport_stitched_images" / f"{view}.png"), dev)
    batch = {"pano": resize_area2(gt[None], (H, W))[:, None], "pano_prompt": [_first_line(result_dir / "prompt.txt")]}
    views = []
    while (result_dir / f"{len(views)}.png").exists() and len(views) < MV_VIEWS:
        v = _load_rgb(result_dir / f"{len(views)}.png")
        if v.shape[:2] != (pers_resolution, pers_resolution):
            raise ValueError(f"{result_dir / f'{len(views)}.png'} is {v.shape[1]}x{v.shape[0]}, not the "
                             f"{pers_resolution}x{pers_resolution} of --pers-resolution; resize the views first")
        views.append(v)
    if (result_dir / "pano.png").exists():
        pred = _load_rgb(result_dir / "pano.png")
        if pred.shape[:2] != (H, W):
            raise ValueError(f"{result_dir / 'pano.png'} is {pred.shape[1]}x{pred.shape[0]}, not {W}x{H}")
        batch["pano_pred"] = _chw(pred, dev)[None, None]
    elif views:
        # MVDiffusion results: stitch the views (PanoDataset.py:208-213)
        from . import ops
        theta = np.rad2deg(horizon_sample_camera(len(views))[0])
        pano = ops.mp2e(torch.from_numpy(np.stack(views)).to(dev), [FOV] * len(views), theta, [0.0] * len(views), (H, W))
        batch["pano_pred"] = pano.permute(2, 0, 1).contiguous()[None, None]
    else:
        raise FileNotFoundError(f"{result_dir}: neither pano.png nor views")
    if views:
        batch["images_pred"] = torch.from_numpy(np.stack(views)).to(dev).permute(0, 3, 1, 2).contiguous()[None]
    prompts = [data_dir / scene / "blip3" / f"{view}_{i * 45}.txt" for i in range(MV_VIEWS)]
    if all(p.exists() for p in prompts):
        batch["prompt"] = [[_first_line(p)] for p in prompts]
    return batch


def main(argv=None, **components) -> dict[str, float]:
    """The command line. `components` (inception=, clip=, faed=, tokenizer=) are passed to EvalPanoGen in place of the
    weights the options name."""
    ap = argparse.ArgumentParser(prog="python -m panfusion_b200.evaluate", description=__doc__.split("\n\n")[0])
    ap.add_argument("--results", required=True, type=Path, help="directory of <scene>_<view>/ results")
    ap.add_argument("--data", required=True, type=Path, help="Matterport3D data directory (<scene>/...)")
    ap.add_argument("--pano-height", type=int, default=512)
    ap.add_argument("--pers-resolution", type=int, default=256, help="size of the generated views {0..7}.png")
    ap.add_argument("--num-eval-crops", type=int, default=20)
    ap.add_argument("--seed", type=int, default=None, help="seeds numpy's and torch's global generators")
    ap.add_argument("--out", type=Path, default=None, help="write the metrics as JSON here")
    ap.add_argument("--inception-weights", default=WEIGHTS)
    ap.add_argument("--clip", default="openai/clip-vit-base-patch16", help="local CLIP ViT-B/16 directory")
    ap.add_argument("--faed-ckpt", default="weights/faed.ckpt")
    ap.add_argument("--device", default="cuda")
    args = ap.parse_args(argv)
    dev = torch.device(args.device)
    results = sorted(p for p in args.results.iterdir() if p.is_dir())
    if not results:
        raise FileNotFoundError(f"no <scene>_<view> directories under {args.results}")
    if args.seed is not None:
        np.random.seed(args.seed)
        torch.manual_seed(args.seed)
    ev = EvalPanoGen(args.num_eval_crops, args.pano_height, inception=components.get("inception", args.inception_weights),
                     clip=components.get("clip", args.clip), faed=components.get("faed", args.faed_ckpt),
                     tokenizer=components.get("tokenizer"), device=dev)
    for r in results:
        ev.test_step(load_result(r, args.data, args.pano_height, args.pers_resolution, dev))
    metrics = ev.compute()
    print(json.dumps(metrics, indent=1))
    if args.out is not None:
        args.out.write_text(json.dumps(metrics, indent=1) + "\n")
    return metrics


if __name__ == "__main__":
    main(sys.argv[1:])
