"""Train the FAED autoencoder on a directory of stitched panoramas and write the checkpoint FAED reads
(`python main.py fit --model=FAED` of the reference, on the sm_90a kernels):

    python -m panfusion_b200.train_faed --images 'data/pano/*.png' --pano-height 512 --batch-size 4 --epochs 60 \\
        --out weights/faed.ckpt [--resume] [--seed 0]

The loader is host code on a thread pool, as dataset/PanoDataset.py prepares a panorama for training: read as RGB
(utils/pano.py Equirectangular.from_file), horizontal flip with p = 0.5, cv2.resize(INTER_AREA) to
pano_height x 2 pano_height, / 127.5 - 1. The last incomplete batch of an epoch is dropped.
"""
from __future__ import annotations

import argparse
import glob
import os
import random
from concurrent.futures import ThreadPoolExecutor

import cv2
import numpy as np
import torch
from PIL import Image


def load_pano(path: str, height: int, flip: bool) -> np.ndarray:
    """fp32 [3, height, 2 height] in [-1, 1]."""
    img = Image.open(path)
    if img.mode != "RGB":
        img = img.convert("RGB")
    a = np.array(img)
    if flip:
        a = np.flip(a, 1)
    a = cv2.resize(np.ascontiguousarray(a), (2 * height, height), interpolation=cv2.INTER_AREA)
    return np.ascontiguousarray((a.astype(np.float32) / 127.5 - 1).transpose(2, 0, 1))


def batches(paths, height, batch_size, rng: random.Random, pool: ThreadPoolExecutor):
    """One epoch of pinned fp32 [B, 3, H, 2H] batches: shuffled order, a flip coin per panorama."""
    order = list(paths)
    rng.shuffle(order)
    jobs = [(p, rng.random() < 0.5) for p in order]
    for i in range(0, len(jobs) - batch_size + 1, batch_size):
        arrs = list(pool.map(lambda j: load_pano(j[0], height, j[1]), jobs[i: i + batch_size]))
        yield torch.from_numpy(np.stack(arrs)).pin_memory() if torch.cuda.is_available() else \
            torch.from_numpy(np.stack(arrs))


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--images", required=True, help="glob of panorama images")
    ap.add_argument("--pano-height", type=int, default=512)
    ap.add_argument("--batch-size", type=int, default=4)
    ap.add_argument("--epochs", type=int, default=60)
    ap.add_argument("--lr", type=float, default=1e-4)
    ap.add_argument("--lr-decay", type=float, default=0.99)
    ap.add_argument("--out", default=os.path.join("weights", "faed.ckpt"))
    ap.add_argument("--resume", action="store_true", help="continue from --out")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--workers", type=int, default=8)
    a = ap.parse_args(argv)
    paths = sorted(glob.glob(a.images))
    if len(paths) < a.batch_size:
        raise SystemExit(f"{a.images}: {len(paths)} images, fewer than one batch of {a.batch_size}")
    if a.pano_height % 32:
        raise SystemExit(f"--pano-height {a.pano_height} must be a multiple of 32")
    from .faed_train import FAEDTrainer
    tr = FAEDTrainer(a.out if a.resume else None, lr=a.lr, lr_decay=a.lr_decay, seed=a.seed)
    with ThreadPoolExecutor(a.workers) as pool:
        for epoch in range(tr.epoch, a.epochs):
            # one generator per (seed, epoch): a --resume run sees the same order and flips as an uninterrupted one
            rng = random.Random(f"{a.seed}:{epoch}")
            losses = []
            for x in batches(paths, a.pano_height, a.batch_size, rng, pool):
                losses.append(tr.training_step(x.to(tr.device, non_blocking=True)))
            mean = torch.stack(losses).nanmean().item()  # a skipped step has a non-finite loss
            tr.on_train_epoch_end()
            print(f"epoch {epoch}: train/loss {mean:.5f} steps {tr.global_step} skipped {tr.skipped_steps} "
                  f"lr {tr.lr:.3e}", flush=True)
            os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
            tr.save_checkpoint(a.out)


if __name__ == "__main__":
    main()
