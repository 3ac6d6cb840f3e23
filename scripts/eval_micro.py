"""Time EvalPanoGen.test_step (panfusion_b200.evaluate) on one GPU: panoramas per second at 512x1024 with the default 20
eval crops and 8 generated views of 256x256, with prompts, after warm-up, between CUDA events. Prints the card's name
and power limit read in the same run, and the Inception forwards per panorama against the reference's.

    python scripts/eval_micro.py [--steps 10] [--warmup 3] [--batch 1]

The networks carry seeded weights of the real shapes (the oracle's): the time does not depend on their values.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from oracle import clip_score as oc  # noqa: E402
from oracle import eval_pano as oe  # noqa: E402
from oracle import faed as of  # noqa: E402
from oracle import inception as oi  # noqa: E402
from panfusion_b200 import evaluate  # noqa: E402
from panfusion_b200.clip_score import CLIPEncoder  # noqa: E402
from panfusion_b200.inception import InceptionV3  # noqa: E402


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    name, power = (q.stdout.strip().split(", ") + ["?", "?"])[:2] if q.returncode == 0 else (torch.cuda.get_device_name(), "?")
    return {"gpu": name, "power_limit": power}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=1)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    B, K = args.batch, 20
    ev = evaluate.EvalPanoGen(K, 512, inception=InceptionV3(oi.synth_state()),
                              clip=CLIPEncoder(oc.seeded_state(), oc.clip_config()), faed=of.synth_state(),
                              tokenizer=oe.tokenizer, device=dev)
    batch = dict(pano=oc.structured_images(1, B, 512, 1024)[:, None].to(dev),
                 pano_pred=oc.structured_images(2, B, 512, 1024)[:, None].to(dev),
                 images_pred=oc.structured_images(3, 8 * B, 256, 256).reshape(B, 8, 3, 256, 256).to(dev),
                 pano_prompt=[f"a living room with a sofa {b}" for b in range(B)],
                 prompt=[[f"view {v} of room {b}" for b in range(B)] for v in range(8)])
    rng = np.random.RandomState(0)
    for _ in range(args.warmup):
        ev.test_step(batch, rng)
    torch.cuda.synchronize()
    ev.inception_forwards = 0
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(args.steps):
        ev.test_step(batch, rng)
    t1.record()
    torch.cuda.synchronize()
    ms = t0.elapsed_time(t1) / args.steps
    counts = evaluate.slot_counts(1, K, 8, True)
    ref = sum(sum(counts[k]) for k in counts if k.endswith("FID")) + sum(counts[k] for k in counts if k.endswith("IS"))
    out = {"workload": f"EvalPanoGen.test_step 512x1024, {K} crops, 8 views 256x256, batch {B}",
           "ms_per_step": round(ms, 2), "panoramas_per_s": round(1000.0 * B / ms, 3),
           "inception_forwards_per_pano": ev.inception_forwards / (args.steps * B),
           "reference_inception_forwards_per_pano": ref, **card()}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
