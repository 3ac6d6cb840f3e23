"""Time one FAED autoencoder training step (B = 4, 512x1024 by default) on the sm_90a kernels against PyTorch eager
fp32 (cuDNN, TF32 convolutions as the reference runs them) of the same module, alternating the two in one process,
and break our step down by kernel family with torch.profiler. Prints the card name and power limit with the numbers.

    python scripts/faed_train_micro.py [--batch 4] [--height 512] [--iters 10] [--warmup 3]
"""
from __future__ import annotations

import argparse
import subprocess
import sys
from collections import defaultdict
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from panfusion_b200 import faed_train as ft  # noqa: E402


def forward_flops(B, H, W):
    """Multiply-adds x 2 of every convolution in AutoEncoder.forward, counted with forward hooks."""
    net = ft.AutoEncoder()
    total = [0]

    def hook(mod, inp, out):
        total[0] += 2 * out.numel() * mod.in_channels * mod.kernel_size[0] * mod.kernel_size[1]

    for m in net.modules():
        if isinstance(m, torch.nn.Conv2d):
            m.register_forward_hook(hook)
    with torch.no_grad(), torch.device("meta"):
        net.to("meta")(torch.empty(B, 3, H, W, device="meta"))
    return total[0]


def family(name: str) -> str:
    for key, fam in (("wgrad", "wgrad"), ("conv_mma", "conv (forward + dgrad)"), ("bn_", "batchnorm"),
                     ("upsample", "upsample"), ("adam", "adam"), ("pack", "weight pack"), ("loss", "loss"),
                     ("interleave", "dgrad interleave")):
        if key in name:
            return fam
    return "other"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--height", type=int, default=512)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print(f"device: {q}")
    B, H, W = a.batch, a.height, 2 * a.height
    fl = forward_flops(1, H, W)
    print(f"forward: {fl / 1e9:.1f} GFLOP per {H}x{W} panorama; training step ~3x: {3 * fl * B / 1e9:.0f} GFLOP "
          f"at B = {B}")
    pano = (torch.rand(B, 3, H, W, device=dev) * 2 - 1)
    tr = ft.FAEDTrainer(seed=0, device=dev)
    net = ft.AutoEncoder().to(dev).train()
    opt = torch.optim.Adam(net.parameters(), lr=1e-4)
    torch.backends.cudnn.allow_tf32 = True

    def ours():
        tr.training_step(pano)

    def eager():
        opt.zero_grad(set_to_none=True)
        (net(pano) - pano).abs().mean().backward()
        opt.step()

    for _ in range(a.warmup):
        ours()
        eager()
    torch.cuda.synchronize()
    times = defaultdict(list)
    for _ in range(a.iters):
        for name, fn in (("ours", ours), ("eager", eager)):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1))
    for name in ("ours", "eager"):
        t = sorted(times[name])
        med = t[len(t) // 2]
        print(f"{name}: median {med:.1f} ms per step (min {t[0]:.1f}, max {t[-1]:.1f}), "
              f"{3 * fl * B / med / 1e9:.1f} TFLOP/s on the ~3x-forward count")
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            ours()
        torch.cuda.synchronize()
    fam = defaultdict(float)
    for ev in prof.key_averages():
        fam[family(ev.key)] += ev.device_time_total / 3 / 1e3
    for k, v in sorted(fam.items(), key=lambda kv: -kv[1]):
        print(f"  {k}: {v:.2f} ms per step")
    print(f"skipped steps: {tr.skipped_steps}")


if __name__ == "__main__":
    main()
