"""Time the image-space tail (SURVEY.md §8f rank 1) at BASELINE size on one GPU: decode_latent of 8 view latents
64x64 + the circularly padded panorama decode (64x144 -> 512x1024) + tensor_to_image, SD-2 VAE decoder widths,
random-init weights. Algorithmic FLOPs: 2.513 TFLOP per 512x512 image (hand count, 2*MAC) => 8 views 20.1 + pano
(512x1152) 5.65 = 25.8 TFLOP. Usage: python scripts/vae_micro.py [--dtype bf16|fp16]"""
import argparse
import json
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import torch  # noqa: E402

from panfusion_b200 import ops, sd2_unet, vae as pv  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dtype", default="bf16")
    ap.add_argument("--iters", type=int, default=5)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    dt = torch.bfloat16 if args.dtype == "bf16" else torch.float16
    dec = pv.VAEDecoder(sd2_unet.build_synthetic_vae(seed=9, device=dev), dt).prepare(dev, dt)
    g = torch.Generator(device=dev).manual_seed(0)
    lat = torch.randn(1, 8, 4, 64, 64, device=dev, generator=g) * 0.18215 * 4
    pano = torch.randn(1, 1, 4, 64, 128, device=dev, generator=g) * 0.18215 * 4

    def run():
        imgs = pv.decode_latent(lat, dec)
        pan = pv.decode_pano(pano, dec, 8)
        return ops.tensor_to_image(imgs), ops.tensor_to_image(pan.contiguous())

    for _ in range(2):
        run()
    torch.cuda.synchronize()
    l0 = ops.LAUNCHES
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.iters):
        a, b = run()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.iters
    flops = 2.513e12 * 8 + 2.513e12 * (512 * 1152) / (512 * 512)
    print(json.dumps(dict(what="VAE decode 8x512^2 views + 512x1024 pano (latent_pad 8) + tensor_to_image", dtype=args.dtype,
                          ms=round(ms, 2), tflops=round(flops / ms / 1e9, 1), launches=(ops.LAUNCHES - l0) // args.iters,
                          denoise_steps_equiv=round(ms / 28.2, 2), shapes=[list(a.shape), list(b.shape)],
                          peak_mem_gb=round(torch.cuda.max_memory_allocated() / 2 ** 30, 2))))


if __name__ == "__main__":
    main()
