"""Speed of the CLIP score on the GPU: images/s of CLIPScore.update at batch 1, 16 and 64 for uint8 512x1024 panoramas
(CS, rot_CS) and fp32 299x299 crops (mv_CS), split into the image tower, the text tower and the whole update, with the
towers' TFLOP/s computed from their shapes.

    python scripts/clip_micro.py [--iters 20] [--prompt-len 20]

Weights are seeded random tensors with the ViT-B/16 geometry (speed does not depend on their values). Prints one line
per case, the card's name and power limit (read-only nvidia-smi query) and one JSON line. Exits non-zero without a GPU.
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

from panfusion_b200.clip_score import CLIPEncoder, CLIPScore, _config, expected_shapes  # noqa: E402

CONFIG = {"text_config": dict(hidden_size=512, num_attention_heads=8, num_hidden_layers=12, intermediate_size=2048,
                              hidden_act="quick_gelu", vocab_size=49408, max_position_embeddings=77),
          "vision_config": dict(hidden_size=768, num_attention_heads=12, num_hidden_layers=12, intermediate_size=3072,
                                hidden_act="quick_gelu", patch_size=16, image_size=224),
          "projection_dim": 512}


def tower_flops(B: int, L: int) -> tuple[float, float]:
    """Multiply-add FLOPs (x2) of the image tower for B images and of the text tower for B prompts of L tokens."""
    def layers(T, C, I, n, L_):
        per = 2 * T * C * 3 * C + 2 * T * C * C + 2 * 2 * T * C * I + 2 * 2 * T * L_ * C
        return n * per
    v = 2 * B * 196 * 768 * 768 + layers(B * 197, 768, 3072, 12, 197) + 2 * B * 768 * 512
    t = layers(B * L, 512, 2048, 12, L) + 2 * B * 512 * 512
    return v, t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--prompt-len", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("clip_micro: no CUDA device")
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(0)
    sd = {}
    for k, shape in expected_shapes(_config(CONFIG)).items():
        fan = shape[1] * (shape[2] * shape[3] if len(shape) == 4 else 1) if len(shape) > 1 else 0
        if fan:
            sd[k] = torch.randn(shape, generator=g) / fan ** 0.5
        elif "norm" in k and k.endswith("weight"):
            sd[k] = torch.ones(shape)
        else:
            sd[k] = 0.02 * torch.randn(shape, generator=g)
    enc = CLIPEncoder(sd, CONFIG)
    L = args.prompt_len
    tok = lambda text, padding=True, return_tensors="pt": {
        "input_ids": torch.cat([torch.full((len(text), 1), 49406), torch.randint(1, 49406, (len(text), L - 2),
                                generator=g), torch.full((len(text), 1), 49407)], 1)}
    metric = CLIPScore(clip=enc, tokenizer=tok, device=dev)

    def timed(fn):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(args.iters):
            fn()
        e.record()
        torch.cuda.synchronize()
        return s.elapsed_time(e) / args.iters

    rows = []
    for name, shape, dtype in (("pano_512x1024_u8", (512, 1024), torch.uint8), ("crop_299_f32", (299, 299), torch.float32)):
        for B in (1, 16, 64):
            x = torch.randint(0, 256, (B, 3, *shape), generator=g, dtype=torch.uint8)
            x = (x.float() / 255 if dtype == torch.float32 else x).to(dev)
            text = ["a prompt"] * B
            ids = metric.token_ids(text)
            t_prep = timed(lambda: enc.prep(x))
            t_img = timed(lambda: enc.encode_image(x))
            t_txt = timed(lambda: enc.encode_text(ids, dev))
            t_upd = timed(lambda: metric.update(x, text))
            fv, ft = tower_flops(B, L)
            r = dict(case=name, batch=B, prep_ms=round(t_prep, 3), image_tower_ms=round(t_img, 3),
                     text_tower_ms=round(t_txt, 3), update_ms=round(t_upd, 3),
                     images_per_s=round(B / t_upd * 1e3, 1), image_tower_tflops=round(fv / t_img / 1e9, 1),
                     text_tower_tflops=round(ft / t_txt / 1e9, 1))
            rows.append(r)
            print(f"{name} B={B:3d}: prep {t_prep:.3f} ms, image tower {t_img:.3f} ms ({r['image_tower_tflops']} TFLOP/s), "
                  f"text tower {t_txt:.3f} ms ({r['text_tower_tflops']} TFLOP/s), update {t_upd:.3f} ms "
                  f"= {r['images_per_s']} images/s")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    card = smi.stdout.strip().splitlines()[0] if smi.returncode == 0 and smi.stdout.strip() else "nvidia-smi unavailable"
    print(f"card: {card}")
    print(json.dumps({"card": card, "prompt_len": L, "rows": rows}))


if __name__ == "__main__":
    main()
