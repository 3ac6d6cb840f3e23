"""MVDiffusion denoiser on one GPU: steps/s of the CFG-batched forward at the default configuration (8 horizon views,
512^2 images = 64^2 latents, CFG pair, SD-2 widths, seeded random weights), the time of each CPAttn kernel per level,
and FLOP / byte accounting computed from shapes. Prints one JSON line; the card's name and power limit are read in the
same run.

    python scripts/mvdiff_bench.py [--steps 10] [--warmup 3] [--dtype bf16]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))


def _events_ms(fn, reps: int) -> float:
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--dtype", choices=["bf16", "fp16"], default="bf16")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mvdiff_bench needs a CUDA device")
    from oracle import mvdiffusion as omv, unet as ou
    from panfusion_b200 import ops
    from panfusion_b200.mvdiffusion import MultiViewBaseModel, homographies
    dt = torch.bfloat16 if args.dtype == "bf16" else torch.float16
    dev = torch.device("cuda:0")
    m, hw = 8, 64
    orc = omv.build_model(omv.MultiViewBaseModel, ou.SD2_CONFIG)
    model = MultiViewBaseModel(orc.unet, compute_dtype=dt)
    model.load_state_dict(orc.state_dict())
    model.prepare(dev, dt)
    inp = omv.step_inputs_cfg(m, hw, ou.SD2_CONFIG["cross_attention_dim"])
    cu = dict(inp, latents=inp["latents"].to(dev), timestep=inp["timestep"].to(dev), prompt_embd=inp["prompt_embd"].to(dev))
    for _ in range(args.warmup):
        model(**cu)
    step_ms = _events_ms(lambda: model(**cu), args.steps)

    # per-level CPAttn kernels on the same inputs' shapes (B = 2 CFG halves, camera tables shared)
    K, R = inp["meta"]["K"], inp["meta"]["R"]
    hl, hr = (t.to(dev).contiguous() for t in homographies(K[:1], R[:1]))
    levels = {}
    for blk, h in ((model.cp_blocks_encoder[0], 64), (model.cp_blocks_encoder[1], 32), (model.cp_blocks_encoder[2], 16),
                   (model.cp_blocks_encoder[3], 8)):
        C, T = blk.dim, 2 * m * h * h
        rows = 18 * T
        x = torch.randn(T, C, device=dev).to(dt)
        w = blk._pack(dev, dt)
        pos, mask = blk.tables.get(blk.tables.camera_key(K, R), h, h, 512, dev)
        keys, st = ops.cpattn_gather(x, 2, m, h, h, pos, mask, w["freq"])
        kv = torch.empty(rows, 2 * C, dtype=dt, device=dev)
        o = torch.empty(T, C, dtype=dt, device=dev)
        reps = 20
        t_tab = _events_ms(lambda: ops.cpattn_tables(hl, hr, h, h, 512), reps)
        t_gather = _events_ms(lambda: ops.cpattn_gather(x, 2, m, h, h, pos, mask, w["freq"]), reps)
        t_kv = _events_ms(lambda: ops.gemm_taps(keys, w["kv_ln"].w, kv, M=rows, Kc=C, bias=w["kv_ln"].b,
                                                ln=(st, w["kv_ln"].colsum, w["kv_ln"].eps)), reps)
        t_attn = _events_ms(lambda: ops.cpattn_attn(x, kv, o, 32 ** -0.5), reps)
        kv_flop = 2.0 * rows * C * 2 * C
        gather_bytes = rows * C * 2 + rows * 16 + T * C * 2            # key rows + stats written, features read once
        attn_bytes = rows * 2 * C * 2 + 2 * T * C * 2
        levels[f"{h}x{h}"] = dict(
            C=C, key_rows=rows,
            tables_ms=round(t_tab, 4), gather_ms=round(t_gather, 4), kv_gemm_ms=round(t_kv, 4), attn_ms=round(t_attn, 4),
            kv_gemm_tflop=kv_flop / 1e12, kv_gemm_tflops=round(kv_flop / t_kv / 1e9, 1),
            gather_gbytes=gather_bytes / 1e9, gather_gbps=round(gather_bytes / t_gather / 1e6, 1),
            attn_gbytes=attn_bytes / 1e9, attn_gbps=round(attn_bytes / t_attn / 1e6, 1))
    # the nine CP blocks of one CFG step: 64^2 (x2), 32^2 (x2), 16^2 (x2), 8^2 (x3)
    per_step = {64: 2, 32: 2, 16: 2, 8: 3}
    kv_total = sum(levels[f"{h}x{h}"]["kv_gemm_tflop"] * n for h, n in per_step.items())
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    print(json.dumps(dict(
        metric="MVDiffusion denoise steps/s (8 views 512^2, CFG pair, SD-2 widths, eager launches)",
        value=round(1000.0 / step_ms, 3), unit="steps/s", ms_per_step=round(step_ms, 2), dtype=args.dtype,
        steps=args.steps, warmup=args.warmup, gpu=smi, cp_levels=levels, cp_kv_gemm_tflop_per_step=round(kv_total, 3))))


if __name__ == "__main__":
    main()
