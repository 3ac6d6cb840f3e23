"""FAED on one GPU: encoder panoramas/s at 512x1024 (batch 1, 8, 16), per-layer time and TFLOP/s at batch 8, and
compute() at pano_height 512 (d = 2048) for a rank-deficient set (n = 16 per side) and a full-rank one (n = 4096 per
side, features with a decaying spectrum), with the Jacobi sweep counts and the error against a symmetric fp64 eigh on
the CPU. Seeded synthetic weights. Every time is the median of --reps CUDA-event windows with its min and max; the SM
clock is sampled every 100 ms by nvidia-smi while the timed work runs and reported as median, min and max."""
import argparse
import ctypes as C
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from oracle import faed as of  # noqa: E402
from panfusion_b200 import _lib, faed  # noqa: E402

PEAK_FP16 = 989e12  # H100 SXM data sheet, dense fp16 tensor core


def layer_flops(L, B, h, w):
    ho, wo = (h + 2 * L["p"] - L["k"]) // L["s"] + 1, (w + 2 * L["p"] - L["k"]) // L["s"] + 1
    cin = 3 if L["cin"] == 16 else L["cin"]
    return 2 * B * ho * wo * L["cout"] * cin * L["k"] ** 2, ho, wo


def timed(fn, iters, reps):
    """median, min, max seconds per call over `reps` windows of `iters` calls"""
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b) / iters / 1e3)
    return statistics.median(out), min(out), max(out)


def spread(t):
    return f"{t[0] * 1e3:8.3f} ms (min {t[1] * 1e3:.3f}, max {t[2] * 1e3:.3f})"


def add_stats(m, side, feats):
    l, st = _lib.lib(), _lib.stream_ptr()
    for f in feats.split(512):
        f = f.contiguous()
        _lib.check(l.pf_faed_stats(C.c_void_p(f.data_ptr()), f.shape[0], f.shape[1],
                                   C.c_void_p(getattr(m, f"{side}_features_sum").data_ptr()),
                                   C.c_void_p(getattr(m, f"{side}_features_cov_sum").data_ptr()), C.c_void_p(st)))
    getattr(m, f"{side}_features_num_samples").add_(feats.shape[0])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "faed_micro needs a CUDA device"
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    enc = faed.FAEDEncoder(of.synth_state(), dev)
    res = {"gpu": q, "encoder": {}, "layers": [], "compute": {}}
    h, w, flops = 512, 1024, 0.0
    for L in enc.layers:
        f, h, w = layer_flops(L, 1, h, w)
        flops += f
    res["gflop_per_pano"] = flops / 1e9
    clock = subprocess.Popen(["nvidia-smi", "-i", "0", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits",
                              "-lms", "100"], stdout=subprocess.PIPE, text=True)
    try:
        t_start = time.time()
        for B in (1, 8, 16):
            x = of.images((B, 3, 512, 1024), "real", B).to(dev)
            t = timed(lambda: enc(x), args.iters, args.reps)
            res["encoder"][B] = {"s": t, "pano_per_s": B / t[0], "tflops": B * flops / t[0] / 1e12,
                                 "share_of_fp16_peak": B * flops / t[0] / PEAK_FP16}
            print(f"batch {B:2d}: {spread(t)}, {B / t[0]:.1f} panoramas/s, {B * flops / t[0] / 1e12:.1f} TFLOP/s")
        B, h, w = 8, 512, 1024
        l, st = _lib.lib(), _lib.stream_ptr()
        x = torch.randn(B, h, w, 16, device=dev).half()
        for i, L in enumerate(enc.layers):
            f, ho, wo = layer_flops(L, B, h, w)
            y = torch.empty(B, ho, wo, L["cout"], device=dev, dtype=torch.float16)
            r = x if L["role"] == "add" else None

            def run(x=x, y=y, i=i, L=L, h=h, w=w, r=r):
                _lib.check(l.pf_conv_circ(C.c_void_p(x.data_ptr()), B, h, w, L["cin"],
                                          C.c_void_p(getattr(enc, f"w{i}").data_ptr()),
                                          C.c_void_p(getattr(enc, f"b{i}").data_ptr()), L["cout"], L["k"], L["s"],
                                          L["p"], int(L["relu"]), C.c_void_p(_lib.ptr(r)), C.c_void_p(y.data_ptr()),
                                          _lib.PF_F16, C.c_void_p(st)))
            t = timed(run, args.iters, args.reps)
            res["layers"].append({"layer": i, "k": L["k"], "s": L["s"], "cin": L["cin"], "cout": L["cout"], "h": h,
                                  "w": w, "s_median_min_max": t, "tflops": f / t[0] / 1e12})
            print(f"layer {i:2d} k{L['k']} s{L['s']} {L['cin']:3d}->{L['cout']:3d} at {h}x{w}: {spread(t)} "
                  f"{f / t[0] / 1e12:6.1f} TFLOP/s")
            x, h, w = y, ho, wo
        g = torch.Generator(device=dev).manual_seed(0)
        basis = torch.linalg.qr(torch.randn(2048, 2048, device=dev, dtype=torch.float64, generator=g))[0]
        decay = torch.exp(-0.01 * torch.arange(2048, device=dev, dtype=torch.float64))  # eigenvalues over 1e-17
        for name, n in (("rank_deficient_n16", 16), ("full_rank_n4096", 4096)):
            m = faed.FrechetAutoEncoderDistance(512, encoder=enc, device=dev)
            for side in ("real", "fake"):
                z = torch.randn(n, 2048, device=dev, dtype=torch.float64, generator=g)
                add_stats(m, side, ((z * decay) @ basis + (0.1 if side == "fake" else 0.0)).float())
            n1, n2 = int(m.real_features_num_samples), int(m.fake_features_num_samples)
            t0 = time.perf_counter()
            v, sweeps = faed.frechet_distance(m.real_features_sum, m.real_features_cov_sum, n1,
                                              m.fake_features_sum, m.fake_features_cov_sum, n2, return_sweeps=True)
            torch.cuda.synchronize()
            t = [time.perf_counter() - t0]
            for _ in range(2):
                t0 = time.perf_counter()
                m.compute()
                torch.cuda.synchronize()
                t.append(time.perf_counter() - t0)
            st_cpu = [(getattr(m, f"{s}_features_sum").cpu(), getattr(m, f"{s}_features_cov_sum").cpu(), k)
                      for s, k in (("real", n1), ("fake", n2))]
            tr = sum(float(of.covariances(*x)[1].trace()) for x in st_cpu)
            e = abs(float(v) - of.faed_eigh(*st_cpu[0], *st_cpu[1])) / tr
            res["compute"][name] = {"s_median_min_max": (statistics.median(t), min(t), max(t)), "sweeps": sweeps,
                                    "faed": float(v), "err_vs_eigh_of_traces": e}
            print(f"compute() d=2048 {name}: {statistics.median(t) * 1e3:.0f} ms (min {min(t) * 1e3:.0f}, max "
                  f"{max(t) * 1e3:.0f}), Jacobi sweeps S1/S2/L1^T L2 {sweeps}, FAED {float(v):.6e}, "
                  f"|d| vs fp64 eigh {e:.1e} of tr S1 + tr S2")
        res["seconds"] = time.time() - t_start
    finally:
        clock.terminate()
        samples = clock.communicate()[0].split()
    mhz = sorted(int(s) for s in samples if s.isdigit())
    res["sm_clock_mhz"] = {"median": statistics.median(mhz), "min": mhz[0], "max": mhz[-1], "samples": len(mhz)}
    print(f"GPU: {q}; SM clock during the run: median {res['sm_clock_mhz']['median']} MHz "
          f"(min {mhz[0]}, max {mhz[-1]}, {len(mhz)} samples)")
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
