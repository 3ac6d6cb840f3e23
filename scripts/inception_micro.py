"""FID InceptionV3 on one GPU: images/s at batch 1, 16 and 64 for 299x299 and 512x1024 uint8 inputs; per-layer kernel
times (CUDA events) and TFLOP/s counted from the layer table at batch 64; compute() time for FID at d = 2048 and for
IS; and, with --faed-tree-before, FAED's encoder (faed_micro.py's 512x1024 batch-8 figure) from a source tree (its
panfusion_b200 package with its library built, and oracle/) from before the convolution core was shared, alternated
with this tree in separate processes. Seeded synthetic weights.
Every time is the median of --reps CUDA-event windows with its min and max. The card's name and power limit are read
in the same run."""
import argparse
import ctypes as C
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from oracle import inception as oi  # noqa: E402
from panfusion_b200 import _lib, inception  # noqa: E402

PEAK_FP16 = 989e12  # H100 SXM data sheet, dense fp16 tensor core


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


def layer_table():
    """(name, Cin, Cout, kh, kw, s, ph, pw, H_in, Ho, Wo) in forward order at 299x299, and the MACs per image (3 real
    input channels for the first layer, plus the fc)."""
    stem = {"Conv2d_1a_3x3": 299, "Conv2d_2a_3x3": 149, "Conv2d_2b_3x3": 147, "Conv2d_3b_1x1": 73,
            "Conv2d_4a_3x3": 73}
    block = {"Mixed_5b": 35, "Mixed_5c": 35, "Mixed_5d": 35, "Mixed_6a": 35, "Mixed_6b": 17, "Mixed_6c": 17,
             "Mixed_6d": 17, "Mixed_6e": 17, "Mixed_7a": 17, "Mixed_7b": 8, "Mixed_7c": 8}
    rows, macs = [], 0
    for name, (cin, cout, kh, kw, s, ph, pw) in inception.CONVS.items():
        h = stem[name] if name in stem else block[name.split(".")[0]]
        ho, wo = (h + 2 * ph - kh) // s + 1, (h + 2 * pw - kw) // s + 1
        macs += ho * wo * cout * (3 if cin == 3 else cin) * kh * kw
        rows.append((name, cin, cout, kh, kw, s, ph, pw, h, ho, wo))
    return rows, macs + 2048 * 1008


FAED_TIMING = """
import json, statistics, sys
sys.path.insert(0, sys.argv[1])
import torch
from oracle import faed as of
from panfusion_b200 import faed
enc = faed.FAEDEncoder(of.synth_state(), "cuda:0")
x = of.images((8, 3, 512, 1024), "real", 8).to("cuda:0")
for _ in range(2):
    enc(x)
torch.cuda.synchronize()
out = []
for _ in range(int(sys.argv[3])):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(int(sys.argv[2])):
        enc(x)
    b.record()
    b.synchronize()
    out.append(a.elapsed_time(b) / int(sys.argv[2]) / 1e3)
print(json.dumps(statistics.median(out)))
"""


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--faed-tree-before", help="source tree (library built) from before the shared conv core")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "inception_micro needs a CUDA device"
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    rows, macs = layer_table()
    flops = 2 * macs
    res = {"gpu": q, "gmac_per_image": macs / 1e9, "images_per_s": {}, "layers": [], "compute": {}}
    print(f"GPU: {q}; {macs / 1e9:.2f} GMAC per image counted from the layer table")
    net = inception.InceptionV3(oi.synth_state(), dev)
    for hw in ((299, 299), (512, 1024)):
        for B in (1, 16, 64):
            x = oi.images(B, hw, "real", B).to(dev)
            t = timed(lambda: net(x), args.iters, args.reps)
            key = f"{hw[0]}x{hw[1]}_b{B}"
            res["images_per_s"][key] = {"s": t, "images_per_s": B / t[0], "tflops": B * flops / t[0] / 1e12}
            print(f"{key:>14}: {spread(t)}, {B / t[0]:8.1f} images/s, {B * flops / t[0] / 1e12:6.1f} TFLOP/s "
                  f"({B * flops / t[0] / PEAK_FP16:.3f} of the fp16 data-sheet peak)")
    B = 64
    l, st = _lib.lib(), _lib.stream_ptr()
    for name, cin, cout, kh, kw, s, ph, pw, h, ho, wo in rows:
        cin_p = 16 if cin == 3 else cin
        x = torch.randn(B, h, h, cin_p, device=dev).half()
        y = torch.empty(B, ho, wo, cout, device=dev, dtype=torch.float16)
        k = name.replace(".", "_")

        def run(x=x, y=y, k=k, cin_p=cin_p, cout=cout, kh=kh, kw=kw, s=s, ph=ph, pw=pw, h=h):
            _lib.check(l.pf_conv2d_nhwc(C.c_void_p(x.data_ptr()), B, h, h, cin_p,
                                        C.c_void_p(getattr(net, f"{k}_w").data_ptr()),
                                        C.c_void_p(getattr(net, f"{k}_b").data_ptr()), cout, kh, kw, s, ph, pw, 1,
                                        C.c_void_p(y.data_ptr()), _lib.PF_F16, cout, 0, C.c_void_p(st)))
        t = timed(run, args.iters, args.reps)
        f = 2 * B * ho * wo * cout * (3 if cin == 3 else cin) * kh * kw
        res["layers"].append({"layer": name, "shape": [cin, cout, kh, kw, s, ph, pw, h], "s": t,
                              "tflops": f / t[0] / 1e12})
        print(f"{name:28s} {cin:4d}->{cout:4d} {kh}x{kw} s{s} @{h:3d}: {spread(t)} {f / t[0] / 1e12:6.1f} TFLOP/s")
    total = sum(r["s"][0] for r in res["layers"])
    print(f"sum of conv layers at batch {B}: {total * 1e3:.2f} ms, {B * flops / total / 1e12:.1f} TFLOP/s")
    res["conv_sum_s_b64"] = total
    # compute(): FID at d = 2048 (n = 4096 random features per side) and IS (n = 5000 logits, 10 splits)
    g = torch.Generator(device=dev).manual_seed(0)
    m = inception.FrechetInceptionDistance(inception=net, device=dev)
    for side in ("real", "fake"):
        z = torch.randn(4096, 2048, device=dev, generator=g).relu() + (0.05 if side == "fake" else 0.0)
        _lib.check(l.pf_faed_stats(C.c_void_p(z.data_ptr()), 4096, 2048,
                                   C.c_void_p(getattr(m, f"{side}_features_sum").data_ptr()),
                                   C.c_void_p(getattr(m, f"{side}_features_cov_sum").data_ptr()), C.c_void_p(st)))
        getattr(m, f"{side}_features_num_samples").add_(4096)
    ts = []
    for _ in range(3):
        t0 = time.perf_counter()
        v = m.compute()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    res["compute"]["fid_d2048_n4096"] = {"s_median_min_max": (statistics.median(ts), min(ts), max(ts)),
                                         "fid": float(v)}
    print(f"FID compute() d=2048 n=4096/side: {statistics.median(ts) * 1e3:.0f} ms (min {min(ts) * 1e3:.0f}, "
          f"max {max(ts) * 1e3:.0f})")
    s = inception.InceptionScore(inception=net, device=dev)
    s.features = [3 * torch.randn(5000, 1008, device=dev, generator=g)]
    t = timed(lambda: s.compute(), 3, args.reps)
    res["compute"]["is_n5000_splits10"] = {"s": t}
    print(f"IS compute() n=5000 splits=10: {spread(t)}")
    if args.faed_tree_before:
        ab = {"before": [], "after": []}
        for _ in range(3):
            for tag, tree in (("before", Path(args.faed_tree_before).resolve()), ("after", ROOT)):
                r = subprocess.run([sys.executable, "-c", FAED_TIMING, str(tree), str(args.iters), str(args.reps)],
                                   capture_output=True, text=True, check=True)
                ab[tag].append(json.loads(r.stdout.strip().splitlines()[-1]))
        res["faed_encoder_b8_512x1024_s"] = ab
        for tag in ("before", "after"):
            v = ab[tag]
            print(f"FAED encoder batch 8 at 512x1024, {tag} the shared core: "
                  f"{', '.join(f'{x * 1e3:.2f}' for x in v)} ms ({8 / statistics.median(v):.1f} panoramas/s median)")
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
