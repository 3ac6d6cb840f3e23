"""Same-call A/B of two builds of the library on the tap-GEMM shapes of a C2 step, then on the step itself.

    python scripts/gemm_occupancy_ab.py LIB_A LIB_B [--rounds 3] [--shapes NAME ...] [--skip-bench] [--list]

LIB_A / LIB_B are two libpanfusion_b200.so of the same C ABI (PF_LIB_PATH selects one per child process). The builds
alternate A, B, A, B, ... for `--rounds` rounds, each in a fresh process:

1. the shapes of SHAPES below, one tap-GEMM each: 20 launches captured in one CUDA graph, rotating over buffer sets
   larger than the 50 MB L2, CUDA events around 10 replays (bench.py's micro_rooflines does the same), with the median
   SM clock sampled by nvidia-smi over the child's run;
2. `bench.py --gpus 1 --steps 20 --warmup 5 --skip-cpu --skip-image --dump-outputs <tmp>` for both builds, and a byte
   comparison of the dumped latents of build A and build B.

Each child also hashes (sha256) the first output buffer of every shape after its timed launches, from inputs seeded per
shape; the report says per shape whether build A's output equals build B's byte for byte.

Prints min / median / max per shape and build, the card's name and power limit (read-only nvidia-smi query), and one
JSON line with everything. Exits non-zero without a GPU. Nothing is written inside the repository.
"""
import argparse
import io
import json
import os
import statistics
import subprocess
import sys
import tempfile
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

T64, T32, T16 = 16 * 64 * 64, 16 * 32 * 32, 16 * 16 * 16  # tokens of the 16 view images at the three UNet levels

# name -> kind, sizes. conv: (images, H, W, Cin, Cout), 3x3 pad 1 over the zero-haloed image, halo-dropping row map
# (direct stores). lin: (M, K, N) with the plain row map (the persistent linear GEMM, TMA tile stores); flags:
# ln = LayerNorm consumer, res = 16-bit residual, stats = row-statistics producer, geglu = GEGLU projection
# (256-wide tile).
SHAPES = {
    "conv3x3_320_16x64x64": ("conv", (16, 64, 64, 320, 320)),       # the dominant conv of the step, 160-wide
    "conv3x3_640_16x32x32": ("conv", (16, 32, 32, 640, 640)),
    "conv3x3_1280_16x16x16": ("conv", (16, 16, 16, 1280, 1280)),
    "conv3x3_512_4x64x64": ("conv", (4, 64, 64, 512, 512)),         # 128-wide direct stores (VAE decoder width)
    "conv3x3_320to64_16x64x64": ("conv", (16, 64, 64, 320, 64)),    # 64-wide direct stores (conv_out's padded tile)
    "lin_320_320": ("lin", (T64, 320, 320), ("stats",)),            # proj_in / to_out
    "lin_320_320_ln": ("lin", (T64, 320, 320), ("ln",)),            # cross-attention q behind a folded LayerNorm
    "lin_320_960_ln": ("lin", (T64, 320, 960), ("ln",)),            # fused q|k|v behind a folded LayerNorm
    "lin_1600_320_res_stats": ("lin", (T64, 1600, 320), ("res", "stats")),  # Transformer tail
    "lin_320_2560_geglu": ("lin", (T64, 320, 2560), ("ln", "geglu")),
    "lin_640_640": ("lin", (T32, 640, 640), ("stats",)),
    "lin_320_640_shortcut": ("lin", (T32, 320, 640), ()),          # resnet 1x1 shortcut
    "lin_1280_10240_geglu": ("lin", (T16, 1280, 10240), ("ln", "geglu")),  # GEGLU at the 16x16 level
    "lin_640_1920_ln": ("lin", (T32, 640, 1920), ("ln",)),
    "lin_1024_1024_res": ("lin", (T64 // 4, 1024, 1024), ("res",)),  # 128-wide TMA stores (text-encoder width)
    "lin_320_64": ("lin", (T64, 320, 64), ()),                      # 64-wide TMA stores
}


def shape_flops(name):
    kind, dims = SHAPES[name][0], SHAPES[name][1]
    if kind == "conv":
        n, h, w, ci, co = dims
        return 2.0 * 9 * ci * co * n * h * w
    m, k, n = dims
    return 2.0 * m * k * n


def nvidia_smi_line():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "nvidia-smi unavailable"


# ------------------------------------------------ child: time the shapes with the library PF_LIB_PATH names
def child(names):
    import hashlib

    import torch
    from bench import ClockSampler
    from panfusion_b200 import _lib, ops
    from panfusion_b200.engine import taps3x3

    if not torch.cuda.is_available():
        sys.exit("gemm_occupancy_ab: no CUDA device")
    dev = torch.device("cuda:0")
    bf = torch.bfloat16

    def timeit(fns, launches=20, reps=10):
        for f in fns:
            f()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for i in range(launches):
                fns[i % len(fns)]()
        g.replay()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            g.replay()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / (reps * launches)

    def n_sets(bytes_per_launch):  # enough buffer sets that a launch never finds its operands in the 50 MB L2
        return max(2, min(8, -(-(128 << 20) // bytes_per_launch)))

    def conv_fns(n, h, w, ci, co):
        hp, wp = h + 2, w + 2
        m = n * hp * wp
        wgt = (torch.randn(co, 9 * ci, device=dev) * 0.02).to(bf)
        sets = n_sets(m * ci * 2 + n * h * w * co * 2)
        As = [torch.randn(m, ci, device=dev).to(bf) for _ in range(sets)]
        outs = [torch.empty(n * h * w, co, dtype=bf, device=dev) for _ in range(sets)]
        return [(lambda a=a, o=o: ops.gemm_taps(a, wgt, o, M=m, Kc=ci, taps=taps3x3(wp), image_map=(hp, wp, 1, 1, h, w)))
                for a, o in zip(As, outs)], outs[0]

    def lin_fns(m, k, n, flags):
        geglu = "geglu" in flags
        n_out = n // 2 if geglu else n
        wgt = (torch.randn(n, k, device=dev) * 0.02).to(bf)
        bias = torch.randn(n, device=dev) * 0.1
        sets = n_sets(m * k * 2 + m * n_out * 2 * (2 if "res" in flags else 1))
        As = [torch.randn(m, k, device=dev).to(bf) for _ in range(sets)]
        outs = [torch.empty(m, n_out, dtype=bf, device=dev) for _ in range(sets)]
        kw = dict(M=m, Kc=k, bias=bias)
        if geglu:
            kw["act"] = _lib.PF_ACT_GEGLU
        if "ln" in flags:  # statistics as a producer of this K would have written them: (sum, sum of squares) per slot
            slots = 2 * (k // ops.pick_block_n(k))
            x = As[0].float()
            st = torch.stack([x.sum(1) / slots, (x * x).sum(1) / slots], 1)[:, None, :].repeat(1, slots, 1).contiguous()
            kw["ln"] = (st, wgt.float().sum(1).contiguous(), 1e-5)
        if "stats" in flags:
            kw["row_stats"] = True
        ress = [torch.randn(m, n_out, device=dev).to(bf) for _ in range(sets)] if "res" in flags else [None] * sets
        return [(lambda a=a, o=o, r=r: ops.gemm_taps(a, wgt, o, residual=r, **kw)) for a, o, r in zip(As, outs, ress)], outs[0]

    res, digest = {}, {}
    with ClockSampler(0) as clk:
        for name in names:
            kind, dims = SHAPES[name][0], SHAPES[name][1]
            torch.manual_seed(0)  # the same operands for both builds
            fns, out0 = conv_fns(*dims) if kind == "conv" else lin_fns(*dims, SHAPES[name][2])
            res[name] = round(timeit(fns) * 1e3, 2)  # us per launch
            torch.cuda.synchronize()
            digest[name] = hashlib.sha256(out0.view(torch.uint8).cpu().numpy().tobytes()).hexdigest()
            del fns, out0
            torch.cuda.empty_cache()
    print(json.dumps(dict(us=res, sha256=digest, sm_mhz=clk.summary()["sm_mhz"])))


# ------------------------------------------------ parent: alternate the two builds
def run_child(lib, argv, what):
    env = dict(os.environ, PF_LIB_PATH=str(lib))
    r = subprocess.run([sys.executable, *argv], env=env, cwd=str(ROOT), capture_output=True, text=True)
    if r.returncode != 0:
        sys.exit(f"gemm_occupancy_ab: {what} failed with {lib}:\n{r.stdout[-2000:]}\n{r.stderr[-4000:]}")
    return json.loads(r.stdout.strip().splitlines()[-1])


def mmm(v):
    return f"{min(v):8.2f} {statistics.median(v):8.2f} {max(v):8.2f}"


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("libs", nargs="*", metavar="LIB", help="two builds of libpanfusion_b200.so: A (before) and B (after)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--shapes", nargs="+", default=list(SHAPES), choices=list(SHAPES))
    ap.add_argument("--skip-bench", action="store_true", help="time the shapes only")
    ap.add_argument("--list", action="store_true", help="print the shapes and their FLOPs, touch no device")
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        return child(args.shapes)
    if args.list:
        for n in args.shapes:
            print(f"{n:28s} {SHAPES[n][0]:4s} {SHAPES[n][1]} {' '.join(SHAPES[n][2]) if len(SHAPES[n]) > 2 else '':12s} "
                  f"{shape_flops(n) / 1e9:8.1f} GFLOP")
        return
    if len(args.libs) != 2:
        ap.error("two library paths are needed")
    libs = [Path(p).resolve() for p in args.libs]
    for p in libs:
        if not p.is_file():
            sys.exit(f"gemm_occupancy_ab: no such library: {p}")
    if args.rounds < 3:
        ap.error("--rounds must be at least 3: a difference is judged against the spread")
    import torch
    if not torch.cuda.is_available():
        sys.exit("gemm_occupancy_ab: no CUDA device; timings come from a GPU or not at all")
    smi = nvidia_smi_line()
    print(f"gpu: {torch.cuda.get_device_name(0)} | name, power limit, max SM clock: {smi}")
    print(f"A = {libs[0]}\nB = {libs[1]}")

    me = str(Path(__file__).resolve())
    us = [{n: [] for n in args.shapes} for _ in libs]
    mhz = [[], []]
    digests = [[], []]
    for _ in range(args.rounds):
        for i, lib in enumerate(libs):
            r = run_child(lib, [me, "--child", "--shapes", *args.shapes], "shape timing")
            for n, v in r["us"].items():
                us[i][n].append(v)
            mhz[i].append(r["sm_mhz"])
            digests[i].append(r["sha256"])
    print(f"\nus per launch, min / median / max over {args.rounds} alternated processes "
          f"(median SM clock A {mhz[0]} MHz, B {mhz[1]} MHz)")
    print(f"{'shape':28s} {'A min':>8s} {'A med':>8s} {'A max':>8s}   {'B min':>8s} {'B med':>8s} {'B max':>8s}   B/A time"
          f"   B TFLOP/s   A == B output")
    same = {}
    for n in args.shapes:
        ma, mb = statistics.median(us[0][n]), statistics.median(us[1][n])
        # each build must repeat itself; then the two builds' outputs are compared byte for byte
        rep = all(d[n] == digests[i][0][n] for i in range(2) for d in digests[i])
        same[n] = "yes" if rep and digests[0][0][n] == digests[1][0][n] else ("NO" if rep else "NOT REPEATABLE")
        print(f"{n:28s} {mmm(us[0][n])}   {mmm(us[1][n])}   {mb / ma:8.3f}   {shape_flops(n) / mb / 1e6:8.1f}   "
              f"{same[n]:>13s}")
    out = dict(gpu=torch.cuda.get_device_name(0), smi=smi, libs=[str(p) for p in libs], us=us, sm_mhz=mhz,
               outputs_identical=same)

    if not args.skip_bench:
        steps = [[], []]
        clocks = [[], []]
        dumps = [[], []]
        with tempfile.TemporaryDirectory(prefix="gemm_ab_") as tmp:
            for rnd in range(args.rounds):
                for i, lib in enumerate(libs):
                    d = Path(tmp) / f"{'AB'[i]}{rnd}"
                    r = run_child(lib, [str(ROOT / "bench.py"), "--gpus", "1", "--steps", "20", "--warmup", "5",
                                        "--skip-cpu", "--skip-image", "--dump-outputs", str(d)], "bench.py")
                    steps[i].append(r["value"])
                    clocks[i].append(r["clocks"]["sm_mhz"])
                    dumps[i].append({f.name: f.read_bytes() for f in sorted(d.glob("*.npy"))})
            same_build = all(d == dumps[i][0] for i in range(2) for d in dumps[i])
            same_ab = dumps[0][0] == dumps[1][0] and len(dumps[0][0]) > 0
            # how far B's latents lie from A's, relative to max|latent| of A
            rel = {}
            for f, ba in dumps[0][0].items():
                if f in dumps[1][0]:
                    xa = np.load(io.BytesIO(ba)).astype(np.float64)
                    xb = np.load(io.BytesIO(dumps[1][0][f])).astype(np.float64)
                    d = np.abs(xb - xa) / max(np.abs(xa).max(), 1e-30)
                    rel[f] = dict(max=float(d.max()), mean=float(d.mean()))
        print(f"\nbench.py steps/s (C2, 1 GPU, 20 steps): A {mmm(steps[0])} (SM MHz {clocks[0]})\n"
              f"{'':39s}B {mmm(steps[1])} (SM MHz {clocks[1]})")
        for f, r in rel.items():
            print(f"--dump-outputs {f}: |B - A| / max|A| max {r['max']:.3g}, mean {r['mean']:.3g}")
        gain = statistics.median(steps[1]) / statistics.median(steps[0]) - 1
        apart = min(steps[1]) > max(steps[0]) or max(steps[1]) < min(steps[0])
        print(f"B vs A: {gain * 100:+.2f} % median, ranges {'do not overlap' if apart else 'OVERLAP'}; "
              f"--dump-outputs: each build identical across its runs: {same_build}; A and B byte-identical: {same_ab}")
        out.update(steps_per_s=steps, bench_sm_mhz=clocks, dumps_identical=same_ab, dumps_repeatable=same_build,
                   dumps_rel_diff=rel)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
