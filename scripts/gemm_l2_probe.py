"""Is the tap-GEMM's main loop bound by operand traffic out of L2? One GEMM shape at every tile width.

    python scripts/gemm_l2_probe.py

Shape: M = 65 536 rows, K = 2 880 as 9 taps x 320 channels (a 3x3 convolution's offsets over a 66-pixel row pitch),
N = 1 280, bf16, direct-store epilogue at every width (so only the tile width changes). Each CTA computes one
128 x block_n tile. The taps of one kernel row lie within 2 rows of each other, so they share one A window of
128 + 8 rows (17 KB) per 64-channel slab, and every tap adds a block_n x 128 B B box: the fill per tile is
windows * 17 KB + slabs * block_n * 128 B, with 3 windows and 9 slabs per 64 channels. The script prints TFLOP/s,
FLOP per byte of that fill, and the fill rate (fill per tile * tiles / time). Every filled byte is read from L2. If
TFLOP/s rises with FLOP/B while the fill rate stays roughly flat, the main loop is L2-bound. For a build that loads a
16 KB A box per tap (the tap-GEMM before A windows), the "slab" columns give the same accounting for
(16 KB + block_n * 128 B) per slab.

Timing follows bench.py's micro_rooflines: 20 launches captured in one CUDA graph, rotating over buffer sets larger
than L2, CUDA events around 25 replays, with the median SM clock sampled by nvidia-smi over the same window.
"""
import json
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import torch  # noqa: E402

from bench import ClockSampler  # noqa: E402
from panfusion_b200 import ops  # noqa: E402

M, N, CI, TAPS, WP = 65536, 1280, 320, 9, 66


def timeit(fns, launches=20, reps=5):
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


def main():
    dev = torch.device("cuda:0")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(f"gpu: {torch.cuda.get_device_name(dev)} | nvidia-smi: {smi}")
    taps = [dy * WP + dx for dy in range(3) for dx in range(3)]
    a_rows = M + taps[-1]
    # 3 x (42 MB A + 168 MB out): consecutive launches never find their operands in the 50 MB L2
    As = [torch.randn(a_rows, CI, device=dev).bfloat16() for _ in range(3)]
    B = (torch.randn(N, CI * TAPS, device=dev) * 0.02).bfloat16()
    outs = [torch.empty(M, N, dtype=torch.bfloat16, device=dev) for _ in range(3)]
    flops = 2.0 * M * N * CI * TAPS
    slabs = CI // 64 * TAPS
    windows = CI // 64 * 3  # one per kernel row and channel slab
    m_tiles = (M + 127) // 128
    rows = []
    for bn in (64, 128, 160):
        fns = [(lambda a=a, o=o: ops.gemm_taps(a, B, o, M=M, Kc=CI, taps=taps, block_n=bn,
                                               image_map=(1, M, 0, 0, 1, M))) for a, o in zip(As, outs)]
        with ClockSampler(dev.index or 0) as clk:
            ms = timeit(fns, reps=25)
        tiles = m_tiles * (N // bn)
        fill = (windows * (128 + 8) * 128 + slabs * bn * 128) * tiles
        fill_slab = (16384 + bn * 128) * slabs * tiles
        r = dict(block_n=bn, ms=round(ms, 4), tflops=round(flops / ms / 1e9, 1),
                 flop_per_byte=round(flops / fill, 1), fill_tbs=round(fill / ms / 1e9, 2),
                 slab_flop_per_byte=round(flops / fill_slab, 1), slab_fill_tbs=round(fill_slab / ms / 1e9, 2),
                 sm_mhz=clk.summary()["sm_mhz"])
        rows.append(r)
        print(f"block_n={bn:3d}: {ms * 1e3:7.1f} us  {r['tflops']:6.1f} TFLOP/s  windows: {r['flop_per_byte']:5.1f} FLOP/B "
              f"{r['fill_tbs']:5.2f} TB/s L2->SMEM fill  (slab: {r['slab_flop_per_byte']:5.1f} FLOP/B "
              f"{r['slab_fill_tbs']:5.2f} TB/s)  median SM clock {r['sm_mhz']} MHz")
    # one spot check of the result, so that a fast but wrong kernel cannot pass for a fast one
    ops.gemm_taps(As[0], B, outs[0], M=M, Kc=CI, taps=taps, block_n=160, image_map=(1, M, 0, 0, 1, M))
    rs = torch.arange(0, M, 4099, device=dev)
    ref = sum(As[0][rs + t].float() @ B[:, i * CI:(i + 1) * CI].float().T for i, t in enumerate(taps))
    err = ((outs[0][rs].float() - ref).abs().max() / ref.abs().max()).item()
    print(f"spot check vs fp32 torch: max err {err:.2e} of max|ref|")
    assert err < 1e-2
    print(json.dumps(dict(gpu=torch.cuda.get_device_name(dev), smi=smi, shape=dict(M=M, N=N, K=CI * TAPS), rows=rows)))


if __name__ == "__main__":
    main()
