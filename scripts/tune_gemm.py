"""Measure, on the GPU, the best tap-GEMM tile width (block_n) for every GEMM shape of a C2 denoise step and write
the table that panfusion_b200/ops.py reads from panfusion_b200/gemm_tuning.json when it exists.
Usage: python scripts/tune_gemm.py [out.json] [workload:layout,...]   e.g.  c2:1x1,c2:2x1,c2:2x2,c2:2x4,c5:1x1
(layouts other than 1x1 are the rank-local shapes of the sharded step, collected with scripts/rank_emulate.py)"""
import collections
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import torch  # noqa: E402

sys.path.insert(0, str(ROOT / "scripts"))
from panfusion_b200 import ops  # noqa: E402


def collect(workload, layout, dev, dt):
    """GEMM shapes of one (rank-local) denoise step of `workload` under `layout` = (batch_shards, view_shards)."""
    from rank_emulate import build
    model, sampler = build(workload, dev, dt, layout, graph=False, overlap=False)
    sampler.step(0)
    ops.GEMM_LOG = []
    sampler.step(1)
    torch.cuda.synchronize()
    shapes = collections.Counter(ops.GEMM_LOG)
    ops.GEMM_LOG = None
    del model, sampler
    torch.cuda.empty_cache()
    return shapes


def main():
    out_path = Path(sys.argv[1] if len(sys.argv) > 1 else ROOT / "gpurun_out" / "gemm_tuning.json")
    # workload:layout list; the single-GPU C2 step first (its counts weight the printed totals)
    spec = sys.argv[2] if len(sys.argv) > 2 else "c2:1x1"
    dev = torch.device("cuda:0")
    dt = torch.bfloat16
    shapes = collections.Counter()
    for item in spec.split(","):
        wl, lay = item.split(":")
        got = collect(wl, tuple(int(v) for v in lay.split("x")), dev, dt)
        new = [k for k in got if k not in shapes]
        print(f"{item}: {len(got)} distinct GEMM shapes ({len(new)} new), {sum(got.values())} launches", flush=True)
        for k in new:
            shapes[k] = got[k]
    print(f"{len(shapes)} distinct GEMM shapes in total")

    ev = lambda: torch.cuda.Event(enable_timing=True)
    results, table = [], {}
    total_before = total_after = 0.0
    for (M, N, Kc, ntaps, act, mapped, has_res, out_f32), count in sorted(shapes.items()):
        if act == ops.PF_ACT_GEGLU:
            continue
        rows = M + 4096
        A = torch.randn(rows, Kc, device=dev).to(dt)
        B = (torch.randn(N, Kc * ntaps, device=dev) * 0.02).to(dt)
        out = torch.empty(M, N, dtype=torch.float32 if out_f32 else dt, device=dev)
        res = torch.randn(M, N, device=dev).to(dt) if has_res else None
        taps = list(range(ntaps))
        imap = None
        if mapped:  # a plausible halo-dropping map: one image of M rows, everything valid (timing only)
            imap = (1, M, 0, 0, 1, M)
        times = {}
        epi_tma = (not mapped) and (not out_f32)
        for bn in (64, 128, 160, 256):
            if N % bn or (bn == 256 and epi_tma):  # the staged 16-bit epilogue has no 256-wide tile
                continue
            fn = lambda: ops.gemm_taps(A, B, out, M=M, Kc=Kc, taps=taps, residual=res, act=act, block_n=bn,
                                       image_map=imap)
            for _ in range(3):
                fn()
            torch.cuda.synchronize()
            a, b = ev(), ev()
            a.record()
            for _ in range(10):
                fn()
            b.record()
            torch.cuda.synchronize()
            times[bn] = a.elapsed_time(b) / 10 * 1e3  # us
        # what the built-in heuristic picks
        fn = lambda: ops.gemm_taps(A, B, out, M=M, Kc=Kc, taps=taps, residual=res, act=act, block_n=-1, image_map=imap)
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        a, b = ev(), ev()
        a.record()
        for _ in range(10):
            fn()
        b.record()
        torch.cuda.synchronize()
        t_default = a.elapsed_time(b) / 10 * 1e3
        best = min(times, key=times.get)
        if times[best] < 0.97 * t_default:
            table[f"{M},{N},{Kc},{ntaps},{int(mapped)},{int(has_res)}"] = best
        total_before += t_default * count
        total_after += min(times[best], t_default) * count
        fl = 2.0 * M * N * Kc * ntaps
        results.append(dict(M=M, N=N, Kc=Kc, taps=ntaps, mapped=mapped, res=has_res, count=count,
                            us={str(k): round(v, 1) for k, v in times.items()},
                            default_us=round(t_default, 1), best=best,
                            tflops_best=round(fl / times[best] / 1e6, 1)))
        del A, B, out, res
    print(f"sum over a step: default {total_before / 1e3:.2f} ms -> tuned {total_after / 1e3:.2f} ms")
    out_path.parent.mkdir(exist_ok=True)
    out_path.write_text(json.dumps(dict(choice=table, detail=results, default_ms=total_before / 1e3,
                                        tuned_ms=total_after / 1e3), indent=1))
    print(f"wrote {out_path} ({len(table)} overrides)")


if __name__ == "__main__":
    main()
