"""Where the time of one denoise step goes: kernel time per kernel family in one eager C2 step.

    python scripts/step_breakdown.py [--workload c2] [--json OUT.json]

Builds the model, inputs and sampler as `bench.py --gpus 1` does, runs 4 eager warm-up steps (camera tables, weights,
allocator), then profiles exactly one eager step with torch.profiler (CUDA activities only) and sums the device time
of every kernel by family. The tap-GEMM is split into classes by its template arguments
<BLOCK_N, STAGES, CTAS, BF16>:
  conv (direct store)   two CTAs per SM: the convolutions (and fp32-output or row-bias GEMMs)
  split-K partials      one CTA per SM: the deep-K convolutions of small images
The persistent linear GEMM, gemm_linear_kernel<BLOCK_N, STAGES, GEGLU, BF16>, which runs the one-tap, plain-row-map
calls with 16-bit output (the linear layers and 1x1 shortcuts), is split by width:
  linear GEMM           the 64-, 128- and 160-wide tiles
  linear GEMM GEGLU     the 256-wide GEGLU tile
The sum is kernel time only: launch gaps, which a CUDA-graph step of bench.py mostly removes, are not counted.
Profile in a run of its own; take step rates from bench.py. Prints the card's name and power limit.
"""
import argparse
import json
import re
import subprocess
import sys
from collections import defaultdict
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import torch  # noqa: E402

import bench  # noqa: E402

GEMM_RE = re.compile(r"gemm_taps_kernel<(\d+),\s*(\d+),\s*(\d+),\s*(\w+)>")
LINEAR_RE = re.compile(r"gemm_linear_kernel<(\d+),\s*(\d+),\s*(\w+),\s*(\w+)>")


def family(name: str) -> str:
    m = LINEAR_RE.search(name)
    if m:
        return "linear GEMM GEGLU 256-wide" if m.group(3) == "true" else "linear GEMM 64/128/160-wide"
    m = GEMM_RE.search(name)
    if m:
        return "tap-GEMM conv (direct store)" if int(m.group(3)) == 2 else "tap-GEMM split-K partials"
    base = name.split("(")[0]
    base = re.sub(r"^void\s+", "", base)
    base = re.sub(r"<.*", "", base)
    return base.split("::")[-1] if "pf::" in name or base.startswith("pf") else f"other: {base[:60]}"


def build_sampler(workload: str, dev):
    from panfusion_b200 import _lib, geometry, sd2_unet
    from panfusion_b200.mvgen import MultiViewBaseModel
    from panfusion_b200.sampler import PanFusionSampler

    _lib.check(_lib.lib().pf_check_device())
    wl = bench.WORKLOADS[workload]
    dtype = torch.bfloat16
    unet = sd2_unet.build_synthetic(seed=1, device=dev)
    pano_unet = sd2_unet.build_synthetic(seed=2, device=dev)
    torch.manual_seed(3)
    pano_cn = sd2_unet.build_synthetic_controlnet(seed=5, device=dev) if wl.get("layout_cond") else None
    model = MultiViewBaseModel(unet, pano_unet, pano_cn=pano_cn, compute_dtype=dtype).to(dev).eval()
    g = torch.Generator(device=dev).manual_seed(4)
    with torch.no_grad():
        for name, p in sorted(model.named_parameters()):
            if "cp_blocks" in name and float(p.abs().sum()) == 0.0:
                p.copy_(torch.randn(p.shape, generator=g, device=dev) * 0.02)
    model.prepare(dev, dtype)
    sampler = PanFusionSampler(model, use_cuda_graph=False)
    inp = bench.synthetic_inputs(wl, 1024, dev, sampler)
    pano = inp["pano"].to(dev)
    cams_flat = {k: v.flatten(0, 1) for k, v in inp["cams"].items()}
    lat = geometry.e2p(pano.expand(-1, wl["m"], -1, -1, -1).flatten(0, 1).contiguous(), cams_flat["FoV"],
                       cams_flat["theta"], cams_flat["phi"], wl["pers_hw"], mode="nearest")[None]
    cond = inp["pano_layout_cond"].to(dev) if "pano_layout_cond" in inp else None
    sampler.start(lat, pano, inp["prompt"].to(dev), inp["pano_prompt"].to(dev), inp["cams"], pano_layout_cond=cond)
    return sampler


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--workload", default="c2", choices=list(bench.WORKLOADS))
    ap.add_argument("--json", default=None, help="also write the table as JSON to this path")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("step_breakdown: no CUDA device; kernel times come from a GPU or not at all")
    dev = torch.device("cuda:0")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(f"gpu: {torch.cuda.get_device_name(dev)} | name, power limit, max SM clock: {smi}")
    sampler = build_sampler(args.workload, dev)
    for i in range(4):
        sampler.step(i)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        sampler.step(4)
        torch.cuda.synchronize()
    us, calls = defaultdict(float), defaultdict(int)
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        if "memcpy" in e.name.lower() or "memset" in e.name.lower():
            fam = "memcpy / memset"
        else:
            fam = family(e.name)
        us[fam] += e.time_range.elapsed_us()
        calls[fam] += 1
    total = sum(us.values())
    print(f"\none eager {args.workload} step: {total / 1e3:.2f} ms of kernel time, {sum(calls.values())} kernels")
    print(f"{'family':40s} {'calls':>6s} {'ms':>9s} {'share':>7s}")
    rows = sorted(us, key=lambda k: -us[k])
    for k in rows:
        print(f"{k:40s} {calls[k]:6d} {us[k] / 1e3:9.3f} {100 * us[k] / total:6.1f} %")
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps(dict(gpu=torch.cuda.get_device_name(dev), smi=smi,
                                                   total_us=total, us=us, calls=calls), indent=1))


if __name__ == "__main__":
    main()
