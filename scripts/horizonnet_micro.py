"""HorizonNet layout network timing on one GPU: CUDA events over the whole forward at B = 1, 8, 32 and per stage
(encoder, height stage, each LSTM layer's projection GEMM and recurrence, head) at each B, with FLOP/s from the
shape-derived counts. Prints the card's name and power limit and the LSTM's cluster occupancy in the same run.

    python scripts/horizonnet_micro.py [--iters 10]
"""
from __future__ import annotations

import argparse
import ctypes as C
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

import torch  # noqa: E402

from oracle import horizonnet as oh  # noqa: E402
from panfusion_b200 import _lib, horizonnet  # noqa: E402

# GFLOP per image, from the layer shapes (2 x MACs)
GFLOP = {"encoder": 86.0, "height": 51.0, "lstm_gemm": 4.3 / 2, "lstm_rec": 2.1 / 2, "head": 2 * 256 * 1024 * 12e-9}


def card() -> str:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def timed(fn, iters):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    print(f"card: {card()}")
    n = C.c_int(0)
    _lib.check(_lib.lib().pf_lstm_bidir_clusters(C.byref(n)))
    print(f"pf_lstm_bidir: cudaOccupancyMaxActiveClusters = {n.value} (16 CTAs, one per direction)")
    net = horizonnet.HorizonNetModule(oh.synth_state(), dev)
    net._l, net._st = _lib.lib(), _lib.stream_ptr()
    for B in (1, 8, 32):
        x = torch.rand(B, 3, 512, 1024, device=dev)
        ms = timed(lambda: net(x), args.iters)
        tot = sum(GFLOP[k] * (2 if k.startswith("lstm") else 1) for k in GFLOP) * B
        print(f"B={B:2d} forward {ms:8.2f} ms  {ms / B:7.2f} ms/image  {tot / ms:6.1f} TFLOP/s (shape-derived)")
        if B > horizonnet.MAX_BATCH:
            continue
        # per stage, on the intermediates of one forward
        p = torch.empty(B, 512, 1024, 16, device=dev, dtype=torch.float16)
        _lib.check(net._l.pf_hnet_prep(C.c_void_p(x.data_ptr()), B, 3, 512, 1024, C.c_void_p(p.data_ptr()),
                                       C.c_void_p(net._st)))
        feats = net._encoder(p)
        y = net._lstm_input(feats)
        y1 = net._lstm(y, 0, B)
        y2 = net._lstm(y1, 1, B)
        stages = {"encoder": lambda: net._encoder(p), "height": lambda: net._lstm_input(feats)}
        for layer, inp in ((0, y), (1, y1)):
            xproj = torch.empty(256 * B, 4096, device=dev)
            out = torch.empty(256 * B, 1024, device=dev, dtype=torch.float16)

            def gemm(inp=inp, layer=layer, xproj=xproj):
                from panfusion_b200 import ops
                ops.gemm_taps(inp, getattr(net, f"wih{layer}"), xproj, M=256 * B, Kc=1024,
                              bias=getattr(net, f"bias{layer}"), block_n=128, k_splits=1)

            def rec(layer=layer, xproj=xproj, out=out):
                _lib.check(net._l.pf_lstm_bidir(C.c_void_p(xproj.data_ptr()),
                                                C.c_void_p(getattr(net, f"whh{layer}").data_ptr()), 256, B,
                                                C.c_void_p(out.data_ptr()), C.c_void_p(net._st)))

            gemm()
            stages[f"lstm{layer + 1}_gemm"], stages[f"lstm{layer + 1}_rec"] = gemm, rec
        stages["head"] = lambda: net._head(y2, B)
        for name, fn in stages.items():
            t = timed(fn, args.iters)
            key = name.split("_", 1)[-1] if name.startswith("lstm") else name
            gf = GFLOP["lstm_" + key] if name.startswith("lstm") else GFLOP[name]
            extra = f"  {t * 1e3 / 256:6.2f} us/step" if name.endswith("rec") else ""
            print(f"   {name:11s} {t:8.3f} ms  {gf * B / t:7.2f} TFLOP/s{extra}")


if __name__ == "__main__":
    main()
