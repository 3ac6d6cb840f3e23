"""GPU: the FAED training convolutions through panfusion_b200.faed_train's call paths against fp64 torch autograd on
the same fp16-rounded operands: the forward convolution and the data gradient (pf_faedt_pack's adjoint weights, the
stride-2 phase convolutions and pf_faedt_interleave together) for every layer shape of the autoencoder at W = 64 and
at a W that is not a multiple of the 128-pixel CTA tile. The weight gradients, BatchNorm, the upsample, the loss, Adam
and the layout kernels are held to fp64 contracts in test_gpu_faedt_contract.py. Gates are about 2x the errors
measured on an H100."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from panfusion_b200 import _lib, faed_train as ft

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


@pytest.fixture(scope="module")
def tr(cuda_device):
    t = ft.FAEDTrainer(seed=0, device=cuda_device)
    t._st = _lib.stream_ptr()
    t._inv_n = 1.0  # with the initial scale S = 1 the gradients come out unscaled
    return t


def _layer(tr, cin, cout, k, s, seed):
    """A _Conv whose weight / bias live at the start of the trainer's parameter and gradient buffers."""
    g = torch.Generator().manual_seed(seed)
    w = torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5
    b = torch.randn(cout, generator=g) * 0.1
    off = {"t.conv2d.weight": 0, "t.conv2d.bias": w.numel()}
    cv = ft._Conv("t", cin, cout, k, s, 1 if s == 2 else k // 2, off, tr.device, cin != 3)
    tr.params[: w.numel()].copy_(w.reshape(-1))
    tr.params[w.numel(): w.numel() + cout].copy_(b)
    tr.out_bias[:3].copy_(b[:3] if cout == 3 else torch.zeros(3))
    _lib.check(_lib.lib().pf_faedt_pack(ft._vp(tr.params), cout, cin, k, s, ft._vp(cv.fwd), cv.x_c, cv.cw,
                                        ft._vp(cv.dg), cv.dy_c, cin, C.c_void_p(tr._st)))
    return cv, w.to(tr.device).double(), b.to(tr.device).double()


def _nhwc(t, c_store):
    """[B, C, H, W] -> fp16 [B, H, W, c_store] with zero channels past C."""
    out = torch.zeros(t.shape[0], t.shape[2], t.shape[3], c_store, device=t.device, dtype=torch.float16)
    out[..., : t.shape[1]] = t.permute(0, 2, 3, 1).half()
    return out


SHAPES = [(3, 32, 9, 1), (32, 32, 9, 1), (32, 64, 4, 2), (64, 64, 7, 1), (64, 128, 4, 2), (128, 128, 5, 1),
          (128, 128, 4, 2), (128, 128, 3, 1), (128, 64, 3, 1), (64, 32, 3, 1), (32, 3, 9, 1)]


@pytest.mark.parametrize("H,W", [(16, 64), (12, 40)])
@pytest.mark.parametrize("cin,cout,k,s", SHAPES)
def test_conv_forward_dgrad_wgrad(tr, cin, cout, k, s, H, W):
    B = 2
    cv, w, b = _layer(tr, cin, cout, k, s, seed=cin * 1000 + cout * 10 + k)
    g = torch.Generator().manual_seed(7)
    x = _nhwc(torch.randn(B, cin, H, W, generator=g).to(tr.device), cv.x_c)
    xr = x[..., :cin].permute(0, 3, 1, 2).double().requires_grad_(True)
    yr = F.conv2d(ft.circular_pad(xr, cv.p), w, b, stride=s)
    dy = _nhwc(torch.randn(yr.shape, generator=g).to(tr.device), cv.dy_c)
    yr.backward(dy[..., :cout].permute(0, 3, 1, 2).double())
    y = tr._conv(cv, x, B, H, W, ft.F32 if cout == 3 else ft.F16)
    e = {"y": _rel(y[..., :cout].permute(0, 3, 1, 2), yr)}
    if cv.dg is not None:
        dx = tr._dgrad(cv, dy, B, H, W)
        e["dx"] = _rel(dx.permute(0, 3, 1, 2), xr.grad)
    print(f"\n{cin}->{cout} k{k} s{s} {H}x{W}: " + ", ".join(f"{n} {v:.2e}" for n, v in e.items()))
    # measured on an H100: y, dx <= 3.0e-4 (fp16 outputs)
    assert e["y"] < 6e-4 and e.get("dx", 0.0) < 6e-4
