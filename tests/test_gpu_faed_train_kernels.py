"""GPU: the FAED training kernels one at a time (csrc/faed_train.cu through panfusion_b200.faed_train's call paths)
against fp64 torch autograd on the same fp16-rounded operands: forward convolution, dgrad and wgrad / db for every
layer shape of the autoencoder at W = 64 and at a W that is not a multiple of the 128-pixel CTA tile, one wgrad shape
large enough that the partial-buffer cap sets the chunk count, BatchNorm forward / running statistics / backward,
the bilinear upsample both ways, and the loss and its seed. Gates are about 2x the errors measured on an H100."""
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
    wr = w.clone().requires_grad_(True)
    br = b.clone().requires_grad_(True)
    F.conv2d(ft.circular_pad(x[..., :cin].permute(0, 3, 1, 2).double(), cv.p), wr, br, stride=s).backward(
        dy[..., :cout].permute(0, 3, 1, 2).double())
    y = tr._conv(cv, x, B, H, W, ft.F32 if cout == 3 else ft.F16)
    tr._wgrad(cv, x, dy, B, H, W)
    dw = tr.grads[: w.numel()].view(w.shape)
    db = tr.grads[w.numel(): w.numel() + cout]
    e = {"y": _rel(y[..., :cout].permute(0, 3, 1, 2), yr), "dw": _rel(dw, wr.grad), "db": _rel(db, br.grad)}
    if cv.dg is not None:
        dx = tr._dgrad(cv, dy, B, H, W)
        e["dx"] = _rel(dx.permute(0, 3, 1, 2), xr.grad)
    print(f"\n{cin}->{cout} k{k} s{s} {H}x{W}: " + ", ".join(f"{n} {v:.2e}" for n, v in e.items()))
    # measured on an H100: y, dx <= 3.0e-4 (fp16 outputs), dw <= 1.2e-6, db <= 9.1e-8
    assert e["y"] < 6e-4 and e.get("dx", 0.0) < 6e-4
    assert e["dw"] < 2.5e-6 and e["db"] < 2e-7


def test_wgrad_where_the_partial_cap_sets_the_chunks(tr):
    """32->32 k9 at 256x1024: ceil(P / 1024) = 256 chunks exceed the 2^24-float cap (202 chunks)."""
    B, H, W = 1, 256, 1024
    cv, w, b = _layer(tr, 32, 32, 9, 1, seed=5)
    g = torch.Generator().manual_seed(8)
    x = _nhwc(torch.randn(B, 32, H, W, generator=g).to(tr.device), 32)
    dy = _nhwc(torch.randn(B, 32, H, W, generator=g).to(tr.device), 32)
    l = _lib.lib()
    l.pf_faedt_wgrad_ws_floats.restype = C.c_longlong
    # the cap allows 202 chunks; chunks rounded up to 32 pixels give 200 (an uncapped split would be 256)
    assert l.pf_faedt_wgrad_ws_floats(B, H, W, 32, 32, 9) == 200 * (81 * 32 * 32 + 32)
    wr = w.clone().requires_grad_(True)
    br = b.clone().requires_grad_(True)
    F.conv2d(ft.circular_pad(x.permute(0, 3, 1, 2).double(), 4), wr, br).backward(dy.permute(0, 3, 1, 2).double())
    tr._wgrad(cv, x, dy, B, H, W)
    e_w = _rel(tr.grads[: w.numel()].view(w.shape), wr.grad)
    e_b = _rel(tr.grads[w.numel(): w.numel() + 32], br.grad)
    print(f"\ncapped wgrad: dw {e_w:.2e} db {e_b:.2e}")
    assert e_w < 3.5e-6 and e_b < 6e-7  # measured 1.6e-6 and 3.0e-7 (1311 pixels per chunk, 200 chunks)


@pytest.mark.parametrize("C_", [32, 64, 128])
def test_batchnorm_forward_running_stats_backward(tr, C_):
    P = 3 * 1000 + 7
    g = torch.Generator().manual_seed(C_)
    # a conv bias before BN makes the mean large against the spread
    z = (40 + 5 * torch.randn(C_, generator=g) + 0.5 * torch.randn(P, C_, generator=g)).half().to(tr.device)
    res = torch.randn(P, C_, generator=g).half().to(tr.device)
    gamma = (0.5 + torch.rand(C_, generator=g)).to(tr.device)
    beta = (0.2 * torch.randn(C_, generator=g)).to(tr.device)
    l, st = _lib.lib(), C.c_void_p(tr._st)
    l.pf_faedt_bn_ws_floats.restype = C.c_longlong
    ws = torch.empty(l.pf_faedt_bn_ws_floats(C.c_longlong(P), C_), device=tr.device)
    stats = torch.empty(3 * C_, device=tr.device)
    pending = torch.empty(2 * C_, device=tr.device)
    _lib.check(l.pf_faedt_bn_stats(ft._vp(z), C.c_longlong(P), C_, ft._vp(ws), ft._vp(stats), ft._vp(pending), st))
    zd = z.double()
    mean, var_b, var_u = zd.mean(0), zd.var(0, unbiased=False), zd.var(0, unbiased=True)
    e_mean = ((stats[:C_].double() - mean).abs().max() / zd.std(0).min()).item()
    e_inv = _rel(stats[C_: 2 * C_], 1 / torch.sqrt(var_b + 1e-5))
    e_pend = max(_rel(pending[:C_], mean), _rel(pending[C_:], var_u))
    outs = {}
    for relu, r in ((1, None), (0, res)):
        out = torch.empty_like(z)
        _lib.check(l.pf_faedt_bn_apply(ft._vp(z), C.c_longlong(P), C_, ft._vp(stats), ft._vp(gamma), ft._vp(beta),
                                       relu, ft._vp(r), ft._vp(out), st))
        outs[relu] = out
    ref = F.batch_norm(zd, None, None, gamma.double(), beta.double(), True, 0.1, 1e-5)
    e_apply = max(_rel(outs[1], ref.relu()), _rel(outs[0], ref + res.double()))
    # backward through relu(bn(z)): mask from the stored ReLU output
    gup = torch.randn(P, C_, generator=g).half().to(tr.device)
    dz = torch.empty_like(z)
    dgam = torch.empty(C_, device=tr.device)
    dbet = torch.empty(C_, device=tr.device)
    flag = torch.zeros(1, device=tr.device, dtype=torch.int32)
    _lib.check(l.pf_faedt_bn_bwd(ft._vp(gup), ft._vp(outs[1]), ft._vp(z), C.c_longlong(P), C_, ft._vp(stats),
                                 ft._vp(gamma), ft._vp(ws), ft._vp(tr.ctl[1:]), C.c_double(1.0), ft._vp(dgam),
                                 ft._vp(dbet), ft._vp(flag), ft._vp(dz), st))
    zr2 = zd.clone().requires_grad_(True)
    gr, br_ = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    F.batch_norm(zr2, None, None, gr, br_, True, 0.1, 1e-5).relu().backward(gup.double())
    e_dz, e_dg, e_db = _rel(dz, zr2.grad), _rel(dgam, gr.grad), _rel(dbet, br_.grad)
    print(f"\nBN C={C_}: mean {e_mean:.2e} (of the std), invstd {e_inv:.2e}, pending {e_pend:.2e}, "
          f"apply {e_apply:.2e}, dz {e_dz:.2e}, dgamma {e_dg:.2e}, dbeta {e_db:.2e}")
    # measured on an H100: mean 1.8e-5 of the std, invstd 3.6e-7, pending 6.9e-7, apply 2.1e-4, dz 2.1e-4,
    # dgamma 5.5e-6, dbeta 5.7e-8
    assert e_mean < 4e-5 and e_inv < 8e-7 and e_pend < 1.5e-6 and e_apply < 5e-4
    assert e_dz < 5e-4 and e_dg < 1.2e-5 and e_db < 1.2e-7 and int(flag) == 0


@pytest.mark.parametrize("H,W", [(5, 7), (16, 32)])
def test_upsample_forward_backward(tr, H, W):
    B, C_ = 2, 32
    g = torch.Generator().manual_seed(H)
    x = torch.randn(B, H, W, C_, generator=g).half().to(tr.device)
    gy = torch.randn(B, 2 * H, 2 * W, C_, generator=g).half().to(tr.device)
    y = torch.empty(B, 2 * H, 2 * W, C_, device=tr.device, dtype=torch.float16)
    dx = torch.empty_like(x)
    l, st = _lib.lib(), C.c_void_p(tr._st)
    _lib.check(l.pf_faedt_upsample(ft._vp(x), B, H, W, C_, ft._vp(y), st))
    _lib.check(l.pf_faedt_upsample_bwd(ft._vp(gy), B, H, W, C_, ft._vp(dx), st))
    xr = x.permute(0, 3, 1, 2).double().requires_grad_(True)
    yr = F.interpolate(xr, scale_factor=2, mode="bilinear", align_corners=False)
    yr.backward(gy.permute(0, 3, 1, 2).double())
    e_y, e_dx = _rel(y.permute(0, 3, 1, 2), yr), _rel(dx.permute(0, 3, 1, 2), xr.grad)
    print(f"\nupsample {H}x{W}: y {e_y:.2e} dx {e_dx:.2e}")
    assert e_y < 5e-4 and e_dx < 5e-4  # measured 2.1e-4 (fp16 outputs)


def test_loss_and_seed(tr):
    B, H, W = 2, 32, 64
    g = torch.Generator().manual_seed(3)
    o = torch.randn(B, H, W, 4, generator=g).to(tr.device)
    t = (torch.rand(B, 3, H, W, generator=g) * 2 - 1).to(tr.device)
    l = _lib.lib()
    ws = torch.empty(1024, device=tr.device)
    loss = torch.empty((), device=tr.device)
    pred = torch.empty(B, 3, H, W, device=tr.device)
    seed = torch.empty(B, H, W, 16, device=tr.device, dtype=torch.float16)
    flag = torch.zeros(1, device=tr.device, dtype=torch.int32)
    _lib.check(l.pf_faedt_loss(ft._vp(o), ft._vp(t), B, H, W, ft._vp(tr.ctl[1:]), ft._vp(ws), ft._vp(loss),
                               ft._vp(pred), ft._vp(seed), ft._vp(flag), C.c_void_p(tr._st)))
    pr = torch.tanh(o[..., :3].permute(0, 3, 1, 2).double())
    d = pr - t.double()
    ref = d.abs().mean()
    want = torch.sign(d) * (1 - pr * pr)
    got = seed[..., :3].permute(0, 3, 1, 2).double()
    clear = d.abs() > 1e-5  # the sign of a difference below fp32 rounding is not defined by either side
    e_loss = abs(loss.item() - ref.item()) / ref.item()
    e_seed = (got - want)[clear].abs().max().item()
    e_pred = _rel(pred, pr)
    print(f"\nloss {e_loss:.2e}, seed max abs {e_seed:.2e}, pred {e_pred:.2e}")
    # measured 3.7e-8 and 2.4e-4 (half an fp16 ulp below 1)
    assert e_loss < 1e-7 and e_seed < 5e-4 and not seed[..., 3:].any() and int(flag) == 0
    assert e_pred < 1e-6
