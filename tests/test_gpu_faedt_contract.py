"""-m gpu: the FAED training step's own kernels (csrc/faed_train.cu: weight gradients, training-mode BatchNorm, the
bilinear upsample both ways, the loss and its seed, Adam and the loss-scale state machine, and the exact layout
kernels prep / interleave / pack) against the fp64 restatements of tests/_contract.py, at the shapes and argument
combinations FAEDTrainer passes.

Every output starts as NaN, including the dw / db slices inside a larger gradient buffer, so a store outside the
contract fails. The weight gradient is checked at three levels: each chunk's fp32 partial where the workspace keeps it
(a dropped 32-pixel stage or a chunk boundary counted twice moves a partial far past its bound, but dw by only about
32 / P), the reduction of those partials, and dw / db end to end. The BatchNorm statistics are checked per chunk (the
Welford counts exactly) and merged. Adam must equal torch.optim.Adam(foreach=False) bit for bit. Repeat launches are
byte-identical. `_Recorder` logs the class of every call FAEDTrainer.training_step and reconstruct make;
`test_faedt_call_table_covers_the_trainer` requires a case for each."""
import ctypes as C

import pytest
import torch

import _contract as ct

pytestmark = pytest.mark.gpu

ENTRIES = ("pf_faedt_prep", "pf_faedt_wgrad", "pf_faedt_bn_stats", "pf_faedt_bn_apply", "pf_faedt_bn_bwd",
           "pf_faedt_upsample", "pf_faedt_upsample_bwd", "pf_faedt_loss", "pf_faedt_adam", "pf_faedt_pack",
           "pf_faedt_interleave")
F16 = torch.float16


def _vp(t):
    return C.c_void_p(0 if t is None else t.data_ptr())


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _nan(shape, dtype, dev):
    return torch.full(shape, float("nan"), dtype=dtype, device=dev)


def _bits(t):
    return t.view({2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


def _same(a, b):
    return torch.equal(_bits(a), _bits(b))


def _lib():
    from panfusion_b200 import _lib as L
    return L


def _ll(v):
    return C.c_longlong(int(v))


def _inv_n(B, H, W):
    """FAEDTrainer's inv_n: 1 / N of the L1 mean over the image batch."""
    return 1.0 / (3.0 * B * H * W)


# ---- call classes ---------------------------------------------------------------------------------------------------

def _p(a):
    return a.value if hasattr(a, "value") else a


def _given(a):
    return _p(a) not in (None, 0)


def wgrad_tile(cin, cdy):
    return (32 if cin <= 32 else 64, 32 if cdy <= 32 else (64 if cdy <= 64 else 128))


def call_class(name, args):
    a = [_p(v) for v in args]
    if name == "pf_faedt_wgrad":  # (x, B, H, W, Cin, dy, Ho, Wo, Cdy, Cin_w, Cout, k, stride, pad, ws, scale, inv_n, dw, db, ..)
        return (name, a[4], a[8], a[9], a[10], a[11], a[12], _given(a[18]), wgrad_tile(a[4], a[8]))
    if name == "pf_faedt_bn_stats":  # (z, P, C, ..)
        return (name, a[2])
    if name == "pf_faedt_bn_apply":  # (z, P, C, stats, gamma, beta, relu, residual, out, st)
        return (name, a[2], bool(a[6]), _given(a[7]))
    if name == "pf_faedt_bn_bwd":  # (g, mask, z, P, C, ..)
        return (name, a[4], _given(a[1]))
    if name == "pf_faedt_loss":  # (o, target, B, H, W, scale, ws, loss, pred, seed, flag, st)
        return (name, _given(a[1]), _given(a[8]))
    if name == "pf_faedt_pack":  # (w, Cout, Cin, k, stride, fwd, cin_pad, cw, dg, ..)
        return (name, a[3], a[4], _given(a[8]))
    return (name,)


class _Recorder:
    """Stands in for the library handle: logs the class of every FAED training-kernel call, then forwards it."""

    def __init__(self, lib):
        self._lib, self.calls = lib, []

    def __getattr__(self, name):
        f = getattr(self._lib, name)
        if name not in ENTRIES:
            return f

        def rec(*args):
            self.calls.append(call_class(name, args))
            return f(*args)
        return rec


@pytest.fixture
def recorder(monkeypatch, cuda_device):
    L = _lib()
    rec = _Recorder(L.lib())
    monkeypatch.setattr(L, "lib", lambda: rec)
    return rec


# ---- weight gradient ------------------------------------------------------------------------------------------------

def trainer_layers(B, H, W):
    """(cin, cout, k, stride, B, H, W) of every convolution FAEDTrainer runs on a B x H x W batch, in forward order."""
    from panfusion_b200.faed_train import DEC, ENC
    out = []
    for plan in (ENC, DEC):
        for kind, _name, args in plan:
            if kind == "up":
                H, W = 2 * H, 2 * W
            elif kind == "rb":
                c, k = args
                out += [(c, c, k, 1, B, H, W)] * 2
            else:
                cin, cout, k, s, _p = args
                out.append((cin, cout, k, s, B, H, W))
                if s == 2:
                    H, W = H // 2, W // 2
    return out


def wg(cin, cout, k, s, B, H, W, S=1.0, inv_n=None, db=True, label=""):
    return dict(cin=cin, cout=cout, k=k, s=s, B=B, H=H, W=W, S=S, inv_n=inv_n, db=db, label=label)


WGRAD_CASES = {
    "trainer_64x128": lambda: [wg(*L, inv_n=_inv_n(2, 64, 128)) for L in dict.fromkeys(trainer_layers(2, 64, 128))],
    "scale_2^10": lambda: [wg(*L, S=2.0 ** 10, inv_n=_inv_n(2, 64, 128))
                           for L in dict.fromkeys(trainer_layers(2, 64, 128)) if L[2] in (9, 4)],
    "P_not_a_multiple_of_32": lambda: [wg(32, 32, 9, 1, 1, 13, 40), wg(64, 128, 4, 2, 2, 12, 40),
                                       wg(3, 32, 9, 1, 1, 13, 40), wg(128, 64, 3, 1, 2, 3, 5)],
    # the smallest W each pad allows (pad < W); k4 s2 at W = 4: the last output column's tap kx = 3 wraps to column 0
    "smallest_W": lambda: [wg(32, 32, 9, 1, 2, 6, 5), wg(64, 64, 7, 1, 2, 6, 4), wg(128, 128, 5, 1, 2, 6, 3),
                           wg(128, 128, 3, 1, 2, 6, 2), wg(64, 128, 4, 2, 2, 6, 2), wg(32, 64, 4, 2, 2, 6, 4),
                           wg(32, 3, 9, 1, 2, 6, 5)],
    "db_null": lambda: [wg(64, 64, 7, 1, 2, 16, 32, db=False), wg(32, 3, 9, 1, 2, 16, 32, db=False)],
    # the largest chunk the trainer makes: 403 chunks of 5216 pixels
    "first_layer_4x512x1024": lambda: [wg(3, 32, 9, 1, 4, 512, 1024, S=2.0 ** 10, inv_n=_inv_n(4, 512, 1024))],
}


CAPPED = wg(32, 32, 9, 1, 1, 256, 1024)  # the shape where the partial-float cap sets the chunk count


def _wgrad_operands(s, g, dev):
    x_c, dy_c = (16 if s["cin"] == 3 else s["cin"]), (16 if s["cout"] == 3 else s["cout"])
    p = 1 if s["s"] == 2 else s["k"] // 2
    Ho, Wo = (s["H"] + 2 * p - s["k"]) // s["s"] + 1, (s["W"] + 2 * p - s["k"]) // s["s"] + 1
    x = torch.randn(s["B"], s["H"], s["W"], x_c, generator=g).to(F16).to(dev)
    dy = torch.randn(s["B"], Ho, Wo, dy_c, generator=g).to(F16).to(dev)
    return x, dy, x_c, dy_c, p, Ho, Wo


def _launch_wgrad(s, x, dy, x_c, dy_c, p, Ho, Wo, flag, inv_n):
    """-> (ws, grads, (dw, db) views): dw / db inside a NaN gradient buffer with NaN on both sides."""
    L = _lib()
    lib, dev = L.lib(), x.device
    B, H, W, k = s["B"], s["H"], s["W"], s["k"]
    ws = _nan((L.lib().pf_faedt_wgrad_ws_floats(B, Ho, Wo, x_c, dy_c, k),), torch.float32, dev)
    n_w = s["cout"] * s["cin"] * k * k
    grads = _nan((5 + n_w + s["cout"] + 5,), torch.float32, dev)
    dw, db = grads[5:5 + n_w], grads[5 + n_w:5 + n_w + s["cout"]]
    scale = torch.tensor([s["S"]], dtype=torch.float64, device=dev)
    L.check(lib.pf_faedt_wgrad(_vp(x), B, H, W, x_c, _vp(dy), Ho, Wo, dy_c, s["cin"], s["cout"], k, s["s"], p, _vp(ws),
                               _vp(scale), C.c_double(inv_n), _vp(dw), _vp(db if s["db"] else None), _vp(flag),
                               _st()))
    return ws, grads, dw, db


def _check_wgrad(s, g, dev):
    x, dy, x_c, dy_c, p, Ho, Wo = _wgrad_operands(s, g, dev)
    inv_n = s["inv_n"] or _inv_n(s["B"], s["H"], s["W"])
    flag = torch.zeros(1, dtype=torch.int32, device=dev)
    ws, grads, dw, db = _launch_wgrad(s, x, dy, x_c, dy_c, p, Ho, Wo, flag, inv_n)
    ws2, grads2, _, _ = _launch_wgrad(s, x, dy, x_c, dy_c, p, Ho, Wo, flag, inv_n)
    torch.cuda.synchronize()
    k, cin, cout = s["k"], s["cin"], s["cout"]
    label = f"{cin}->{cout} k{k} s{s['s']} B={s['B']} {s['H']}x{s['W']} S={s['S']:g} db={s['db']}"
    assert int(flag) == 0, label
    assert _same(ws, ws2) and _same(grads, grads2), f"repeat launch differs: {label}"
    r = ct.wgrad_ref(x, dy, Ho=Ho, Wo=Wo, k=k, stride=s["s"], pad=p)
    nch, taps = r["nch"], k * k
    n_part = nch * taps * x_c * dy_c
    assert ws.numel() == n_part + nch * dy_c, label  # the documented workspace layout
    part = ws[:n_part].view(nch, taps, x_c, dy_c)
    f = ct.faedt_factor(inv_n, s["S"])
    res = {"part": ct.worst_ratio(part, r["part"], r["part_bound"])}
    ref, bound = ct.wgrad_reduce_ref(part, f)
    res["dw reduce"] = ct.worst_ratio(dw.view(cout, cin, k, k), ct.wgrad_layout(ref, cin, cout, k),
                                      ct.wgrad_layout(bound, cin, cout, k))
    e2e = f * r["w"]
    res["dw"] = ct.worst_ratio(dw.view(cout, cin, k, k), ct.wgrad_layout(e2e, cin, cout, k),
                               ct.wgrad_layout(f * r["w_bound"] + ct.U * e2e.abs() + ct.EXACT, cin, cout, k))
    assert torch.isnan(grads[:5]).all() and torch.isnan(grads[-5:]).all(), f"store outside dw / db: {label}"
    if s["db"]:
        dbpart = ws[n_part:].view(nch, dy_c)
        res["dbpart"] = ct.worst_ratio(dbpart, r["dbpart"], r["dbpart_bound"])
        ref, bound = ct.wgrad_reduce_ref(dbpart, f)
        res["db reduce"] = ct.worst_ratio(db, ref[:cout], bound[:cout])
        eb = f * r["b"][:cout]
        res["db"] = ct.worst_ratio(db, eb, f * r["b_bound"][:cout] + ct.U * eb.abs() + ct.EXACT)
    else:
        assert torch.isnan(db).all() and torch.isnan(ws[n_part:]).all(), f"db written with db = NULL: {label}"
    print(f"[contract] wgrad {label} ({nch} chunks of {r['chunk']}): "
          + ", ".join(f"{n} {v:.3f}" for n, v in res.items()))
    return max(res.values())


@pytest.mark.parametrize("case", list(WGRAD_CASES))
def test_wgrad_contract(cuda_device, case):
    g = torch.Generator().manual_seed(sum(map(ord, case)))
    worst = max(_check_wgrad(s, g, cuda_device) for s in WGRAD_CASES[case]())
    print(f"[contract] wgrad {case}: worst err/bound {worst:.3f}")
    assert worst <= 1.0, worst


def test_wgrad_capped_chunks_contract(cuda_device):
    """32 -> 32 k9 at 256 x 1024: ceil(P / 1024) = 256 chunks would exceed the 2^24-float cap, which allows 202; chunks
    rounded up to 32 pixels give 200 of 1312. The workspace is sized for them and every partial, the reduction and dw /
    db meet their bounds."""
    s = CAPPED
    assert ct.wgrad_chunk(256 * 1024, 81, 32, 32) == 1312
    assert _lib().lib().pf_faedt_wgrad_ws_floats(1, 256, 1024, 32, 32, 9) == 200 * (81 * 32 * 32 + 32)
    worst = _check_wgrad(s, torch.Generator().manual_seed(5), cuda_device)
    assert worst <= 1.0, worst


# ---- BatchNorm ------------------------------------------------------------------------------------------------------

def _bn_z(P, C, g, dev, mean=40.0, spread=0.5):
    """A conv output before BN: each channel's bias large against its spread."""
    m = mean + 5 * torch.randn(C, generator=g)
    return (m + spread * torch.randn(P, C, generator=g)).to(F16).to(dev)


def _bn_params(C, g, dev):
    return (0.5 + torch.rand(C, generator=g)).to(dev), (0.2 * torch.randn(C, generator=g)).to(dev)


def _launch_bn_stats(z, Cc):
    L = _lib()
    P, dev = z.shape[0], z.device
    ws = _nan((L.lib().pf_faedt_bn_ws_floats(_ll(P), Cc),), torch.float32, dev)
    stats, pending = _nan((3, Cc), torch.float32, dev), _nan((2, Cc), torch.float32, dev)
    L.check(L.lib().pf_faedt_bn_stats(_vp(z), _ll(P), Cc, _vp(ws), _vp(stats), _vp(pending), _st()))
    return ws, stats, pending


def _launch_bn_apply(z, Cc, stats, gamma, beta, relu, residual):
    L = _lib()
    out = _nan(z.shape, F16, z.device)
    L.check(L.lib().pf_faedt_bn_apply(_vp(z), _ll(z.shape[0]), Cc, _vp(stats), _vp(gamma), _vp(beta), int(relu),
                                      _vp(residual), _vp(out), _st()))
    return out


def _launch_bn_bwd(gup, mask, z, Cc, stats, gamma, S, inv_n, flag):
    L = _lib()
    P, dev = z.shape[0], z.device
    ws = _nan((L.lib().pf_faedt_bn_ws_floats(_ll(P), Cc),), torch.float32, dev)
    grads = _nan((2 * Cc + 4,), torch.float32, dev)
    dgamma, dbeta = grads[2:2 + Cc], grads[2 + Cc:2 + 2 * Cc]
    dz = _nan(z.shape, F16, dev)
    scale = torch.tensor([S], dtype=torch.float64, device=dev)
    L.check(L.lib().pf_faedt_bn_bwd(_vp(gup), _vp(mask), _vp(z), _ll(P), Cc, _vp(stats), _vp(gamma), _vp(ws),
                                    _vp(scale), C.c_double(inv_n), _vp(dgamma), _vp(dbeta), _vp(flag), _vp(dz), _st()))
    return ws, grads, dgamma, dbeta, dz


def bn(P, C, mean=40.0, spread=0.5, label=""):
    return dict(P=P, C=C, mean=mean, spread=spread, label=label)


BN_CASES = {
    "large_mean_small_spread": lambda: [bn(3007, C) for C in (32, 64, 128)],
    "last_chunk_one_row": lambda: [bn(257, C) for C in (32, 64, 128)],
    # FAEDTrainer at B = 2, 64 x 128: every BatchNorm's P and C, and the spread-dominated decoder side
    "trainer_64x128": lambda: ([bn(16384, 32), bn(4096, 64), bn(1024, 128), bn(256, 128), bn(64, 128), bn(16, 128),
                                bn(4096, 32, mean=0.2, spread=1.0), bn(1024, 64, mean=0.2, spread=1.0)]),
    # batch 4 at 512 x 1024: the encoder's first level
    "trainer_4x512x1024": lambda: [bn(4 * 512 * 1024, 32)],
    # past 2^24 rows: the counts are kept in fp32
    "P_past_2^24": lambda: [bn((1 << 24) + 1001, 32, mean=0.5, spread=1.0)],
}


def _check_bn(s, g, dev, S=2.0 ** 10):
    P, Cc = s["P"], s["C"]
    z = _bn_z(P, Cc, g, dev, s["mean"], s["spread"])
    gamma, beta = _bn_params(Cc, g, dev)
    ws, stats, pending = _launch_bn_stats(z, Cc)
    ws2, stats2, _ = _launch_bn_stats(z, Cc)
    torch.cuda.synchronize()
    label = f"P={P} C={Cc} mean~{s['mean']} spread {s['spread']}"
    assert _same(ws, ws2) and _same(stats, stats2), f"repeat launch differs: {label}"
    assert _same(pending[0], stats[0]) and _same(pending[1], stats[2]), label
    r = ct.bn_stats_ref(z)
    nch = r["nch"]
    part = ws[:nch * 3 * Cc].view(nch, 3, Cc)
    assert torch.equal(part[:, 0].double(), r["count"]), f"chunk counts: {label}"
    res = {"chunk mean": ct.worst_ratio(part[:, 1], r["mean"], r["mean_bound"]),
           "chunk M2": ct.worst_ratio(part[:, 2], r["m2"], r["m2_bound"]),
           "stats": ct.worst_ratio(stats, r["stats"], r["stats_bound"])}
    del r
    out_relu = _launch_bn_apply(z, Cc, stats, gamma, beta, True, None)
    res["apply relu"] = ct.worst_ratio(out_relu, *ct.bn_apply_ref(z, stats, gamma, beta, True))
    if P > (1 << 22):  # past 2^24 rows only the statistics and one apply: the fp64 backward would not fit
        print(f"[contract] bn {label} ({nch} chunks): " + ", ".join(f"{n} {v:.3f}" for n, v in res.items()))
        return max(res.values())
    residual = torch.randn(P, Cc, generator=g).to(F16).to(dev)
    out_res = _launch_bn_apply(z, Cc, stats, gamma, beta, False, residual)
    res["apply residual"] = ct.worst_ratio(out_res, *ct.bn_apply_ref(z, stats, gamma, beta, False, residual))
    # eval mode: FAEDTrainer._bn_fwd's statistics from the running mean and variance
    run = torch.stack([stats[0], stats[2] * 1.5])
    ev = torch.cat([run[0], torch.rsqrt(run[1] + 1e-5), run[1]]).view(3, Cc)
    out_ev = _launch_bn_apply(z, Cc, ev, gamma, beta, True, None)
    res["apply eval"] = ct.worst_ratio(out_ev, *ct.bn_apply_ref(z, ev, gamma, beta, True))
    gup = torch.randn(P, Cc, generator=g).to(F16).to(dev)
    inv_n = _inv_n(2, 64, 128)
    f = ct.faedt_factor(inv_n, S)
    flag = torch.zeros(1, dtype=torch.int32, device=dev)
    for mask in (out_relu, None):
        ws_b, grads, dgamma, dbeta, dz = _launch_bn_bwd(gup, mask, z, Cc, stats, gamma, S, inv_n, flag)
        ws_b2, grads2, _, _, dz2 = _launch_bn_bwd(gup, mask, z, Cc, stats, gamma, S, inv_n, flag)
        torch.cuda.synchronize()
        assert _same(ws_b, ws_b2) and _same(grads, grads2) and _same(dz, dz2), f"repeat bwd differs: {label}"
        assert torch.isnan(grads[:2]).all() and torch.isnan(grads[-2:]).all(), f"store outside dgamma / dbeta: {label}"
        b = ct.bn_bwd_ref(gup, mask, z, stats, gamma, f)
        tag = "masked" if mask is not None else "unmasked"
        sums = ws_b[nch * 3 * Cc:nch * 3 * Cc + 2 * Cc].view(2, Cc)
        res[f"bwd part {tag}"] = ct.worst_ratio(ws_b[:nch * 2 * Cc].view(nch, 2, Cc), b["part"], b["part_bound"])
        res[f"bwd sums {tag}"] = ct.worst_ratio(sums, b["sums"], b["sums_bound"])
        res[f"dgamma {tag}"] = ct.worst_ratio(dgamma, b["dgamma"], b["dgamma_bound"])
        res[f"dbeta {tag}"] = ct.worst_ratio(dbeta, b["dbeta"], b["dbeta_bound"])
        res[f"dz {tag}"] = ct.worst_ratio(dz, *b["dz_ref"](sums))
        del b
    assert int(flag) == 0, label
    print(f"[contract] bn {label} ({nch} chunks): " + ", ".join(f"{n} {v:.3f}" for n, v in res.items()))
    return max(res.values())


@pytest.mark.parametrize("case", list(BN_CASES))
def test_bn_contract(cuda_device, case):
    g = torch.Generator().manual_seed(sum(map(ord, case)))
    worst = max(_check_bn(s, g, cuda_device) for s in BN_CASES[case]())
    print(f"[contract] bn {case}: worst err/bound {worst:.3f}")
    assert worst <= 1.0, worst


# ---- upsample -------------------------------------------------------------------------------------------------------

UP_SHAPES = [(2, 1, 5, 32), (2, 5, 1, 32), (1, 1, 1, 32), (2, 3, 7, 64), (2, 2, 4, 128), (2, 4, 8, 128), (2, 8, 16, 128),
             (2, 16, 32, 64), (2, 32, 64, 32), (4, 256, 512, 32)]


def _launch_up(x, gy):
    L = _lib()
    B, H, W, Cc = x.shape
    y = _nan((B, 2 * H, 2 * W, Cc), F16, x.device)
    dx = _nan(x.shape, F16, x.device)
    L.check(L.lib().pf_faedt_upsample(_vp(x), B, H, W, Cc, _vp(y), _st()))
    L.check(L.lib().pf_faedt_upsample_bwd(_vp(gy), B, H, W, Cc, _vp(dx), _st()))
    return y, dx


@pytest.mark.parametrize("shape", UP_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_upsample_contract(cuda_device, shape):
    """H or W = 1, odd sizes, every decoder level of a 64 x 128 pair and the last level at 4 x 512 x 1024."""
    B, H, W, Cc = shape
    g = torch.Generator().manual_seed(H * 1000 + W)
    x = torch.randn(B, H, W, Cc, generator=g).to(F16).to(cuda_device)
    gy = torch.randn(B, 2 * H, 2 * W, Cc, generator=g).to(F16).to(cuda_device)
    y, dx = _launch_up(x, gy)
    y2, dx2 = _launch_up(x, gy)
    torch.cuda.synchronize()
    assert _same(y, y2) and _same(dx, dx2)
    rf = ct.worst_ratio(y, *ct.upsample_ref(x))
    rb = ct.worst_ratio(dx, *ct.upsample_bwd_ref(gy, H, W))
    print(f"[contract] upsample {shape}: forward err/bound {rf:.3f}, backward {rb:.3f}")
    assert max(rf, rb) <= 1.0, (rf, rb)


# ---- loss -----------------------------------------------------------------------------------------------------------

def _launch_loss(o, t, S, with_pred, flag):
    L = _lib()
    B, H, W = o.shape[:3]
    dev = o.device
    ws = _nan((L.lib().pf_faedt_loss_ws_floats(),), torch.float32, dev)
    loss = _nan((), torch.float32, dev)
    pred = _nan((B, 3, H, W), torch.float32, dev) if with_pred else None
    seed = _nan((B, H, W, 16), F16, dev)
    scale = torch.tensor([S], dtype=torch.float64, device=dev)
    L.check(L.lib().pf_faedt_loss(_vp(o), _vp(t), B, H, W, _vp(scale), _vp(ws), _vp(loss), _vp(pred), _vp(seed),
                                  _vp(flag), _st()))
    return loss, pred, seed


def _check_loss(dev, B, H, W, S):
    """-> worst err/bound of one loss shape and scale, with the target given and NULL."""
    g = torch.Generator().manual_seed(B * H + W)
    o = (torch.randn(B, H, W, 4, generator=g) * 2)
    t = torch.rand(B, 3, H, W, generator=g) * 2 - 1
    o[:, :2, :5] = 0
    t[:, :, :1, :5] = 0  # tanh(0) - 0 = 0: sign(0) = 0
    o[0, 2, :4, :3] = torch.tensor([1e-3, -1e-3, 20.0, -20.0])[:, None]
    o, t = o.to(dev), t.to(dev)
    worst = 0.0
    for target in (t, None):
        flag = torch.zeros(1, dtype=torch.int32, device=dev)
        loss, pred, seed = _launch_loss(o, target, S, True, flag)
        loss2, _, seed2 = _launch_loss(o, target, S, False, flag)
        loss3, _, _ = _launch_loss(o, target, S, False, flag)
        torch.cuda.synchronize()
        assert int(flag) == 0
        assert _same(seed, seed2) and _same(loss, loss2) and _same(loss2, loss3), "pred = NULL changes the result"
        r = ct.loss_ref(o, target, B, H, W)
        rp = ct.worst_ratio(pred, r["pred"], r["pred_bound"])
        rl = float((loss.double() - r["loss"]).abs() / r["loss_bound"])
        rs, n_clear = ct.seed_check(seed, pred, r["d"], r["pred_bound"], S)
        n_inf = int(torch.isinf(seed).sum())
        assert (S < 2 ** 16) == (n_inf == 0), n_inf
        print(f"[contract] loss {B}x{H}x{W} S={S:g} target={'given' if target is not None else 'NULL'}: pred {rp:.3f}, "
              f"loss {rl:.3f}, seed {rs:.3f} ({n_clear} signs defined, {n_inf} inf seeds)")
        worst = max(worst, rp, rl, rs)
    return worst


def test_loss_contract(cuda_device):
    """pred within 2 ulp of tanh, the L1 mean within its partition's bound, the seed sign (1 - pred^2) S, at a 32 x 64
    pair and at a 256 x 1024 pair (two pixels per thread), S in {1, 2^15, 2^16}; target = NULL (reconstruct) and
    pred = NULL (training_step). At S = 2^16 seeds with (1 - pred^2) S >= 65520 round to inf in fp16, which is the
    correct rounding: the loss launch sets the flag only for a non-finite loss, so the flag stays clear and the inf
    seeds set it later, through the gradients they produce."""
    worst = max(_check_loss(cuda_device, B, H, W, S) for B, H, W in ((2, 32, 64), (2, 256, 1024))
                for S in (1.0, 2.0 ** 15, 2.0 ** 16))
    print(f"[contract] loss: worst err/bound {worst:.3f}")
    assert worst <= 1.0, worst


# ---- the non-finite flag --------------------------------------------------------------------------------------------

def test_nonfinite_flag_is_set_by_bad_inputs_and_cleared_only_by_the_step_end(cuda_device):
    """An inf in dy (wgrad), a NaN in z (BN backward) and a NaN in o (loss) each set the flag; with finite inputs a set
    flag stays set through every kernel that writes it; only pf_faedt_adam's step end clears it."""
    dev = cuda_device
    g = torch.Generator().manual_seed(70)
    s = wg(32, 32, 3, 1, 2, 8, 16)

    def run_all(flag, bad):
        x, dy, x_c, dy_c, p, Ho, Wo = _wgrad_operands(s, g, dev)
        if bad == "dy":
            dy[1, 3, 4, 5] = float("inf")
        _launch_wgrad(s, x, dy, x_c, dy_c, p, Ho, Wo, flag, 1e-3)
        z = _bn_z(300, 32, g, dev)
        if bad == "z":
            z[17, 3] = float("nan")
        gamma, _ = _bn_params(32, g, dev)
        stats = torch.stack([z.float().mean(0), torch.ones(32, device=dev), torch.ones(32, device=dev)])
        _launch_bn_bwd(torch.randn(300, 32, generator=g).to(F16).to(dev), None, z, 32, stats, gamma, 1.0, 1e-3, flag)
        o = torch.randn(2, 8, 16, 4, generator=g).to(dev)
        if bad == "o":
            o[1, 2, 3, 1] = float("nan")
        _launch_loss(o, None, 1.0, False, flag)
        torch.cuda.synchronize()
        return int(flag)

    for bad in ("dy", "z", "o"):
        assert run_all(torch.zeros(1, dtype=torch.int32, device=dev), bad) == 1, bad
    assert run_all(torch.zeros(1, dtype=torch.int32, device=dev), None) == 0
    assert run_all(torch.ones(1, dtype=torch.int32, device=dev), None) == 1


# ---- exact kernels --------------------------------------------------------------------------------------------------

def test_prep_and_interleave_are_exact(cuda_device):
    L = _lib()
    dev = cuda_device
    g = torch.Generator().manual_seed(80)
    for B, H, W in ((2, 5, 7), (1, 64, 128)):
        src = (torch.randn(B, 3, H, W, generator=g) * 3).to(dev)
        dst = _nan((B, H, W, 16), F16, dev)
        L.check(L.lib().pf_faedt_prep(_vp(src), B, H, W, _vp(dst), _st()))
        torch.cuda.synchronize()
        assert _same(dst, ct.prep_ref(src))
    for B, H, W, Cc in ((2, 2, 4, 64), (2, 64, 128, 32), (1, 6, 10, 128)):
        ph = torch.randn(4, B, H // 2, W // 2, Cc, generator=g).to(F16).to(dev)
        dx = _nan((B, H, W, Cc), F16, dev)
        L.check(L.lib().pf_faedt_interleave(_vp(ph), B, H, W, Cc, _vp(dx), _st()))
        torch.cuda.synchronize()
        assert _same(dx, ct.interleave_ref(ph))


def _trainer_convs():
    """(cin, cout, k, stride, dgrad) of every distinct convolution FAEDTrainer packs."""
    return sorted({(cin, cout, k, s, not (cin == 3)) for cin, cout, k, s, *_ in trainer_layers(1, 64, 128)})


@pytest.mark.parametrize("conv", _trainer_convs(), ids=lambda c: f"{c[0]}-{c[1]}-k{c[2]}-s{c[3]}")
def test_pack_is_exact(cuda_device, conv):
    """Forward layout, stride-1 flipped kernel, the four stride-2 phase kernels and the zero padding, as
    FAEDTrainer._repack calls it (x_c, cw = max(cout, 32), dg [k^2][dy_c][cin])."""
    L = _lib()
    cin, cout, k, s, dgrad = conv
    dev = cuda_device
    x_c, dy_c, cw = (16 if cin == 3 else cin), (16 if cout == 3 else cout), max(cout, 32)
    w = torch.randn(cout, cin, k, k, generator=torch.Generator().manual_seed(cin + cout + k)).to(dev)
    fwd = _nan((k * k, x_c, cw), F16, dev)
    dg = _nan((k * k, dy_c, cin), F16, dev) if dgrad else None
    L.check(L.lib().pf_faedt_pack(_vp(w), cout, cin, k, s, _vp(fwd), x_c, cw, _vp(dg), dy_c, cin, _st()))
    torch.cuda.synchronize()
    rf, rd = ct.pack_ref(w, k, s, x_c, cw, dy_c, cin)
    assert _same(fwd, rf)
    assert dg is None or _same(dg, rd)


# ---- Adam and the step end ------------------------------------------------------------------------------------------

LR, BETAS, EPS = 1e-4, (0.9, 0.999), 1e-8


def _launch_adam(p, gr, m, v, run, pend, ctl, ictl, nb):
    L = _lib()
    L.check(L.lib().pf_faedt_adam(_vp(p), _vp(gr), _vp(m), _vp(v), _ll(p.numel()), _vp(run), _vp(pend),
                                  _ll(run.numel()), _vp(ctl), _vp(ictl), _vp(nb), C.c_double(BETAS[0]),
                                  C.c_double(BETAS[1]), C.c_double(EPS), _st()))


def _adam_state(dev, n=70001, n_run=513, seed=90):
    g = torch.Generator().manual_seed(seed)
    p = (torch.randn(n, generator=g) * 0.05).to(dev)
    run = torch.randn(n_run, generator=g).abs().to(dev)
    pend = torch.randn(n_run, generator=g).abs().to(dev)
    return g, p, run, pend


def test_adam_is_bit_equal_to_torch(cuda_device):
    """Steps 1, 2 and 3 from zero moments and step 100000 from given ones, n = 70001 (not a multiple of 256) with 513
    running statistics: p, exp_avg and exp_avg_sq equal torch.optim.Adam(foreach=False) bit for bit on the same device;
    the running statistics fold as 0.9 run + 0.1 pending within 3u; step, num_batches count up."""
    dev = cuda_device
    g, p, run, pend = _adam_state(dev)
    n = p.numel()
    tp = torch.nn.Parameter(p.clone())
    opt = torch.optim.Adam([tp], lr=LR, betas=BETAS, eps=EPS, foreach=False)
    m, v = torch.zeros(n, device=dev), torch.zeros(n, device=dev)
    ctl = torch.tensor([LR, 1.0], dtype=torch.float64, device=dev)
    ictl = torch.zeros(4, dtype=torch.int32, device=dev)
    nb = torch.zeros((), dtype=torch.int64, device=dev)
    for step in (1, 2, 3, 100000):
        gr = torch.randn(n, generator=g).to(dev) * (10.0 ** torch.randint(-6, 1, (n,), generator=g)).to(dev)
        if step == 100000:
            m = (torch.randn(n, generator=g) * 1e-3).to(dev)
            v = (torch.rand(n, generator=g) * 1e-5).to(dev)
            opt.state[tp] = {"step": torch.tensor(float(step - 1)), "exp_avg": m.clone(), "exp_avg_sq": v.clone()}
            ictl[0] = step - 1
        tp.grad = gr.clone()
        opt.step()
        run_before = run.clone()
        nb_before = int(nb)
        _launch_adam(p, gr, m, v, run, pend, ctl, ictl, nb)
        torch.cuda.synchronize()
        st = opt.state[tp]
        same = {"p": _same(p, tp.data), "exp_avg": _same(m, st["exp_avg"]), "exp_avg_sq": _same(v, st["exp_avg_sq"])}
        if not all(same.values()):
            diff = {k: int((_bits(a) != _bits(b)).sum()) for k, a, b in
                    (("p", p, tp.data), ("exp_avg", m, st["exp_avg"]), ("exp_avg_sq", v, st["exp_avg_sq"]))}
            print(f"[contract] adam step {step}: elements that differ {diff}")
        assert all(same.values()), (step, same)
        want = 0.9 * run_before.double() + 0.1 * pend.double()
        # fl32(0.1) and fl32(1 - fl32(0.1)) are within 0.25u and 0.44u of 0.1 and 0.9; the product and the fused add
        # round once each: 3u of the terms
        fold = float(((run.double() - want).abs() / (3 * ct.U * (0.9 * run_before.double() + 0.1 * pend.double()).abs()
                                                     + 2.0 ** -149)).max())
        assert fold <= 1.0, fold
        assert int(ictl[0]) == step and int(nb) == nb_before + 1 and int(ictl[3]) == 0
        print(f"[contract] adam step {step}: bit-equal to torch; running fold err/bound {fold:.3f}")


def test_flagged_step_changes_nothing_and_halves_the_scale(cuda_device):
    dev = cuda_device
    g, p, run, pend = _adam_state(dev, seed=91)
    n = p.numel()
    gr, m, v = torch.randn(n, generator=g).to(dev), torch.randn(n, generator=g).to(dev), torch.rand(n, generator=g).to(dev)
    ctl = torch.tensor([LR, 8.0], dtype=torch.float64, device=dev)
    ictl = torch.tensor([7, 123, 2, 1], dtype=torch.int32, device=dev)
    nb = torch.full((), 7, dtype=torch.int64, device=dev)
    before = [t.clone() for t in (p, m, v, run, nb)]
    _launch_adam(p, gr, m, v, run, pend, ctl, ictl, nb)
    torch.cuda.synchronize()
    assert all(_same(a, b) for a, b in zip((p, m, v, run, nb), before))
    assert ctl.tolist() == [LR, 4.0] and ictl.tolist() == [7, 0, 3, 0]


def test_clean_step_at_growth_tracker_1999_doubles_the_scale(cuda_device):
    """A checkpoint's faed_train.growth_tracker = 1999 and loss_scale = 4: one clean training_step doubles S to 8 and
    resets the tracker; from 1998 the step only counts."""
    from panfusion_b200.faed_train import FAEDTrainer, init_state
    pano = (torch.rand(1, 3, 32, 64, generator=torch.Generator().manual_seed(3)) * 2 - 1).to(cuda_device)
    for tracker, want_scale, want_tracker in ((1999, 8.0, 0), (1998, 4.0, 1999)):
        ck = {"state_dict": init_state(0), "faed_train": {"growth_tracker": tracker, "loss_scale": 4.0}}
        tr = FAEDTrainer(ck, device=cuda_device)
        tr.training_step(pano)
        torch.cuda.synchronize()
        assert tr.skipped_steps == 0 and tr.loss_scale == want_scale and int(tr.ictl[1]) == want_tracker, \
            (tracker, tr.loss_scale, int(tr.ictl[1]))


# ---- the table covers the trainer -----------------------------------------------------------------------------------

def _launch_all_cases(dev):
    """Every case above once, launches only."""
    g = torch.Generator().manual_seed(0)
    flag = torch.zeros(1, dtype=torch.int32, device=dev)
    for build in list(WGRAD_CASES.values()) + [lambda: [CAPPED]]:
        for s in build():
            x, dy, x_c, dy_c, p, Ho, Wo = _wgrad_operands(s, g, dev)
            _launch_wgrad(s, x, dy, x_c, dy_c, p, Ho, Wo, flag, 1e-3)
            del x, dy
    for Cc in (32, 64, 128):
        z = _bn_z(300, Cc, g, dev)
        gamma, beta = _bn_params(Cc, g, dev)
        _, stats, _ = _launch_bn_stats(z, Cc)
        out = _launch_bn_apply(z, Cc, stats, gamma, beta, True, None)
        _launch_bn_apply(z, Cc, stats, gamma, beta, False, z)
        for mask in (out, None):
            _launch_bn_bwd(z, mask, z, Cc, stats, gamma, 1.0, 1e-3, flag)
    _launch_up(torch.zeros(1, 2, 2, 32, dtype=F16, device=dev), torch.zeros(1, 4, 4, 32, dtype=F16, device=dev))
    o = torch.zeros(1, 2, 2, 4, device=dev)
    for t in (torch.zeros(1, 3, 2, 2, device=dev), None):
        for with_pred in (True, False):
            _launch_loss(o, t, 1.0, with_pred, flag)
    test_prep_and_interleave_are_exact(dev)
    for conv in _trainer_convs():
        test_pack_is_exact(dev, conv)
    test_flagged_step_changes_nothing_and_halves_the_scale(dev)
    torch.cuda.synchronize()


def test_faedt_call_table_covers_the_trainer(recorder, cuda_device):
    """Every call class of one training_step at B = 2, 64 x 128, one at B = 1, 32 x 96, and one reconstruct is one a
    case above launches."""
    from panfusion_b200.faed_train import FAEDTrainer
    dev = cuda_device
    _launch_all_cases(dev)
    covered = set(recorder.calls)
    recorder.calls.clear()
    g = torch.Generator().manual_seed(1)
    tr = FAEDTrainer(seed=0, device=dev)
    for B, H, W in ((2, 64, 128), (1, 32, 96)):
        tr.training_step((torch.rand(B, 3, H, W, generator=g) * 2 - 1).to(dev))
    tr.reconstruct((torch.rand(1, 3, 64, 128, generator=g) * 2 - 1).to(dev))
    torch.cuda.synchronize()
    seen = set(recorder.calls)
    assert {c[0] for c in seen} == set(ENTRIES), "the trainer made no call of one of the entry points"
    for c in sorted(seen, key=str):
        print(f"[contract] faedt call class {c}{'' if c in covered else '  <- no case'}")
    missing = sorted(seen - covered, key=str)
    assert not missing, f"call classes without a contract case: {missing}"
