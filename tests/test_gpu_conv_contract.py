"""-m gpu: the implicit-GEMM convolution of csrc/conv_mma.cuh through all four of its entry points (pf_conv_circ,
pf_faedt_conv, pf_conv2d_nhwc, pf_hnet_conv), against the fp64 restatement tests/_contract.py:conv_ref with a bound
scaled by each element's own magnitude.

CONV_CASES has one case per compiled kernel (entry point x <KC, BN> instantiation, 20 in all). Each case launches the
layer shapes its models make plus the edges where a tile or address computation can go wrong: B >= 2 with a last
128-row tile that is partial and a tile that spans two images, ReLU on and off, a residual and an fp32 output wherever
the entry point takes them, Cout < Cw, output slices, the smallest W a circular pad allows, the deepest K. Weights are
packed by the packers the models use. Every output is NaN-filled over all the rows the grid covers (and, for the
stride-2 data gradient, over all four phase buffers), so a store outside the contract fails as well.
`test_conv_call_table_covers_the_models` keeps the table honest: every call class the FAED encoder, one FAED training
step, InceptionV3 and HorizonNet make must have a case here."""
import ctypes as C
import math

import pytest
import torch

import _contract as ct

pytestmark = pytest.mark.gpu

ENTRIES = ("pf_conv_circ", "pf_faedt_conv", "pf_conv2d_nhwc", "pf_hnet_conv")
BM = 128  # output pixels per CTA


def _given(p) -> bool:
    return p is not None and (p.value if isinstance(p, C.c_void_p) else p) not in (None, 0)


def _conv2d_inst(cin, cout):
    """pf_conv2d_nhwc's selection: KC by Cin % 64 / % 32, the N tile by pf_conv2d_packed_cout."""
    kc = 64 if cin % 64 == 0 else (32 if cin % 32 == 0 else 16)
    cw = 32 if cout <= 32 else (cout + 63) // 64 * 64
    if cw == 32:
        return (16 if kc == 16 else 32, 32)
    return (kc, 64)


def call_class(entry, a):
    """(entry, (KC, BN), stride kind, (kh, kw), relu, residual given, output dtype, sliced output) of one call's
    arguments, with each entry point's own instantiation rule."""
    dt = lambda code: "f32" if code == 0 else "f16"  # PF_F32 / PF_F16
    if entry == "pf_conv_circ":
        _x, _B, _H, _W, cin, _w, _b, cout, k, s, _p, relu, res, _o, odt, _st = a
        return (entry, (64 if cin >= 64 else cin, cout), f"{s}x{s}", (k, k), bool(relu), _given(res), dt(odt), False)
    if entry == "pf_faedt_conv":
        _x, _B, _H, _W, cin, _w, _b, cout, cw, kh, kw, s, _ph, _pw, _Ho, _Wo, res, _o, ld, odt, _st = a
        kind = "phase" if (kh, kw) == (2, 2) else f"{s}x{s}"  # the stride-2 data gradient's 2x2 phase convolutions
        return (entry, (64 if cin >= 64 else cin, cw), kind, (kh, kw), False, _given(res), dt(odt), ld != cout)
    if entry == "pf_conv2d_nhwc":
        _x, _B, _H, _W, cin, _w, _b, cout, kh, kw, s, _ph, _pw, relu, _o, odt, ld, off, _st = a
        return (entry, _conv2d_inst(cin, cout), f"{s}x{s}", (kh, kw), bool(relu), False, dt(odt),
                ld != cout or off != 0)
    _x, _B, _H, _W, cin, _w, _b, cout, k, sh, sw, relu, res, _o, odt, _st = a
    inst = (16, 64) if cin == 16 else {32: (32, 32), 64: (64, 64)}.get(cout, (64, 128))
    return (entry, inst, f"{sh}x{sw}", (k, k), bool(relu), _given(res), dt(odt), False)


class _Recorder:
    """Stands in for the library handle: records the arguments of every call of the four entry points and forwards
    every call."""

    def __init__(self, lib):
        self._lib, self.calls = lib, []

    def __getattr__(self, name):
        f = getattr(self._lib, name)
        if name not in ENTRIES:
            return f

        def rec(*args):
            self.calls.append((name, args))
            return f(*args)
        return rec


@pytest.fixture
def recorder(monkeypatch, cuda_device):
    from panfusion_b200 import _lib
    rec = _Recorder(_lib.lib())
    monkeypatch.setattr(_lib, "lib", lambda: rec)
    return rec


# ---- launch specs ---------------------------------------------------------------------------------------------------
# A spec is a dict of the launch's arguments; the helpers below fill in each entry point's fixed ones.

def circ(B, H, W, cin, cout, k, s=1, relu=True, res=False, f32=False, off=0.0, cin_real=None):
    p = 1 if s == 2 else k // 2
    return dict(entry="pf_conv_circ", B=B, H=H, W=W, cin=cin, cin_real=cin_real or cin, cout=cout, kh=k, kw=k, sh=s,
                sw=s, ph=p, pw=p, relu=relu, res=res, f32=f32, off=off)


def conv2d(B, H, W, cin, cout, kh, kw, s=1, ph=0, pw=0, relu=True, f32=False, ld=None, out_off=0, off=0.0,
           cin_real=None):
    return dict(entry="pf_conv2d_nhwc", B=B, H=H, W=W, cin=cin, cin_real=cin_real or cin, cout=cout, kh=kh, kw=kw,
                sh=s, sw=s, ph=ph, pw=pw, relu=relu, res=False, f32=f32, ld=ld or cout, out_off=out_off, off=off)


def hnet(B, H, W, cin, cout, k, sh=1, sw=1, relu=True, res=False, f32=False, off=0.0, cin_real=None):
    return dict(entry="pf_hnet_conv", B=B, H=H, W=W, cin=cin, cin_real=cin_real or cin, cout=cout, kh=k, kw=k, sh=sh,
                sw=sw, ph=k // 2, pw=k // 2, relu=relu, res=res, f32=f32, off=off)


def ft_fwd(B, H, W, cin, cout, k, s=1, f32=False, cw=None, ld=None, Wo=None, off=0.0):
    """FAEDTrainer._conv: weights packed by pf_faedt_pack from the fp32 [cout, cin, k, k] parameters; cin = 3 is
    stored as 16 channels and cout = 3 as 4 (Cw 32). Wo (default: the layer's own) may run up to the wrap limit."""
    p = 1 if s == 2 else k // 2
    x_c, out_c = (16 if cin == 3 else cin), (4 if cout == 3 else cout)
    Ho = (H + 2 * p - k) // s + 1
    return dict(entry="pf_faedt_conv", kind="fwd", B=B, H=H, W=W, cin=x_c, cin_real=cin, cout=out_c, fcout=cout,
                fk=k, fs=s, cw=cw or max(cout, 32), kh=k, kw=k, sh=s, sw=s, ph=p, pw=p, Ho=Ho,
                Wo=Wo or (W + 2 * p - k) // s + 1, relu=False, res=False, f32=f32, ld=ld or out_c, off=off)


def ft_dgrad(B, H, W, cin, cout, k, s=1, res=False, off=0.0):
    """FAEDTrainer._dgrad of the forward layer cin -> cout (k, s) on an H x W input: the stride-1 adjoint, or the four
    2x2 phase convolutions (pads (1 - r, 1 - c)) of the stride-2 one, with pf_faedt_pack's data-gradient weights."""
    p = 1 if s == 2 else k // 2
    ho, wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    dy_c = 16 if cout == 3 else cout
    base = dict(entry="pf_faedt_conv", B=B, H=ho, W=wo, cin=dy_c, cin_real=dy_c, cout=cin, cw=cin, fcin=cin,
                fcout=cout, fk=k, fs=s, sh=1, sw=1, relu=False, f32=False, ld=cin, off=off)
    if s == 1:
        return dict(base, kind="dgrad", kh=k, kw=k, ph=p, pw=p, Ho=H, Wo=W, res=res)
    assert not res
    return dict(base, kind="phases", kh=2, kw=2, ph=None, pw=None, Ho=ho, Wo=wo, res=False)


def _out_hw(s):
    if "Ho" in s:
        return s["Ho"], s["Wo"]
    return (s["H"] + 2 * s["ph"] - s["kh"]) // s["sh"] + 1, (s["W"] + 2 * s["pw"] - s["kw"]) // s["sw"] + 1


def _phase_pads(s):
    return [(1 - r, 1 - c) for r in (0, 1) for c in (0, 1)] if s.get("kind") == "phases" else [(s["ph"], s["pw"])]


def _args(s, x=None, w=None, bias=None, res=None, out=None, pads=None):
    """The C-ABI argument tuple of the spec's launch (pointers as c_void_p)."""
    vp = lambda t: C.c_void_p(0 if t is None else t.data_ptr())
    ph, pw = pads or (s["ph"], s["pw"])
    odt = 0 if s["f32"] else 1
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream if x is not None else 0)
    e = s["entry"]
    rp = vp(res) if s["res"] else vp(None)
    if x is None:  # static class of the spec: any non-null pointer for a given residual
        rp = C.c_void_p(1) if s["res"] else C.c_void_p(0)
    if e == "pf_conv_circ":
        return (vp(x), s["B"], s["H"], s["W"], s["cin"], vp(w), vp(bias), s["cout"], s["kh"], s["sh"], ph,
                int(s["relu"]), rp, vp(out), odt, st)
    if e == "pf_faedt_conv":
        Ho, Wo = _out_hw(s)
        return (vp(x), s["B"], s["H"], s["W"], s["cin"], vp(w), vp(bias), s["cout"], s["cw"], s["kh"], s["kw"],
                s["sh"], ph, pw, Ho, Wo, rp, vp(out), s["ld"], odt, st)
    if e == "pf_conv2d_nhwc":
        return (vp(x), s["B"], s["H"], s["W"], s["cin"], vp(w), vp(bias), s["cout"], s["kh"], s["kw"], s["sh"], ph, pw,
                int(s["relu"]), vp(out), odt, s["ld"], s["out_off"], st)
    return (vp(x), s["B"], s["H"], s["W"], s["cin"], vp(w), vp(bias), s["cout"], s["kh"], s["sh"], s["sw"],
            int(s["relu"]), rp, vp(out), odt, st)


def spec_classes(s):
    return {call_class(s["entry"], _args(s, pads=p)) for p in _phase_pads(s)}


def _operands(s, g, dev):
    """(x, [packed weight per launch], bias) built the way the spec's call site builds them."""
    from panfusion_b200 import _lib, faed, horizonnet, inception
    B, H, W = s["B"], s["H"], s["W"]
    x = torch.zeros(B, H, W, s["cin"])
    x[..., :s["cin_real"]] = torch.randn(B, H, W, s["cin_real"], generator=g) + s["off"]
    x = x.half().to(dev)
    e = s["entry"]
    if e == "pf_faedt_conv":
        cin, cout, k = s.get("fcin", s["cin_real"]), s["fcout"], s["fk"]
        wf = (torch.randn(cout, cin, k, k, generator=g) / math.sqrt(cin * k * k)).to(dev)
        x_c = 16 if cin == 3 else cin
        cw = s["cw"] if s["kind"] == "fwd" else max(cout, 32)
        fwd = torch.empty(k * k, x_c, cw, device=dev, dtype=torch.float16)
        dg = None if s["kind"] == "fwd" else torch.empty(k * k, 16 if cout == 3 else cout, cin, device=dev,
                                                         dtype=torch.float16)
        _lib.check(_lib.lib().pf_faedt_pack(C.c_void_p(wf.data_ptr()), cout, cin, k, s["fs"], C.c_void_p(fwd.data_ptr()),
                                            x_c, cw, C.c_void_p(0 if dg is None else dg.data_ptr()),
                                            0 if dg is None else dg.shape[1], 0 if dg is None else cin,
                                            C.c_void_p(torch.cuda.current_stream().cuda_stream)))
        ws = [fwd] if s["kind"] == "fwd" else ([dg] if s["kind"] == "dgrad" else [dg[4 * i:4 * i + 4] for i in range(4)])
        # the trainer's data gradients carry no bias (a zero vector); the forward layers carry theirs
        bias = torch.zeros(s["cw"]) if s["kind"] != "fwd" else torch.randn(s["cw"], generator=g) * 0.5
        return x, ws, bias.to(dev)
    w = torch.randn(s["cout"], s["cin_real"], s["kh"], s["kw"], generator=g, dtype=torch.float64)
    w /= math.sqrt(s["cin_real"] * s["kh"] * s["kw"])
    if e == "pf_conv_circ":
        wp = faed.pack_weight(w, s["cin"], torch.float16)
    elif e == "pf_conv2d_nhwc":
        wp = inception.pack_weight(w, s["cin"])
    else:
        wp = horizonnet.pack_weight(w, s["cin"])
    bias = torch.randn(wp.shape[2], generator=g) * 0.5  # also past Cout: a kernel must not read or store those
    return x, [wp.to(dev)], bias.to(dev)


def run_spec(s, g, dev, name):
    """Launch the spec on NaN-filled outputs -> [(label, got, ref, bound)]."""
    from panfusion_b200 import _lib
    x, ws, bias = _operands(s, g, dev)
    Ho, Wo = _out_hw(s)
    M = s["B"] * Ho * Wo
    rows = -(-M // BM) * BM  # every row the grid covers
    cout, ld = s["cout"], s.get("ld", s["cout"])
    odt = torch.float32 if s["f32"] else torch.float16
    res = (torch.randn(M, cout, generator=g) * 0.7).half().to(dev) if s["res"] else None
    pads = _phase_pads(s)
    n = len(pads)
    out = torch.full((n * rows, ld), float("nan"), dtype=odt, device=dev)
    ref = torch.full((n * rows, ld), float("nan"), dtype=torch.float64, device=dev)
    bound = ref.clone()
    for i, (ph, pw) in enumerate(pads):
        _lib.check(getattr(_lib.lib(), s["entry"])(*_args(s, x, ws[i], bias, res, out[i * rows:], (ph, pw))))
        r, b = ct.conv_ref(x, ws[i], bias, Cout=cout, kh=s["kh"], kw=s["kw"], stride_h=s["sh"], stride_w=s["sw"],
                           ph=ph, pw=pw, circ=s["entry"] != "pf_conv2d_nhwc", relu=s["relu"], out_dtype=odt,
                           residual=res, res_before_relu=s["entry"] == "pf_hnet_conv", Ho=Ho, Wo=Wo, out_rows=rows,
                           out_ld=ld, out_off=s.get("out_off", 0))
        ref[i * rows:(i + 1) * rows], bound[i * rows:(i + 1) * rows] = r, b
    return (name, out, ref, bound), (x, ws, bias, res)


def _label(s):
    k = f"{s['kh']}x{s['kw']}"
    parts = [f"B{s['B']} {s['H']}x{s['W']}", f"{s['cin']}->{s['cout']}", k, f"s{s['sh']}x{s['sw']}"]
    if s.get("kind") in ("dgrad", "phases"):
        parts.append(s["kind"])
    if s["relu"]:
        parts.append("relu")
    if s["res"]:
        parts.append("res")
    if s["f32"]:
        parts.append("f32")
    if s.get("ld", s["cout"]) != s["cout"] or s.get("out_off", 0):
        parts.append(f"slice[{s.get('out_off', 0)}:+{s['cout']}]/{s['ld']}")
    if s["off"]:
        parts.append(f"mean {s['off']}")
    return " ".join(parts)


# ---- the case table: one case per kernel ----------------------------------------------------------------------------
# Shapes: B = 3 (or 2) images of Ho x Wo = 30..120 pixels, so M is not a multiple of 128 and a 128-row tile spans two
# or more images; the K of each entry point's deepest layer is in its <64, BN> cases.

CONV_CASES = {
    # FAED encoder (faed.py): stride-1 k 3/5/7/9 ResBlocks (ReLU / residual), stride-2 k4 ConvBlocks, fp32 `fuse`
    "circ <16,32>": ("pf_conv_circ", (16, 32), [
        circ(3, 6, 20, 16, 32, 9, relu=False, cin_real=3), circ(3, 6, 20, 16, 32, 9, off=0.5),
        circ(2, 5, 5, 16, 32, 9, res=True, f32=True)]),  # W = pad + 1
    "circ <32,32>": ("pf_conv_circ", (32, 32), [
        circ(3, 6, 20, 32, 32, 9), circ(3, 6, 20, 32, 32, 9, relu=False, res=True, off=0.5),
        circ(2, 7, 5, 32, 32, 9, f32=True, relu=False), circ(3, 12, 20, 32, 32, 4, s=2)]),
    "circ <32,64>": ("pf_conv_circ", (32, 64), [
        circ(3, 12, 20, 32, 64, 4, s=2, off=0.5), circ(2, 4, 2, 32, 64, 4, s=2, relu=False, f32=True),
        circ(3, 6, 20, 32, 64, 3, relu=False, res=True)]),
    "circ <64,64>": ("pf_conv_circ", (64, 64), [
        circ(3, 6, 20, 64, 64, 7), circ(3, 6, 20, 64, 64, 7, relu=False, res=True, off=0.5),
        circ(2, 5, 4, 64, 64, 7, f32=True), circ(3, 12, 20, 64, 64, 4, s=2, relu=False)]),
    "circ <64,128>": ("pf_conv_circ", (64, 128), [
        circ(3, 12, 20, 64, 128, 4, s=2, off=0.5), circ(3, 12, 20, 128, 128, 4, s=2), circ(2, 2, 2, 128, 128, 4, s=2),
        circ(3, 6, 20, 128, 128, 5), circ(3, 6, 20, 128, 128, 5, relu=False, res=True),  # K = 25 x 128
        circ(3, 6, 20, 128, 128, 3), circ(3, 6, 20, 128, 128, 3, relu=False, res=True, off=0.5),
        circ(3, 6, 20, 128, 128, 3, relu=False, f32=True), circ(2, 3, 2, 128, 128, 3, res=True, f32=True)]),
    # FAED autoencoder training (faed_train.py): forward layers, stride-1 data gradients (the ResBlock conv1's with
    # the block's residual), the stride-2 data gradients' four phases; Cout < Cw and out_ld > Cout; the wrap limit
    "ft <16,32>": ("pf_faedt_conv", (16, 32), [
        ft_fwd(3, 6, 20, 3, 32, 9), ft_fwd(2, 5, 5, 3, 32, 9, Wo=6, off=0.5),  # (Wo - 1) + 8 - 4 = 2W - 1
        ft_fwd(3, 6, 20, 3, 26, 9, cw=32, ld=30, f32=True),
        ft_dgrad(3, 6, 20, 32, 3, 9)]),  # outconv_rgb's adjoint: 16 stored gradient channels
    "ft <32,32>": ("pf_faedt_conv", (32, 32), [
        ft_fwd(3, 6, 20, 32, 32, 9), ft_fwd(3, 6, 20, 32, 3, 9, f32=True, off=0.5),  # outconv_rgb: Cout 4 of Cw 32
        ft_fwd(3, 6, 20, 32, 3, 9), ft_fwd(3, 6, 20, 32, 20, 9, cw=32, ld=24),
        ft_dgrad(3, 6, 20, 32, 32, 9), ft_dgrad(3, 6, 20, 32, 32, 9, res=True, off=0.5)]),
    "ft <32,64>": ("pf_faedt_conv", (32, 64), [
        ft_fwd(3, 12, 20, 32, 64, 4, s=2), ft_fwd(2, 4, 2, 32, 64, 4, s=2, f32=True),
        ft_fwd(3, 12, 20, 32, 40, 4, s=2, cw=64, ld=42),
        ft_dgrad(3, 6, 20, 64, 32, 3), ft_dgrad(3, 6, 20, 64, 32, 3, res=True)]),
    "ft <64,32>": ("pf_faedt_conv", (64, 32), [
        ft_fwd(3, 6, 20, 64, 32, 3), ft_fwd(3, 6, 20, 64, 32, 3, f32=True, off=0.5),
        ft_fwd(3, 6, 20, 64, 10, 3, cw=32, ld=12),
        ft_dgrad(3, 12, 20, 32, 64, 4, s=2), ft_dgrad(2, 4, 4, 32, 64, 4, s=2, off=0.5)]),
    "ft <64,64>": ("pf_faedt_conv", (64, 64), [
        ft_fwd(3, 6, 20, 64, 64, 7), ft_fwd(3, 6, 20, 128, 64, 3), ft_fwd(3, 6, 20, 64, 64, 7, f32=True),
        ft_fwd(3, 6, 20, 64, 30, 7, cw=64, ld=34),  # column tile 32..63 of the warp's half skipped whole
        ft_dgrad(3, 6, 20, 64, 64, 7), ft_dgrad(3, 6, 20, 64, 64, 7, res=True, off=0.5),
        ft_dgrad(3, 12, 20, 64, 128, 4, s=2)]),
    "ft <64,128>": ("pf_faedt_conv", (64, 128), [
        ft_fwd(3, 12, 20, 64, 128, 4, s=2), ft_fwd(3, 12, 20, 128, 128, 4, s=2, off=0.5),
        ft_fwd(3, 6, 20, 128, 128, 5), ft_fwd(3, 6, 20, 128, 128, 3), ft_fwd(3, 6, 20, 128, 128, 3, f32=True),
        ft_fwd(3, 6, 20, 128, 58, 5, cw=128, ld=64),
        ft_dgrad(3, 6, 20, 128, 128, 3), ft_dgrad(3, 6, 20, 128, 128, 3, res=True),
        ft_dgrad(3, 6, 20, 128, 128, 5), ft_dgrad(3, 6, 20, 128, 128, 5, res=True, off=0.5),  # K = 25 x 128
        ft_dgrad(3, 6, 20, 128, 64, 3), ft_dgrad(3, 12, 20, 128, 128, 4, s=2)]),
    # FID InceptionV3 (inception.py): ReLU, fp16 (Mixed_7c: fp32) into column slices of the block's concat buffer
    "conv2d <16,32>": ("pf_conv2d_nhwc", (16, 32), [
        conv2d(3, 13, 13, 16, 32, 3, 3, s=2, cin_real=3), conv2d(3, 9, 14, 16, 24, 3, 3, relu=False, f32=True),
        conv2d(3, 9, 14, 48, 30, 1, 1, ld=64, out_off=32, off=0.5)]),
    "conv2d <32,32>": ("pf_conv2d_nhwc", (32, 32), [
        conv2d(3, 13, 13, 32, 32, 3, 3), conv2d(3, 9, 14, 192, 32, 1, 1, ld=256, out_off=224, off=0.5),
        conv2d(3, 9, 14, 96, 24, 3, 3, ph=1, pw=1, relu=False, f32=True, ld=40, out_off=6)]),
    "conv2d <16,64>": ("pf_conv2d_nhwc", (16, 64), [
        conv2d(3, 13, 13, 80, 192, 3, 3), conv2d(3, 9, 14, 48, 64, 5, 5, ph=2, pw=2, ld=288, out_off=64, off=0.5),
        conv2d(3, 9, 14, 48, 80, 3, 3, s=2, relu=False, f32=True, ld=86, out_off=2)]),
    "conv2d <32,64>": ("pf_conv2d_nhwc", (32, 64), [
        conv2d(3, 13, 13, 32, 64, 3, 3, ph=1, pw=1), conv2d(3, 9, 14, 96, 96, 3, 3, ph=1, pw=1, ld=288, out_off=128),
        conv2d(3, 9, 14, 288, 64, 1, 1, ld=288, out_off=224), conv2d(3, 9, 14, 288, 48, 1, 1, off=0.5),
        conv2d(3, 17, 17, 288, 384, 3, 3, s=2, ld=768, out_off=0), conv2d(3, 17, 17, 96, 96, 3, 3, s=2, ld=768, out_off=384),
        conv2d(3, 9, 14, 160, 160, 1, 7, pw=3), conv2d(3, 9, 14, 160, 160, 7, 1, ph=3),
        conv2d(3, 9, 14, 160, 192, 7, 1, ph=3, ld=768, out_off=192), conv2d(3, 9, 14, 160, 192, 1, 7, pw=3, ld=768, out_off=384),
        conv2d(3, 9, 14, 160, 320, 1, 7, pw=3, relu=False, f32=True, off=0.5)]),
    "conv2d <64,64>": ("pf_conv2d_nhwc", (64, 64), [
        conv2d(3, 9, 14, 64, 80, 1, 1), conv2d(3, 9, 14, 64, 96, 3, 3, ph=1, pw=1, off=0.5),
        conv2d(3, 9, 14, 192, 64, 1, 1, ld=256, out_off=0), conv2d(3, 9, 14, 768, 128, 1, 7, pw=3),
        conv2d(3, 9, 14, 128, 128, 7, 1, ph=3), conv2d(3, 9, 14, 128, 192, 7, 1, ph=3, ld=768, out_off=192),
        conv2d(3, 9, 14, 192, 192, 1, 7, pw=3, ld=768, out_off=384), conv2d(3, 17, 17, 192, 320, 3, 3, s=2, ld=1280),
        conv2d(3, 9, 14, 1280, 320, 1, 1, ld=2048), conv2d(3, 9, 14, 384, 384, 1, 3, pw=1, ld=2048, out_off=320),
        conv2d(3, 9, 14, 384, 384, 3, 1, ph=1, ld=2048, out_off=704),
        conv2d(3, 9, 14, 448, 384, 3, 3, ph=1, pw=1, off=0.5),  # K = 9 x 448
        conv2d(3, 9, 14, 2048, 320, 1, 1, f32=True, ld=2048), conv2d(3, 9, 14, 384, 384, 1, 3, pw=1, f32=True, ld=2048, out_off=1088),
        conv2d(3, 9, 14, 384, 384, 3, 1, ph=1, f32=True, ld=2048, out_off=1472),
        conv2d(3, 9, 14, 2048, 192, 1, 1, f32=True, ld=2048, out_off=1856), conv2d(3, 9, 14, 64, 48, 3, 3, relu=False)]),
    # HorizonNet (horizonnet.py): stem, bottlenecks (residual before the ReLU, shortcut without ReLU), ConvCompressH
    "hnet <16,64>": ("pf_hnet_conv", (16, 64), [
        hnet(3, 24, 28, 16, 64, 7, 2, 2, cin_real=3), hnet(2, 10, 4, 16, 64, 7, 2, 2, relu=False, res=True, f32=True),
        hnet(3, 12, 10, 16, 64, 3, 2, 1, res=True, off=0.5)]),  # W = pad + 1
    "hnet <32,32>": ("pf_hnet_conv", (32, 32), [
        hnet(3, 12, 20, 64, 32, 3, 2, 1), hnet(3, 12, 20, 64, 32, 3, 2, 1, relu=False, f32=True, off=0.5),
        hnet(3, 6, 20, 64, 32, 1, res=True), hnet(2, 6, 2, 128, 32, 3, res=True, relu=False)]),
    "hnet <64,64>": ("pf_hnet_conv", (64, 64), [
        hnet(3, 6, 20, 64, 64, 1), hnet(3, 6, 20, 256, 64, 1, off=0.5), hnet(3, 6, 20, 64, 64, 3),
        hnet(3, 12, 20, 128, 64, 3, 2, 1), hnet(3, 12, 20, 64, 64, 3, 2, 2, res=True, f32=True),
        hnet(3, 6, 20, 64, 64, 1, relu=False, res=True, off=0.5), hnet(2, 6, 2, 64, 64, 3, res=True)]),
    "hnet <64,128>": ("pf_hnet_conv", (64, 128), [
        hnet(3, 6, 20, 64, 256, 1, res=True), hnet(3, 6, 20, 64, 256, 1, relu=False), hnet(3, 6, 20, 256, 128, 1),
        hnet(3, 12, 20, 128, 128, 3, 2, 2), hnet(3, 12, 20, 256, 512, 1, 2, 2, relu=False, off=0.5),
        hnet(3, 6, 20, 128, 128, 3, off=0.5), hnet(3, 12, 20, 256, 128, 3, 2, 1),
        hnet(2, 6, 10, 2048, 1024, 3, 2, 1, off=0.5),  # K = 9 x 2048, the deepest of any model
        hnet(3, 6, 20, 128, 512, 1, relu=False, res=True, f32=True), hnet(2, 6, 2, 128, 128, 3, 1, 1, res=True)]),
}

CASE_CLASSES = {name: set().union(*(spec_classes(s) for s in specs)) for name, (_e, _i, specs) in CONV_CASES.items()}


def test_table_names_all_twenty_kernels():
    """The table has one case per kernel, every case reaches only its own, and each meets the M-tile edges."""
    kernels = {(e, inst) for e, inst, _ in CONV_CASES.values()}
    assert len(kernels) == len(CONV_CASES) == 20
    for name, (entry, inst, specs) in CONV_CASES.items():
        assert {c[:2] for c in CASE_CLASSES[name]} == {(entry, inst)}, name
        edges = False
        for s in specs:
            Ho, Wo = _out_hw(s)
            edges |= s["B"] >= 2 and (s["B"] * Ho * Wo) % BM != 0 and (Ho * Wo) % BM != 0
        assert edges, f"{name}: no launch with B >= 2, a partial last tile and a tile spanning two images"


@pytest.mark.parametrize("case", list(CONV_CASES))
def test_conv_contract(recorder, case):
    entry, inst, specs = CONV_CASES[case]
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(sum(map(ord, case)))
    checks = []
    for s in specs:
        checks.append(run_spec(s, g, dev, _label(s))[0])
    logged = {call_class(n, a) for n, a in recorder.calls}
    assert logged == CASE_CLASSES[case], f"the case makes calls of classes {logged}, declared {CASE_CLASSES[case]}"
    torch.cuda.synchronize()
    worst = 0.0
    for name, got, ref, bound in checks:
        r = ct.worst_ratio(got, ref, bound)
        print(f"[contract] conv {case} / {name}: worst err/bound {r:.3f}")
        worst = max(worst, r)
    assert worst <= 1.0, worst


def test_faed_last_layer_fourth_column_is_the_bias(recorder):
    """outconv_rgb: Cout = 4 of Cw = 32 for 3 real channels; column 3 is exactly bias[3] (its weights are zero)."""
    s = ft_fwd(2, 6, 20, 32, 3, 9, f32=True)
    (name, out, ref, bound), (_x, _ws, bias, _r) = run_spec(s, torch.Generator().manual_seed(3), torch.device("cuda:0"),
                                                           "outconv_rgb")
    M = 2 * 6 * 20
    assert torch.equal(out[:M, 3], bias[3].expand(M))
    assert ct.worst_ratio(out, ref, bound) <= 1.0


@pytest.mark.parametrize("entry", ["pf_conv_circ", "pf_faedt_conv", "pf_hnet_conv"])
def test_circular_wrap_limits_are_refused(cuda_device, entry):
    """One step past what a single conditional wrap handles is an argument error, and launches nothing."""
    from panfusion_b200 import _lib
    dev = cuda_device
    if entry == "pf_conv_circ":
        s = circ(1, 4, 4, 32, 32, 9)  # pad 4 needs W > 4
    elif entry == "pf_hnet_conv":
        s = hnet(1, 8, 3, 64, 64, 7)  # pad 3 needs W > 3
    else:
        s = ft_fwd(1, 5, 5, 32, 32, 9, Wo=7)  # (Wo - 1) + 8 - 4 = 2W: wraps twice
    x = torch.zeros(1, s["H"], s["W"], s["cin"], dtype=torch.float16, device=dev)
    w = torch.zeros(s["kh"] * s["kw"], s["cin"], 128, dtype=torch.float16, device=dev)
    b = torch.zeros(128, device=dev)
    out = torch.full((64, s["cout"]), float("nan"), dtype=torch.float16, device=dev)
    with pytest.raises(ValueError):
        _lib.check(getattr(_lib.lib(), entry)(*_args(s, x, w, b, None, out)))
    torch.cuda.synchronize()
    assert torch.isnan(out).all()


FULL_RES = {
    "circ 512x1024 downconv1": circ(1, 512, 1024, 16, 32, 9, relu=False, cin_real=3),
    "ft 512x1024 downconv1": ft_fwd(1, 512, 1024, 3, 32, 9),
    "conv2d 299x299 Conv2d_1a": conv2d(1, 299, 299, 16, 32, 3, 3, s=2, cin_real=3),
    "hnet 512x1024 stem": hnet(1, 512, 1024, 16, 64, 7, 2, 2, cin_real=3),
}


@pytest.mark.parametrize("case", list(FULL_RES))
def test_conv_contract_full_resolution(cuda_device, case):
    """The first layer of each model at the model's own resolution, where the index arithmetic is largest."""
    g = torch.Generator().manual_seed(sum(map(ord, case)))
    (name, out, ref, bound), _ = run_spec(FULL_RES[case], g, cuda_device, case)
    r = ct.worst_ratio(out, ref, bound)
    print(f"[contract] conv full resolution {case}: worst err/bound {r:.3f}")
    assert r <= 1.0, r


@pytest.mark.parametrize("case", list(CONV_CASES))
def test_conv_repeat_and_batch_invariance(cuda_device, case):
    """A repeat launch is bit-identical, and each image alone equals the same image inside the batch."""
    from panfusion_b200 import _lib
    s = CONV_CASES[case][2][0]
    g = torch.Generator().manual_seed(7)
    (_n, out, _r, _b), (x, ws, bias, res) = run_spec(s, g, cuda_device, case)
    Ho, Wo = _out_hw(s)
    M, P = s["B"] * Ho * Wo, Ho * Wo
    again = torch.full_like(out, float("nan"))
    _lib.check(getattr(_lib.lib(), s["entry"])(*_args(s, x, ws[0], bias, res, again, _phase_pads(s)[0])))
    for b in range(s["B"]):
        one = torch.full((P, out.shape[1]), float("nan"), dtype=out.dtype, device=cuda_device)
        s1 = dict(s, B=1)
        r1 = None if res is None else res[b * P:(b + 1) * P]
        _lib.check(getattr(_lib.lib(), s["entry"])(*_args(s1, x[b:b + 1], ws[0], bias, r1, one,
                                                             _phase_pads(s)[0])))
        assert torch.equal(one.nan_to_num(0.5), out[b * P:(b + 1) * P].nan_to_num(0.5)), (case, b)
    assert torch.equal(again[:M].nan_to_num(0.5), out[:M].nan_to_num(0.5)), case


# ---- the table covers the models ------------------------------------------------------------------------------------

def _model_calls(dev, rec):
    """One run of each model that uses the convolution core, on synthetic weights; returns the recorded calls."""
    from oracle import faed as of, inception as oi
    from panfusion_b200 import faed, faed_train as ft, horizonnet, inception
    g = torch.Generator().manual_seed(0)
    faed.FAEDEncoder(of.synth_state(1), dev)(of.images((2, 3, 64, 128), "real", 1).to(dev))
    tr = ft.FAEDTrainer(seed=0, device=dev)
    tr.training_step((torch.rand(2, 3, 64, 128, generator=g) * 2 - 1).to(dev))
    inception.InceptionV3(oi.synth_state(1), dev)(oi.images(2, (299, 299), "real", 1).to(dev))
    sd = {}
    for k, shape in horizonnet.state_shapes().items():  # shapes are all the call classes depend on
        sd[k] = torch.rand(shape, generator=g) + 0.5 if k.endswith("running_var") else torch.randn(shape, generator=g) * 0.05
    horizonnet.HorizonNetModule(sd, dev)(torch.rand(1, 3, 512, 1024, generator=g).to(dev))
    torch.cuda.synchronize()
    return list(rec.calls)


def test_conv_call_table_covers_the_models(recorder, cuda_device):
    """Every conv_mma call class of the FAED encoder, one FAED training step, InceptionV3 and HorizonNet (B = 1,
    512 x 1024) has a case in CONV_CASES."""
    calls = _model_calls(cuda_device, recorder)
    seen = {call_class(n, a) for n, a in calls}
    assert {c[0] for c in seen} == set(ENTRIES), "a model made no call of one of the entry points"
    covered = set().union(*CASE_CLASSES.values())
    missing = sorted(seen - covered, key=str)
    assert not missing, f"call classes without a contract case: {missing}"
