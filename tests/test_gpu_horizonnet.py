"""GPU: the HorizonNet kernels (pf_hnet_prep, pf_hnet_conv, pf_hnet_height_upsample, pf_lstm_bidir with the
pf_gemm_taps input projections, pf_hnet_head) and panfusion_b200.horizonnet against fp64 torch and
tests/golden/horizonnet.npz (minted by executing the reference's external/HorizonNet/model.py; the seeded weights and
images are regenerated from oracle/horizonnet.py and checked against the golden's digests on the CPU)."""
import ctypes as C
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import horizonnet as oh
from panfusion_b200 import _lib, horizonnet, ops

pytestmark = pytest.mark.gpu
GOLD = np.load(Path(__file__).parent / "golden" / "horizonnet.npz")


@pytest.fixture(scope="module")
def sd():
    return oh.synth_state(int(GOLD["seed"]))


@pytest.fixture(scope="module")
def net(sd, cuda_device):
    return horizonnet.HorizonNetModule(sd, cuda_device)


def _st():
    return C.c_void_p(_lib.stream_ptr())


def test_lstm_clusters_fit(cuda_device):
    n = C.c_int(0)
    _lib.check(_lib.lib().pf_lstm_bidir_clusters(C.byref(n)))
    print(f"pf_lstm_bidir: {n.value} active 16-CTA clusters")
    assert n.value >= 1


def test_prep_bit_exact(cuda_device):
    g = torch.Generator().manual_seed(1)
    x = torch.rand(2, 4, 512, 1024, generator=g).to(cuda_device)
    out = torch.empty(2, 512, 1024, 16, device=cuda_device, dtype=torch.float16)
    _lib.check(_lib.lib().pf_hnet_prep(C.c_void_p(x.data_ptr()), 2, 4, 512, 1024, C.c_void_p(out.data_ptr()), _st()))
    mean = oh.MEAN.to(cuda_device)[None, :, None, None]
    std = oh.STD.to(cuda_device)[None, :, None, None]
    ref = ((x[:, :3] - mean) / std).half().permute(0, 2, 3, 1)
    assert torch.equal(out[..., :3], ref)
    assert not out[..., 3:].any()


# (Cin, Cout, k, stride_h, stride_w): every distinct layer shape of the encoder and the GlobalHeightStage
SHAPES = sorted({(3, 64, 7, 2, 2)} | {(ci, co, k, s[0], s[1]) for _n, (_w, _b, _bk, ci, co, k, s)
                                      in horizonnet.CONVS.items() if ci != 3})


@pytest.mark.parametrize("cin,cout,k,sh,sw", SHAPES)
@pytest.mark.parametrize("mode", ["relu", "residual", "fp32"])
def test_conv_vs_fp64(cin, cout, k, sh, sw, mode, cuda_device):
    g = torch.Generator().manual_seed(cin * 7 + cout + k)
    B = 2
    Hi, Wi = (16, 24) if cin < 1024 else (8, 12)  # W = 24 / 12: not a power of two
    if (cin, k) == (3, 7):
        Hi, Wi = 24, 40
    x = torch.randn(B, cin, Hi, Wi, generator=g).half()
    w = torch.randn(cout, cin, k, k, generator=g, dtype=torch.float64) / (cin * k * k) ** 0.5
    b = 0.1 * torch.randn(cout, generator=g, dtype=torch.float64)
    ref = oh.conv(x.double(), w, b, k, (sh, sw))
    res = None
    if mode == "residual":
        res = torch.randn(ref.shape, generator=g).half()
        ref = ref + res.double()
    if mode != "fp32":
        ref = ref.relu()
    cin_p = 16 if cin == 3 else cin
    xin = torch.zeros(B, Hi, Wi, cin_p, dtype=torch.float16)
    xin[..., :cin] = x.permute(0, 2, 3, 1)
    xin = xin.to(cuda_device)
    wp = horizonnet.pack_weight(w, cin_p).to(cuda_device)
    bias = b.float().to(cuda_device)
    f32 = mode == "fp32"
    out = torch.empty(B, ref.shape[2], ref.shape[3], cout, device=cuda_device,
                      dtype=torch.float32 if f32 else torch.float16)
    resd = res.permute(0, 2, 3, 1).contiguous().to(cuda_device) if res is not None else None
    _lib.check(_lib.lib().pf_hnet_conv(
        C.c_void_p(xin.data_ptr()), B, Hi, Wi, cin_p, C.c_void_p(wp.data_ptr()), C.c_void_p(bias.data_ptr()), cout, k,
        sh, sw, int(not f32), C.c_void_p(resd.data_ptr() if resd is not None else 0), C.c_void_p(out.data_ptr()),
        _lib.PF_F32 if f32 else _lib.PF_F16, _st()))
    # the kernel multiplies the fp16-rounded weight: compare against fp64 with the same weight
    ref16 = oh.conv(x.double(), horizonnet.pack_weight(w, cin).double().reshape(k, k, cin, cout).permute(3, 2, 0, 1),
                    b.float().double(), k, (sh, sw))
    if res is not None:
        ref16 = ref16 + res.double()
    if mode != "fp32":
        ref16 = ref16.relu()
    got = out.double().cpu().permute(0, 3, 1, 2)
    err = ((got - ref16).abs().max() / ref16.abs().max()).item()
    print(f"conv {cin}->{cout} k{k} s({sh},{sw}) {mode}: {err:.2e}")
    assert err <= (4e-5 if f32 else 1e-3), err  # about 2x the 1.95e-5 / 4.5e-4 measured on an H100


@pytest.mark.parametrize("scale", range(4))
def test_height_upsample_bit_exact(scale, cuda_device):
    C_, h, w = [(32, 8, 256), (64, 4, 128), (128, 2, 64), (256, 1, 32)][scale]
    B = 3
    g = torch.Generator().manual_seed(scale)
    x = torch.randn(B, h, w, C_, generator=g).relu().half().to(cuda_device)
    out = torch.zeros(256 * B, 1024, device=cuda_device, dtype=torch.float16)
    off = 256 * scale
    _lib.check(_lib.lib().pf_hnet_height_upsample(C.c_void_p(x.data_ptr()), B, h, w, C_, 256,
                                                  C.c_void_p(out.data_ptr()), off, _st()))
    xc = x.float().permute(0, 3, 1, 2)
    f = 256 // w
    y = torch.cat([xc[..., -1:], xc, xc[..., :1]], 3)
    y = F.interpolate(y, size=(h, 256 + 2 * f), mode="bilinear", align_corners=False)[..., f:-f]
    ref = y.reshape(B, C_ * h, 256).permute(2, 0, 1).reshape(256 * B, C_ * h).half()
    assert torch.equal(out[:, off:off + C_ * h], ref)
    assert not out[:, :off].any() and not out[:, off + C_ * h:].any()


def _lstm_ref(x, wih, whh, bih, bhh):
    ref = torch.nn.LSTM(1024, 512, bidirectional=True).double()
    sdl = {}
    for r, sfx in enumerate(("l0", "l0_reverse")):
        sdl[f"weight_ih_{sfx}"], sdl[f"weight_hh_{sfx}"] = wih[r].double(), whh[r].double()
        sdl[f"bias_ih_{sfx}"], sdl[f"bias_hh_{sfx}"] = bih[r].double(), bhh[r].double()
    ref.load_state_dict(sdl)
    with torch.no_grad():
        return ref(x.double())[0]


@pytest.mark.parametrize("T,B", [(1, 1), (5, 3), (256, 1), (256, 3), (256, 8), (5, 16)])
def test_lstm_vs_fp64(T, B, cuda_device):
    g = torch.Generator().manual_seed(T * 100 + B)
    kr = 1 / 512 ** 0.5
    x = torch.randn(T, B, 1024, generator=g).relu().half()
    errs = []
    for layer in range(2):
        wih = ((torch.rand(2, 2048, 1024, generator=g) * 2 - 1) * kr).half()
        whh = ((torch.rand(2, 2048, 512, generator=g) * 2 - 1) * kr).half()
        bih, bhh = (torch.rand(2, 2048, generator=g) * 2 - 1) * kr, (torch.rand(2, 2048, generator=g) * 2 - 1) * kr
        xproj = torch.empty(T * B, 4096, device=cuda_device)
        ops.gemm_taps(x.reshape(T * B, 1024).to(cuda_device), wih.reshape(4096, 1024).to(cuda_device), xproj,
                      M=T * B, Kc=1024, bias=(bih.double() + bhh.double()).float().reshape(4096).to(cuda_device),
                      block_n=128, k_splits=1)
        whp = torch.stack([horizonnet.pack_whh(whh[r]) for r in range(2)]).contiguous().to(cuda_device)
        out = torch.empty(T * B, 1024, device=cuda_device, dtype=torch.float16)
        _lib.check(_lib.lib().pf_lstm_bidir(C.c_void_p(xproj.data_ptr()), C.c_void_p(whp.data_ptr()), T, B,
                                            C.c_void_p(out.data_ptr()), _st()))
        got = out.cpu().reshape(T, B, 1024)
        ref = _lstm_ref(x, wih, whh, bih, bhh)
        errs.append((got.double() - ref).abs().max().item())
        x = got  # layer 2 reads layer 1's fp16 output, as the network does
    print(f"lstm T={T} B={B}: max |h - ref| layer 1 {errs[0]:.2e}, layer 2 {errs[1]:.2e}")
    assert max(errs) <= 5e-4, errs  # about 2x the 2.45e-4 measured on an H100 (fp16 output rounding)


def test_lstm_batch_invariant(cuda_device):
    """Each sample's h is bit-identical alone and inside a batch of 8."""
    g = torch.Generator().manual_seed(5)
    T, B = 64, 8
    xproj = torch.randn(T, B, 4096, generator=g).to(cuda_device)
    whh = ((torch.rand(2, 16, 128, 512, generator=g) * 2 - 1) / 512 ** 0.5).half().to(cuda_device)

    def run(xp, b):
        xp = xp.contiguous()
        out = torch.empty(T * b, 1024, device=cuda_device, dtype=torch.float16)
        _lib.check(_lib.lib().pf_lstm_bidir(C.c_void_p(xp.data_ptr()), C.c_void_p(whh.data_ptr()), T, b,
                                            C.c_void_p(out.data_ptr()), _st()))
        return out.reshape(T, b, 1024)

    full = run(xproj, B)
    for b in (0, 5):
        assert torch.equal(run(xproj[:, b:b + 1], 1)[:, 0], full[:, b])


def _golden_errors(bon, cor):
    out = {}
    for name, got in (("bon", bon), ("cor", cor)):
        ref = GOLD[name]
        d = np.abs(got.double().cpu().numpy() - ref)
        out[name] = (d.max() / np.abs(ref).max(), d.mean() / np.abs(ref).max(), d.max())
    return out


def test_end_to_end_vs_golden(net, cuda_device):
    x = oh.images(int(GOLD["seed"]))
    bon, cor = net(x.to(cuda_device))
    assert bon.shape == (3, 2, 1024) and cor.shape == (3, 1, 1024)
    assert bon.dtype == torch.float32 and cor.dtype == torch.float32
    errs = _golden_errors(bon, cor)
    for name, (mx, mean, absmax) in errs.items():
        print(f"{name}: max {mx:.2e}, mean {mean:.2e} of max|ref|")
        assert mx <= 5e-3 and mean <= 1e-3, (name, mx, mean)  # measured on an H100: 2.2e-3 / 4.9e-4 (bon)
    # bon is the boundary's latitude in radians: the error in image rows is x 512 / pi
    print(f"bon max error {errs['bon'][2] * 512 / np.pi:.3f} image rows")


def test_repeat_and_batch_bit_identical(net, cuda_device):
    x = oh.images(int(GOLD["seed"])).to(cuda_device)
    batch = torch.cat([x, x[1:2]])
    bon4, cor4 = net(batch)
    bon4b, cor4b = net(batch)
    assert torch.equal(bon4, bon4b) and torch.equal(cor4, cor4b)
    for i in range(3):
        bon, cor = net(x[i:i + 1])
        assert torch.equal(bon[0], bon4[i]) and torch.equal(cor[0], cor4[i]), i
    assert torch.equal(bon4[3], bon4[1])


def test_chunked_batch(net, cuda_device, monkeypatch):
    """Batches above MAX_BATCH run in chunks with the same bits."""
    x = oh.images(int(GOLD["seed"])).to(cuda_device)
    bon, cor = net(x)
    monkeypatch.setattr(horizonnet, "MAX_BATCH", 2)
    bon2, cor2 = net(x)
    assert torch.equal(bon, bon2) and torch.equal(cor, cor2)


def test_refusals_and_module_moves(sd, net, cuda_device):
    with pytest.raises(NotImplementedError):
        net(torch.zeros(1, 3, 256, 512, device=cuda_device))
    with pytest.raises(_lib.PFError):
        net(torch.zeros(1, 3, 512, 1024))
    with pytest.raises(ValueError):
        net(torch.zeros(1, 3, 512, 1024, device=cuda_device, dtype=torch.float16))
    md = torch.nn.ModuleDict({"hnet": horizonnet.HorizonNetModule(sd)}).to(cuda_device)
    assert md["hnet"].head_w.device.type == "cuda" and md["hnet"].whh0.device.type == "cuda"
    x = oh.images(int(GOLD["seed"]))[:1].to(cuda_device)
    b1, c1 = md["hnet"](x)
    b2, c2 = net(x)
    assert torch.equal(b1, b2) and torch.equal(c1, c2)
