"""GPU: the FID InceptionV3 kernels (pf_inception_prep, pf_conv2d_nhwc, pf_pool2d_nhwc, pf_inception_head,
pf_inception_score) and panfusion_b200.inception against fp64 torch, the oracle's prep and tests/golden/inception.npz
(minted by oracle/inception.py; the seeded weights and images are regenerated and checked against the golden's
digests on the CPU)."""
import ctypes as C
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import faed as of
from oracle import inception as oi
from panfusion_b200 import _lib, inception

pytestmark = pytest.mark.gpu
GOLD = np.load(Path(__file__).parent / "golden" / "inception.npz")


@pytest.fixture(scope="module")
def sd():
    return oi.synth_state(int(GOLD["seed"]))


@pytest.fixture(scope="module")
def net(sd, cuda_device):
    return inception.InceptionV3(sd, cuda_device)


# (Cin, Cout, kh, kw, stride, ph, pw, H): every distinct convolution shape of the network at its own resolution
SHAPES = ([(16, 32, 3, 3, 2, 0, 0, 299), (32, 32, 3, 3, 1, 0, 0, 149), (32, 64, 3, 3, 1, 1, 1, 147),
           (64, 80, 1, 1, 1, 0, 0, 73), (80, 192, 3, 3, 1, 0, 0, 73)]
          + [(ci, co, 1, 1, 1, 0, 0, 35) for ci in (192, 256, 288) for co in (64, 48, 32)]
          + [(48, 64, 5, 5, 1, 2, 2, 35), (64, 96, 3, 3, 1, 1, 1, 35), (96, 96, 3, 3, 1, 1, 1, 35),
             (288, 384, 3, 3, 2, 0, 0, 35), (96, 96, 3, 3, 2, 0, 0, 35)]
          + [s for c7 in (128, 160, 192) for s in (
              (768, c7, 1, 1, 1, 0, 0, 17), (c7, c7, 1, 7, 1, 0, 3, 17), (c7, c7, 7, 1, 1, 3, 0, 17),
              (c7, 192, 1, 7, 1, 0, 3, 17), (c7, 192, 7, 1, 1, 3, 0, 17))]
          + [(768, 192, 1, 1, 1, 0, 0, 17), (192, 320, 3, 3, 2, 0, 0, 17), (192, 192, 3, 3, 2, 0, 0, 17)]
          + [(ci, co, 1, 1, 1, 0, 0, 8) for ci in (1280, 2048) for co in (320, 384, 448, 192)]
          + [(384, 384, 1, 3, 1, 0, 1, 8), (384, 384, 3, 1, 1, 1, 0, 8), (448, 384, 3, 3, 1, 1, 1, 8)])
SHAPES = list(dict.fromkeys(SHAPES))


def _conv(x, w, b, cout, kh, kw, s, ph, pw, out, off):
    B, H, W, cin = x.shape
    _lib.check(_lib.lib().pf_conv2d_nhwc(C.c_void_p(x.data_ptr()), B, H, W, cin, C.c_void_p(w.data_ptr()),
                                         C.c_void_p(b.data_ptr()), cout, kh, kw, s, ph, pw, 1,
                                         C.c_void_p(out.data_ptr()),
                                         _lib.PF_F32 if out.dtype == torch.float32 else _lib.PF_F16, out.shape[-1],
                                         off, C.c_void_p(_lib.stream_ptr())))


@pytest.mark.parametrize("cin,cout,kh,kw,s,ph,pw,H", SHAPES)
@pytest.mark.parametrize("mode", ["fp16_slice", "fp32"])
def test_conv2d_vs_fp64(cin, cout, kh, kw, s, ph, pw, H, mode, cuda_device):
    g = torch.Generator().manual_seed(cin * 1000 + cout + kh * 10 + kw + H)
    B = 2
    real_cin = 3 if cin == 16 else cin
    x = torch.randn(B, real_cin, H, H, generator=g).half()
    w = torch.randn(cout, real_cin, kh, kw, generator=g, dtype=torch.float64) / (real_cin * kh * kw) ** 0.5
    b = 0.1 * torch.randn(cout, generator=g, dtype=torch.float64)
    xd = torch.zeros(B, H, H, cin, dtype=torch.float16)
    xd[..., :real_cin] = x.permute(0, 2, 3, 1)
    wp = inception.pack_weight(w, cin)
    bias = torch.zeros(inception.packed_cout(cout))
    bias[:cout] = b.float()
    ho, wo = (H + 2 * ph - kh) // s + 1, (H + 2 * pw - kw) // s + 1
    f32 = mode == "fp32"
    off, ld = (0, cout) if f32 else (16, cout + 48)  # fp16: a slice of a wider concat buffer
    out = torch.full((B, ho, wo, ld), 7.0, device=cuda_device, dtype=torch.float32 if f32 else torch.float16)
    _conv(xd.to(cuda_device), wp.to(cuda_device), bias.to(cuda_device), cout, kh, kw, s, ph, pw, out, off)
    wq = wp[:, :real_cin, :cout].double().reshape(kh, kw, real_cin, cout).permute(3, 2, 0, 1)
    ref = torch.nn.functional.conv2d(x.double(), wq, b.float().double(), stride=s, padding=(ph, pw)).relu()
    got = out[..., off:off + cout].double().cpu().permute(0, 3, 1, 2)
    err = (got - ref).abs().max().item() / ref.abs().max().item()
    print(f"conv {cin}->{cout} {kh}x{kw} s{s} p({ph},{pw}) @{H} {mode}: max err {err:.2e} of max|ref|")
    assert err <= (1e-5 if f32 else 1e-3), err
    if not f32:
        assert bool((out[..., :off] == 7).all()) and bool((out[..., off + cout:] == 7).all())


POOLS = [(inception.MAX, 2, 0, 64, 147, 0), (inception.MAX, 2, 0, 288, 35, 480), (inception.AVG, 1, 1, 192, 35, 0),
         (inception.AVG, 1, 1, 1280, 8, 8), (inception.MAX, 1, 1, 2048, 8, 0)]


@pytest.mark.parametrize("mode,stride,pad,ch,H,off", POOLS)
def test_pools_vs_torch(mode, stride, pad, ch, H, off, cuda_device):
    g = torch.Generator().manual_seed(ch + H)
    x = torch.randn(2, ch, H, H, generator=g).abs().half()  # post-ReLU activations
    ho = (H + 2 * pad - 3) // stride + 1
    ld = off + ch + 8
    out = torch.full((2, ho, ho, ld), 7.0, device=cuda_device, dtype=torch.float16)
    xd = x.permute(0, 2, 3, 1).contiguous().to(cuda_device)
    _lib.check(_lib.lib().pf_pool2d_nhwc(C_ptr(xd), 2, H, H, ch, mode, stride, pad, C_ptr(out), ld, off,
                                         C_ptr_stream()))
    got = out[..., off:off + ch].cpu().permute(0, 3, 1, 2)
    if mode == inception.MAX:
        ref = torch.nn.functional.max_pool2d(x.float(), 3, stride, pad).half()
        assert torch.equal(got, ref)
    else:
        ref = torch.nn.functional.avg_pool2d(x.float(), 3, stride, pad, count_include_pad=False).half()
        ulps = (got.view(torch.int16).int() - ref.view(torch.int16).int()).abs().max().item()
        print(f"avg pool C={ch} @{H}: max {ulps} fp16 ulp")
        assert ulps <= 1
    assert bool((out[..., :off] == 7).all()) and bool((out[..., off + ch:] == 7).all())


def C_ptr(t):
    return C.c_void_p(t.data_ptr())


def C_ptr_stream():
    return C.c_void_p(_lib.stream_ptr())


def _prep(src, is_u8, cuda_device):
    B, _, H, W = src.shape
    out = torch.empty(B, 299, 299, 16, device=cuda_device, dtype=torch.float16)
    _lib.check(_lib.lib().pf_inception_prep(C_ptr(src), is_u8, B, H, W, C_ptr(out), C_ptr_stream()))
    return out.cpu()


@pytest.mark.parametrize("hw", [(512, 1024), (512, 512), (299, 299), (64, 48)])
def test_prep_bit_equal_to_oracle(hw, cuda_device):
    imgs = oi.images(2, hw, "real", 3)
    got = _prep(imgs.to(cuda_device), 1, cuda_device)
    ref = oi.prep(imgs).half().permute(0, 2, 3, 1)
    assert torch.equal(got[..., :3], ref) and not got[..., 3:].any()
    # normalize=True: fp32 in [0, 1], (x * 255).byte() inside the kernel
    x = torch.rand(2, 3, *hw, generator=torch.Generator().manual_seed(5))
    x[0, 0, 0, :4] = torch.tensor([0.0, 1.0, 1 / 255, 254.5 / 255])
    got = _prep(x.to(cuda_device), 0, cuda_device)
    ref = oi.prep((x * 255).byte()).half().permute(0, 2, 3, 1)
    assert torch.equal(got[..., :3], ref)


@pytest.mark.parametrize("i", range(len(oi.FEATURE_SIZES)))
def test_features_vs_golden(net, i, cuda_device):
    h, w = oi.FEATURE_SIZES[i]
    pool3, logits = net(oi.feature_images(i).to(cuda_device))
    for name, got in (("pool3", pool3), ("logits", logits)):
        ref = GOLD[f"{name}_{h}x{w}"].astype(np.float64)
        d = np.abs(got.cpu().double().numpy() - ref)
        scale = np.abs(ref).max()
        mx, mean = d.max() / scale, d.mean() / scale
        print(f"{name} {h}x{w}: max err {mx:.2e}, mean err {mean:.2e} of max|ref|")
        # measured on an H100: pool3 <= 5.8e-4 / 5.1e-5, logits <= 2.5e-3 / 5.4e-4. The logits' mean gate is 1e-3, not
        # 5e-4: they are differences of much larger terms (fc rows orthogonal to the dominant pool3 direction), which
        # scales pool3's error up against max|logits| (DESIGN.md 5d).
        assert mx <= 3e-3 and mean <= (5e-4 if name == "pool3" else 1e-3), (name, mx, mean)


def test_repeatability_and_batch_invariance(net, cuda_device):
    x = oi.images(8, (512, 1024), "fake", 11).to(cuda_device)
    a, b = net(x), net(x)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    for j in range(8):
        p, l = net(x[j:j + 1])
        assert torch.equal(p, a[0][j:j + 1]) and torch.equal(l, a[1][j:j + 1]), j


def _fid_run(net, case, dev):
    m = inception.FrechetInceptionDistance(inception=net, device=dev)
    for side in ("real", "fake"):
        for x in oi.set_images(case, side):
            for i in range(0, x.shape[0], 100):
                m.update(x[i:i + 100].to(dev), real=side == "real")
    return m


@pytest.mark.parametrize("tag", ["rd", "fr"])
def test_fid_end_to_end_vs_golden(net, tag, cuda_device):
    case = {"rd": oi.RANK_DEFICIENT, "fr": oi.FULL_RANK}[tag]
    m = _fid_run(net, case, cuda_device)
    got = m.compute()
    assert got.dtype == torch.float32 and got.dim() == 0 and got.is_cuda
    ref = float(GOLD[f"{tag}_fid"])
    e = abs(float(got) - ref) / abs(ref)
    print(f"FID {tag}: {float(got)!r} vs golden {ref!r}: rel err {e:.1e}")
    assert e <= 2e-3, e
    for side in ("real", "fake"):
        assert int(getattr(m, f"{side}_features_num_samples")) == int(GOLD[f"{tag}_{side}_num_samples"])
    st = [(getattr(m, f"{side}_features_sum").cpu(), getattr(m, f"{side}_features_cov_sum").cpu(),
           int(getattr(m, f"{side}_features_num_samples"))) for side in ("real", "fake")]
    tr = sum(float(of.covariances(*x)[1].trace()) for x in st)
    dev = float(inception.frechet_distance(m.real_features_sum, m.real_features_cov_sum, st[0][2],
                                           m.fake_features_sum, m.fake_features_cov_sum, st[1][2]))
    e_same = abs(dev - oi.fid(*st[0], *st[1])) / tr
    print(f"FID {tag}: device distance vs eigvals on the same device statistics: {e_same:.1e} of tr S1 + tr S2")
    # measured 7.4e-7 (n = 20 < d = 2048) / 2.0e-7 (n = 2100) on an H100: ~2000 (near-)null eigenvalues each add a sqrt
    # of their rounding at d = 2048, four times FAED's d = 512 (DESIGN.md 5d)
    assert e_same <= (2e-6 if tag == "rd" else 5e-7), e_same


@pytest.mark.parametrize("n,splits,seed", oi.IS_CASES)
def test_inception_score_vs_golden(net, n, splits, seed, cuda_device):
    m = inception.InceptionScore(splits=splits, inception=net, device=cuda_device)
    x = oi.is_logits_images()[:n].to(cuda_device)
    m.update(x[:n // 2])
    m.update(x[n // 2:])
    torch.manual_seed(seed)
    mean, std = m.compute()
    assert mean.dtype == torch.float32 and mean.is_cuda
    rm, rs = float(GOLD[f"is_{n}_mean"]), float(GOLD[f"is_{n}_std"])
    em, es = abs(float(mean) - rm) / rm, abs(float(std) - rs) / rm
    print(f"IS n={n}: ({float(mean):.6f}, {float(std):.6f}) vs golden ({rm:.6f}, {rs:.6f}): mean rel err {em:.1e}, "
          f"std err {es:.1e} of the mean")
    # the std is the spread of ten chunk scores that each carry the mean's error, so it is gated against the mean:
    # measured 4.2e-4 / 2.6e-4 (mean) and 3.9e-4 / 2.7e-4 (std, of the mean) on an H100, 1.2e-2 / 1.0e-2 of the std
    assert em <= 1e-3 and es <= 1e-3, (em, es)


def test_inception_score_reduction_vs_torch(cuda_device):
    """pf_inception_score alone, on given logits, against the torchmetrics restatement in fp64 (one chunk: std nan)."""
    g = torch.Generator().manual_seed(9)
    l = _lib.lib()
    l.pf_inception_score_ws_doubles.restype = C.c_longlong
    for n, splits in ((25, 10), (40, 10), (7, 1)):
        logits = 3 * torch.randn(n, 1008, generator=g)
        torch.manual_seed(n)
        perm = torch.randperm(n)
        ws = torch.empty(l.pf_inception_score_ws_doubles(n, 1008, splits), device=cuda_device, dtype=torch.float64)
        out = torch.empty(2, device=cuda_device)
        ld, pd = logits.to(cuda_device), perm.to(cuda_device)
        _lib.check(l.pf_inception_score(C_ptr(ld), C_ptr(pd), n, 1008, splits, C_ptr(ws), C_ptr(out),
                                        C_ptr_stream()))
        mean, std = out.cpu().double().tolist()
        rm, rs = oi.inception_score(logits.double(), splits, n)
        print(f"IS reduction n={n} splits={splits}: ({mean}, {std}) vs ({rm}, {rs})")
        assert abs(mean - rm) <= 1e-6 * rm
        if splits == 1:
            assert np.isnan(std) and np.isnan(rs)
        else:
            assert abs(std - rs) <= 1e-5 * rs + 1e-7


def test_e2p_crops_normalize_matches_byte_path(net, cuda_device):
    """EvalPanoGen's crop FIDs: geometry.e2p crops of a [0, 1] panorama through update(normalize=True) give the same
    features as (crop * 255).byte() through normalize=False."""
    from panfusion_b200 import geometry
    pano = oi.images(1, (512, 1024), "real", 31).float().div(255).to(cuda_device)
    crops = torch.cat([geometry.e2p(pano, 90, u, 0, (299, 299)) for u in (0, 90, 180, 270)]).contiguous()
    a = net(crops, normalize=True)
    b = net((crops * 255).byte(), normalize=False)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    f = inception.FrechetInceptionDistance(normalize=True, inception=net, device=cuda_device)
    f.update(crops, real=True)
    assert int(f.real_features_num_samples) == 4


def test_modules_in_a_module_dict_move_with_to(sd, cuda_device):
    """EvalPanoGen's use: one shared network, metrics built on the CPU inside an nn.ModuleDict, requires_grad_(False),
    moved with .to(device); the device-mismatch and one-sample errors."""
    shared = inception.InceptionV3(sd)
    d = torch.nn.ModuleDict({"FID": inception.FrechetInceptionDistance(inception=shared),
                             "IS": inception.InceptionScore(inception=shared)})
    d.requires_grad_(False)
    x = oi.images(3, (299, 299), "real", 21)
    with pytest.raises(ValueError, match="move the metric"):
        d["FID"].update(x.to(cuda_device), real=True)
    d.to(cuda_device)
    assert d["FID"].real_features_cov_sum.is_cuda and shared.fc_w.is_cuda
    m = d["FID"]
    assert not m._update_called
    m.update(x.to(cuda_device), real=True)
    m.update(x[:1].to(cuda_device), real=False)
    assert m._update_called
    with pytest.raises(RuntimeError, match="More than one sample"):
        m.compute()
    m.update(oi.images(2, (299, 299), "fake", 22).to(cuda_device), real=False)
    v = m.compute()
    assert v.is_cuda and v.dtype == torch.float32 and torch.isfinite(v) and float(v) > 0
    m.reset()
    assert not m._update_called and int(m.real_features_num_samples) == 0 and not m.real_features_cov_sum.any()
    d["IS"].update(x.to(cuda_device))
    assert d["IS"]._update_called and len(d["IS"].features) == 1
    with pytest.raises(Exception):
        m.update(x, real=True)  # CPU images
