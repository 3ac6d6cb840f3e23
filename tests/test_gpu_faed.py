"""GPU: the FAED kernels (pf_faed_prep, pf_conv_circ, pf_faed_pool, pf_faed_stats, pf_frechet_fp64) and
panfusion_b200.faed against fp64 torch and tests/golden/faed.npz (minted by executing the reference's
models/faed/modules.py and FAED.py; the seeded weights and images are regenerated from oracle/faed.py and checked
against the golden's digests on the CPU)."""
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import faed as of
from panfusion_b200 import faed

pytestmark = pytest.mark.gpu
GOLD = np.load(Path(__file__).parent / "golden" / "faed.npz")


@pytest.fixture(scope="module")
def sd():
    return of.synth_state(int(GOLD["seed"]))


@pytest.fixture(scope="module")
def enc(sd, cuda_device):
    return faed.FAEDEncoder(sd, cuda_device)


def _conv_ref(x, w, b, k, s, p, relu, res):
    y = torch.nn.functional.conv2d(of.circular_pad(x.double(), p), w, b, stride=s)
    if relu:
        y = y.relu()
    return y if res is None else y + res.double()


# (Cin, Cout, k, stride, H, W): every layer shape of the encoder, at small sizes and a W that is not a power of two
SHAPES = [(3, 32, 9, 1, 24, 48), (32, 32, 9, 1, 16, 96), (32, 64, 4, 2, 16, 96), (64, 64, 7, 1, 8, 48),
          (64, 128, 4, 2, 8, 48), (128, 128, 5, 1, 8, 40), (128, 128, 4, 2, 8, 40), (128, 128, 3, 1, 4, 12),
          (128, 128, 3, 1, 1, 2), (32, 32, 9, 1, 33, 160)]


@pytest.mark.parametrize("cin,cout,k,s,H,W", SHAPES)
@pytest.mark.parametrize("mode", ["relu", "residual", "fp32"])
def test_conv_circ_vs_fp64(cin, cout, k, s, H, W, mode, cuda_device):
    import ctypes as C
    from panfusion_b200 import _lib
    g = torch.Generator().manual_seed(cin * 1000 + k * 10 + H)
    B, p = 2, (1 if s == 2 else k // 2)
    x = torch.randn(B, cin, H, W, generator=g).half()
    w = torch.randn(cout, cin, k, k, generator=g, dtype=torch.float64) / (cin * k * k) ** 0.5
    b = 0.1 * torch.randn(cout, generator=g, dtype=torch.float64)
    ho, wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    res = torch.randn(B, cout, ho, wo, generator=g).half() if mode == "residual" and s == 1 else None
    relu = mode == "relu"
    cin_p = 16 if cin == 3 else cin
    xd = torch.zeros(B, H, W, cin_p, dtype=torch.float16)
    xd[..., :cin] = x.permute(0, 2, 3, 1)
    xd = xd.to(cuda_device)
    wp = faed.pack_weight(w, cin_p, torch.float16).to(cuda_device)
    bd = b.float().to(cuda_device)
    rd = None if res is None else res.permute(0, 2, 3, 1).contiguous().to(cuda_device)
    f32 = mode == "fp32"
    out = torch.empty(B, ho, wo, cout, device=cuda_device, dtype=torch.float32 if f32 else torch.float16)
    _lib.check(_lib.lib().pf_conv_circ(C.c_void_p(xd.data_ptr()), B, H, W, cin_p, C.c_void_p(wp.data_ptr()),
                                       C.c_void_p(bd.data_ptr()), cout, k, s, p, int(relu), C.c_void_p(_lib.ptr(rd)),
                                       C.c_void_p(out.data_ptr()), _lib.PF_F32 if f32 else _lib.PF_F16,
                                       C.c_void_p(_lib.stream_ptr())))
    ref = _conv_ref(x, faed.pack_weight(w, cin, torch.float16).double().reshape(k, k, cin, cout).permute(3, 2, 0, 1),
                    b.float().double(), k, s, p, relu, res)
    got = out.double().cpu().permute(0, 3, 1, 2)
    err = (got - ref).abs().max().item() / ref.abs().max().item()
    print(f"conv {cin}->{cout} k{k} s{s} {H}x{W} {mode}: max err {err:.2e} of max|ref|")
    # measured on an H100: <= 4.4e-4 with fp16 output (its rounding), <= 4.1e-6 with fp32 output
    assert err <= (1e-5 if f32 else 1e-3), err


def test_prep_matches_reference_normalisation(cuda_device):
    import ctypes as C
    from panfusion_b200 import _lib
    imgs = of.images((2, 4, 32, 64), "real", 7)
    d = imgs.to(cuda_device)
    out = torch.empty(2, 32, 64, 16, device=cuda_device, dtype=torch.float16)
    _lib.check(_lib.lib().pf_faed_prep(C.c_void_p(d.data_ptr()), 1, 2, 4, 32, 64, C.c_void_p(out.data_ptr()),
                                       C.c_void_p(_lib.stream_ptr())))
    ref = (imgs[:, :3].float() / 127.5 - 1).half().permute(0, 2, 3, 1)
    assert torch.equal(out[..., :3].cpu(), ref) and not out[..., 3:].any()


@pytest.mark.parametrize("i", range(len(of.FEATURE_SIZES)))
def test_encoder_features_vs_golden(enc, i, cuda_device):
    h, w = of.FEATURE_SIZES[i]
    got = enc(of.feature_images(i).to(cuda_device)).cpu().double().numpy()
    ref = GOLD[f"features_{h}"].astype(np.float64)
    scale = np.abs(ref).max()
    mx, mean = np.abs(got - ref).max() / scale, np.abs(got - ref).mean() / scale
    print(f"features {h}x{w}: max err {mx:.2e}, mean err {mean:.2e} of max|ref|")
    assert mx <= 2e-3 and mean <= 3e-4, (mx, mean)  # measured <= 5.4e-4 / 1.2e-4 on an H100


def test_repeatability_and_batch_invariance(enc, cuda_device):
    x = of.images((4, 3, 128, 256), "fake", 11).to(cuda_device)
    a, b = enc(x), enc(x)
    assert torch.equal(a, b)
    for j in range(4):
        assert torch.equal(enc(x[j:j + 1]), a[j:j + 1]), j
    m = faed.FrechetAutoEncoderDistance(128, encoder=enc, device=cuda_device)
    states = []
    for _ in range(2):
        m.reset()
        m.update(x, real=True)
        m.update(x[:2], real=True)
        states.append((m.real_features_sum.clone(), m.real_features_cov_sum.clone()))
    assert torch.equal(states[0][0], states[1][0]) and torch.equal(states[0][1], states[1][1])


def test_stats_vs_fp64_torch(cuda_device):
    g = torch.Generator().manual_seed(3)
    m = faed.FrechetAutoEncoderDistance(128, encoder=of.synth_state(2), device=cuda_device)
    ref_s, ref_c = torch.zeros(512, dtype=torch.float64), torch.zeros(512, 512, dtype=torch.float64)
    import ctypes as C
    from panfusion_b200 import _lib
    for n in (5, 17, 1):
        f = torch.randn(n, 512, generator=g)
        fd = f.to(cuda_device)
        _lib.check(_lib.lib().pf_faed_stats(C.c_void_p(fd.data_ptr()), n, 512,
                                            C.c_void_p(m.fake_features_sum.data_ptr()),
                                            C.c_void_p(m.fake_features_cov_sum.data_ptr()),
                                            C.c_void_p(_lib.stream_ptr())))
        ref_s += f.double().sum(0)
        ref_c += f.double().t().mm(f.double())
    es = ((m.fake_features_sum.cpu() - ref_s).abs().max() / ref_s.abs().max()).item()
    ec = ((m.fake_features_cov_sum.cpu() - ref_c).abs().max() / ref_c.abs().max()).item()
    print(f"stats: sum rel err {es:.1e}, cov_sum rel err {ec:.1e}")
    assert es <= 1e-12 and ec <= 1e-12


def _golden_stats(tag, case, dev):
    out = []
    for side in ("real", "fake"):
        f = torch.from_numpy(GOLD[f"{tag}_{side}_features"])
        s, c, n = of.stats(list(f.split(list(case["batches"]))))
        out += [s.to(dev), c.to(dev), n]
    return out


@pytest.mark.parametrize("tag,case", [("rd", of.RANK_DEFICIENT), ("fr", of.FULL_RANK)])
def test_distance_from_golden_statistics(tag, case, cuda_device):
    s1, c1, n1, s2, c2, n2 = _golden_stats(tag, case, cuda_device)
    tr = sum(float(of.covariances(s.cpu(), c.cpu(), n)[1].trace()) for s, c, n in ((s1, c1, n1), (s2, c2, n2)))
    got = faed.frechet_distance(s1, c1, n1, s2, c2, n2)
    assert got.dtype == torch.float64 and got.dim() == 0 and got.is_cuda
    ref, ref_eigh = float(GOLD[f"{tag}_faed"]), float(GOLD[f"{tag}_faed_eigh"])
    e, e_eigh = abs(float(got) - ref) / tr, abs(float(got) - ref_eigh) / tr
    print(f"distance {tag}: {float(got)!r} vs golden {ref!r}: {e:.1e} of tr S1 + tr S2 ({e_eigh:.1e} vs eigh)")
    # full rank: the issue's 1e-8 of the traces. Rank deficient (n < d): every fp64 method carries sqrt-of-rounding
    # terms from the ~500 null eigenvalues; the reference's eigvals and a symmetric eigh already differ by 6e-8.
    gate = 1e-8 if tag == "fr" else 2e-7
    assert e <= gate and e_eigh <= gate, (e, e_eigh)
    assert float(faed.frechet_distance(s1, c1, n1, s2, c2, n2)) == float(got)
    same = float(faed.frechet_distance(s1, c1, n1, s1, c1, n1))
    tr1 = 2 * float(of.covariances(s1.cpu(), c1.cpu(), n1)[1].trace())
    print(f"distance {tag} of identical statistics: {same:.1e} ({abs(same) / tr1:.1e} of the trace)")
    assert abs(same) <= 1e-8 * tr1


@pytest.mark.parametrize("tag,case", [("rd", of.RANK_DEFICIENT), ("fr", of.FULL_RANK), ("frl", of.FULL_RANK_LAT)])
def test_end_to_end_vs_golden(enc, tag, case, cuda_device):
    m = faed.FrechetAutoEncoderDistance(case["hw"][0], encoder=enc, device=cuda_device)
    for side in ("real", "fake"):
        for x in of.set_images(case, side):
            m.update(x.to(cuda_device), real=side == "real")
    got = m.compute()
    ref = float(GOLD[f"{tag}_faed"])
    e = abs(float(got) - ref) / abs(ref)
    print(f"end to end {tag}: {float(got)!r} vs golden {ref!r}: rel err {e:.1e}")
    assert e <= 1e-3, e  # measured 8.5e-5 (rank deficient) and 1.2e-4 (full rank) on an H100
    for side in ("real", "fake"):
        assert int(getattr(m, f"{side}_features_num_samples")) == int(GOLD[f"{tag}_{side}_num_samples"])
    # the Jacobi distance against the reference's eigvals(S1 S2) on the same device statistics
    st = [(getattr(m, f"{side}_features_sum").cpu(), getattr(m, f"{side}_features_cov_sum").cpu(),
           int(getattr(m, f"{side}_features_num_samples"))) for side in ("real", "fake")]
    tr = sum(float(of.covariances(*x)[1].trace()) for x in st)
    ref_same = of.faed(*st[0], *st[1])
    e_same = abs(float(got) - ref_same) / tr
    print(f"end to end {tag}: vs the reference's eigvals on the same statistics: {e_same:.1e} of tr S1 + tr S2")
    assert e_same <= (2e-7 if tag == "rd" else 1e-8), e_same


def test_errors(enc, cuda_device):
    m = faed.FrechetAutoEncoderDistance(64, encoder=enc, device=cuda_device)
    x = of.images((1, 3, 64, 128), "real", 5).to(cuda_device)
    m.update(x, real=True)
    m.update(torch.cat([x, x]), real=False)
    with pytest.raises(RuntimeError, match="More than one sample"):
        m.compute()
    with pytest.raises(ValueError):
        m.update(of.images((1, 3, 32, 64), "real", 5).to(cuda_device), real=True)  # H != pano_height
    with pytest.raises(ValueError):
        enc(of.images((1, 3, 64, 120), "real", 5).to(cuda_device))  # W not a multiple of 32
    with pytest.raises(Exception):
        m.update(x.cpu(), real=True)


def test_metric_in_a_module_dict_moves_with_to(cuda_device):
    """EvalPanoGen's use: built on the CPU inside an nn.ModuleDict, requires_grad_(False), moved with .to(device),
    update / compute, _update_called, reset."""
    d = torch.nn.ModuleDict({"FAED": faed.FrechetAutoEncoderDistance(128, encoder=of.synth_state(int(GOLD["seed"])))})
    d.requires_grad_(False)
    m = d["FAED"]
    x = of.images((3, 3, 128, 256), "real", 21)
    with pytest.raises(ValueError, match="move the metric"):
        m.update(x.to(cuda_device), real=True)  # states still on the CPU
    d.to(cuda_device)
    assert m.real_features_cov_sum.is_cuda and m.encoder.w0.is_cuda
    assert not m._update_called
    m.update(x.to(cuda_device), real=True)
    m.update(of.images((3, 3, 128, 256), "fake", 22).to(cuda_device), real=False)
    assert m._update_called
    v = m.compute()
    assert v.is_cuda and v.dtype == torch.float64 and torch.isfinite(v)
    m.reset()
    assert not m._update_called and int(m.real_features_num_samples) == 0 and not m.real_features_cov_sum.any()
