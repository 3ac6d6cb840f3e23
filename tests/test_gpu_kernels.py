"""-m gpu: the bandwidth-bound kernels (GroupNorm stats / conv-prep / LayerNorm / conv_in / conv_out / CFG+DDIM /
timestep embedding) against plain PyTorch fp32 on the same 16-bit-rounded inputs, and the EPPA tables against the
oracle's get_masks / get_coords / SphericalPE (models/pano/utils.py:10-106, transformer.py:185-201)."""
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _tokens(x):  # NCHW -> [N*H*W, C]
    n, c, h, w = x.shape
    return x.permute(0, 2, 3, 1).reshape(n * h * w, c).contiguous()


@pytest.mark.parametrize("N,C,H,W,circ", [(2, 320, 16, 32, 2), (3, 64, 8, 8, 0), (2, 1920, 8, 16, 2), (1, 640, 64, 128, 2),
                                          (16, 320, 64, 64, 0)])
def test_groupnorm_stats(cuda_device, N, C, H, W, circ):
    from panfusion_b200 import ops
    from oracle.eppa import pad_pano
    x = (torch.randn(N, C, H, W, generator=torch.Generator().manual_seed(1)) * 1.7 + 0.3).bfloat16()
    xp = pad_pano(x.float(), circ)
    g = xp.reshape(N, 32, -1)
    mean, var = g.mean(-1), g.var(-1, unbiased=False)
    got = ops.groupnorm_stats(_tokens(x).to(cuda_device), N, H, W, 32, 1e-5, circ).cpu()
    torch.testing.assert_close(got[..., 0], mean, rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(got[..., 1], (var + 1e-5).rsqrt(), rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize("circ,up,phases,halo", [(0, 1, 1, 1), (2, 1, 1, 1), (0, 1, 1, 0), (1, 2, 1, 1), (0, 2, 1, 1),
                                                 (2, 1, 4, 1), (0, 1, 4, 1)])
def test_conv_prep(cuda_device, circ, up, phases, halo):
    """GroupNorm + SiLU + circular pad / upsample / zero halo / stride-2 phase split == the torch composition."""
    from panfusion_b200 import ops
    from oracle.eppa import pad_pano
    N, C, H, W = 2, 128, 8, 12
    g = torch.Generator().manual_seed(2)
    x = torch.randn(N, C, H, W, generator=g).half()
    gamma, beta = torch.randn(C, generator=g), torch.randn(C, generator=g)
    xp = pad_pano(x.float(), circ)
    ref = F.silu(F.group_norm(xp, 32, gamma, beta, 1e-5))  # stats over the padded tensor, like the reference
    if up == 2:
        ref = F.interpolate(ref, scale_factor=2.0, mode="nearest")
    if halo:
        ref = F.pad(ref, [1, 1, 1, 1])
    if phases == 4:
        ref = torch.stack([ref[:, :, py::2, px::2] for py in (0, 1) for px in (0, 1)], 0)  # [4,N,C,Ho+1,Wo+1]
        ref = ref.permute(0, 1, 3, 4, 2)
    else:
        ref = ref.permute(0, 2, 3, 1)
    xt = _tokens(x).to(cuda_device)
    stats = ops.groupnorm_stats(xt, N, H, W, 32, 1e-5, circ)
    got = ops.conv_prep(xt, N, H, W, stats=stats, gamma=gamma.to(cuda_device), beta=beta.to(cuda_device), groups=32,
                        act=ops.PF_ACT_SILU, circ=circ, up=up, phases=phases, halo=halo)
    torch.testing.assert_close(got.float().cpu().reshape(ref.shape), ref, rtol=2e-3, atol=2e-3)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("N,C1,C2,H,W,circ_stats,circ,halo,act", [
    (2, 128, 0, 8, 12, 0, 0, 1, "silu"),       # ResnetBlock2D norm1 / norm2, perspective branch
    (2, 320, 0, 16, 32, 2, 2, 1, "silu"),      # panorama norm1: pad_pano(2) statistics and layout
    (16, 320, 0, 64, 64, 0, 0, 1, "silu"),     # the level-0 shape of the benchmark (9 CTAs per image)
    (3, 640, 0, 8, 8, 0, 0, 0, "none"),        # Transformer2DModel.norm: plain apply, no halo
    (2, 320, 0, 8, 16, 0, 1, 1, "silu"),       # conv_norm_out: statistics of the un-padded tensor, pad_pano(1) layout
    (2, 1280, 640, 8, 8, 0, 0, 1, "silu"),     # decoder: cat([hidden, skip]) with a group (60 ch) straddling the seam
    (1, 640, 320, 16, 32, 2, 2, 1, "silu"),    # the same on the panorama branch
    (20, 64, 64, 4, 4, 0, 0, 1, "silu"),       # many tiny images: one CTA per image
])
def test_gn_prep(cuda_device, dtype, N, C1, C2, H, W, circ_stats, circ, halo, act):
    """pf_gn_prep (statistics + apply + layout + skip concatenation) against the torch composition pad_pano -> GroupNorm
    -> SiLU -> pad of the reference (MVGenModel.py:110-115,223-231; diffusers ResnetBlock2D norm1/norm2) and against
    pf_groupnorm_stats -> pf_conv_prep; the raw concatenation output is exact. Launched 3 times in a row with the same
    bits each time: the per-image counters must re-arm themselves."""
    from panfusion_b200 import ops
    from oracle.eppa import pad_pano
    g = torch.Generator().manual_seed(N + C1 + C2 + H)
    C = C1 + C2
    x = (torch.randn(N, C, H, W, generator=g) * 1.3 + 0.4).to(dtype)
    gamma, beta = torch.randn(C, generator=g), torch.randn(C, generator=g)
    xs = pad_pano(x.float(), circ_stats)
    mean = xs.reshape(N, 32, -1).mean(-1)
    var = xs.reshape(N, 32, -1).var(-1, unbiased=False)
    cpg = C // 32
    sc = (var + 1e-5).rsqrt().repeat_interleave(cpg, 1)[:, :, None, None] * gamma[None, :, None, None]
    sh = beta[None, :, None, None] - mean.repeat_interleave(cpg, 1)[:, :, None, None] * sc
    ref = pad_pano(x.float() * sc + sh, circ)
    if act == "silu":
        ref = F.silu(ref)
    if halo:
        ref = F.pad(ref, [1, 1, 1, 1])
    ref = ref.permute(0, 2, 3, 1)
    dev = cuda_device
    xt = _tokens(x).to(dev)
    x1, x2 = (xt[:, :C1].contiguous(), xt[:, C1:].contiguous()) if C2 else (xt, None)
    kw = dict(gamma=gamma.to(dev), beta=beta.to(dev), groups=32, eps=1e-5,
              act=ops.PF_ACT_SILU if act == "silu" else ops.PF_ACT_NONE, circ_stats=circ_stats, circ=circ, halo=halo)
    outs = []
    for _ in range(3):
        r = ops.gn_prep(x1, N, H, W, x2=x2, want_cat=bool(C2), **kw)
        got, cat = r if C2 else (r, None)
        outs.append(got.clone())
    torch.cuda.synchronize()
    assert all(torch.equal(outs[0], o) for o in outs[1:])
    if C2:
        assert torch.equal(cat, xt)
    tol = dict(rtol=2e-3, atol=2e-3) if dtype == torch.float16 else dict(rtol=1.6e-2, atol=1.6e-2)
    torch.testing.assert_close(got.float().cpu().reshape(ref.shape), ref, **tol)
    # the two-kernel path computes the same thing with a different partial-sum order: at most an output ulp apart
    st = ops.groupnorm_stats(xt, N, H, W, 32, 1e-5, circ_stats)
    two = ops.conv_prep(xt, N, H, W, stats=st, gamma=kw["gamma"], beta=kw["beta"], groups=32, act=kw["act"], circ=circ,
                        halo=halo)
    d = (got.float() - two.float()).abs()
    assert (d > 0).float().mean().item() < 1e-3 and d.max().item() <= (2e-3 if dtype == torch.float16 else 3.2e-2) * max(1.0, two.float().abs().max().item())


@pytest.mark.parametrize("T,C,with_pe", [(100, 320, True), (64, 1280, False), (33, 64, True), (256, 640, True)])
def test_layernorm(cuda_device, T, C, with_pe):
    from panfusion_b200 import ops
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2 * T, C, generator=g).half()
    gamma, beta = torch.randn(C, generator=g), torch.randn(C, generator=g)
    pe = torch.randn(T, C, generator=g) if with_pe else None
    ref = F.layer_norm(x.float() + (pe.repeat(2, 1) if with_pe else 0), (C,), gamma, beta, 1e-5)
    got = ops.layernorm(x.to(cuda_device), gamma.to(cuda_device), beta.to(cuda_device), 1e-5,
                        pe.to(cuda_device) if with_pe else None)
    torch.testing.assert_close(got.float().cpu(), ref, rtol=1e-3, atol=2e-3)


@pytest.mark.parametrize("circ", [False, True])
def test_conv_in_and_branch_conv_out(cuda_device, circ):
    from panfusion_b200 import engine, ops
    from panfusion_b200.packing import pack_conv3x3
    from oracle.eppa import pad_pano, unpad_pano
    g = torch.Generator().manual_seed(4)
    N, H, W, C = 2, 16, 32, 320
    lat = torch.randn(N, 4, H, W, generator=g)
    w_in, b_in = torch.randn(C, 4, 3, 3, generator=g) * 0.2, torch.randn(C, generator=g)
    conv = lambda x, w, b: unpad_pano(F.conv2d(pad_pano(x, 1), w, b, padding=1), 1) if circ else F.conv2d(x, w, b, padding=1)
    ref = conv(lat, w_in, b_in)
    got = ops.conv_in(lat.to(cuda_device), w_in.to(cuda_device), b_in.to(cuda_device), torch.float16, circ)
    torch.testing.assert_close(got.float().cpu().reshape(N, H, W, C).permute(0, 3, 1, 2), ref, rtol=1e-3, atol=2e-3)
    # conv_norm_out -> SiLU -> conv_out, as Branch.conv_out runs it: pf_gn_prep, then the 64-wide tap-GEMM
    x = torch.randn(N, C, H, W, generator=g).half()
    gamma, beta = torch.randn(C, generator=g), torch.randn(C, generator=g)
    w_out, b_out = torch.randn(4, C, 3, 3, generator=g) * 0.05, torch.randn(4, generator=g)
    ref = conv(F.silu(F.group_norm(x.float(), 32, gamma, beta, 1e-5)), w_out, b_out)
    # the fields of engine.UNetPack that Branch.conv_out reads: 4 output channels zero-padded to one 64-wide tile
    wpad, bpad = torch.zeros(64, C, 3, 3), torch.zeros(64)
    wpad[:4], bpad[:4] = w_out, b_out
    norm = SimpleNamespace(weight=gamma, bias=beta, eps=1e-5, num_groups=32)
    pack = SimpleNamespace(dt=torch.float16, groups=32, norm_out=engine._Norm(norm, cuda_device), conv_out_c=4,
                           conv_out_packed=pack_conv3x3(wpad).to(cuda_device, torch.float16).contiguous(),
                           conv_out_bpad=bpad.to(cuda_device))
    br = engine.Branch(pack, circular=circ)
    got = br.conv_out(engine.img_from_nchw(x.to(cuda_device), torch.float16))
    # the prepared activations and the packed weights are rounded to fp16
    torch.testing.assert_close(got.cpu(), ref, rtol=2e-3, atol=3e-3)


@pytest.mark.parametrize("W", [32, 30])  # 4-pixel register-blocked path and the generic one
def test_conv_in_silu_layout_image(cuda_device, W):
    """pf_conv_in with act = SiLU on a 3-channel image: first conv of the ControlNet conditioning embedding, output
    channels zero-padded 16 -> 64 (padded channels must come out exactly 0 = silu(0))."""
    from panfusion_b200 import ops
    g = torch.Generator().manual_seed(9)
    N, H = 2, 24
    img = torch.rand(N, 3, H, W, generator=g)
    w, b = torch.randn(16, 3, 3, 3, generator=g) * 0.3, torch.randn(16, generator=g)
    ref = F.silu(F.conv2d(img, w, b, padding=1))
    wp, bp = torch.zeros(64, 3, 3, 3), torch.zeros(64)
    wp[:16], bp[:16] = w, b
    got = ops.conv_in(img.to(cuda_device), wp.to(cuda_device), bp.to(cuda_device), torch.float16, False,
                      act=ops.PF_ACT_SILU).float().cpu().reshape(N, H, W, 64).permute(0, 3, 1, 2)
    torch.testing.assert_close(got[:, :16], ref, rtol=1e-3, atol=1e-3)
    assert got[:, 16:].abs().max().item() == 0.0


def test_timestep_embed_and_copy(cuda_device):
    from panfusion_b200 import ops
    from oracle.unet import Timesteps
    t = torch.tensor([981.0, 1.0, 500.0, 21.0])
    ref = Timesteps(320)(t)
    got = ops.timestep_embed(t.to(cuda_device), 320, torch.float16).float().cpu()
    torch.testing.assert_close(got, ref, rtol=0, atol=2e-3)
    src = torch.randn(50, 64).half().to(cuda_device)
    dst = torch.zeros(50, 192, dtype=torch.float16, device=cuda_device)
    ops.copy2d(src, dst[:, 64:128])
    assert torch.equal(dst[:, 64:128], src) and dst[:, :64].abs().sum() == 0 and dst[:, 128:].abs().sum() == 0


def test_cfg_ddim_step(cuda_device):
    from panfusion_b200 import ops
    from oracle.sampler import DDIM
    g = torch.Generator().manual_seed(5)
    x = torch.randn(1, 1, 4, 16, 32, generator=g)
    eps = torch.randn(2, 1, 4, 16, 32, generator=g)
    sched = DDIM()
    sched.set_timesteps(50)
    t = sched.timesteps[3]
    e = eps[:1] + 9.0 * (eps[1:] - eps[:1])
    ref = torch.roll(sched.step(e, t, x), 8, dims=-1)
    a_t = sched.alphas_cumprod[int(t)].item()
    a_p = sched.alphas_cumprod[int(t) - 20].item()
    out = torch.empty_like(x, device=cuda_device)
    ops.cfg_ddim_step(x.to(cuda_device), eps.to(cuda_device), out, 9.0, a_t, a_p, roll=8)
    torch.testing.assert_close(out.cpu(), ref, rtol=1e-5, atol=1e-5)


def _cams(n, seed=0):
    rng = np.random.default_rng(seed)
    return dict(FoV=torch.tensor(rng.uniform(70, 100, n), dtype=torch.float32),
                theta=torch.tensor(rng.uniform(0, 360, n), dtype=torch.float32),
                phi=torch.tensor(rng.uniform(-60, 60, n), dtype=torch.float32))


@pytest.mark.parametrize("ph,pw,eh,ew,V,m", [(8, 8, 8, 16, 3, 3), (16, 16, 16, 32, 4, 2), (8, 8, 16, 32, 2, 1),
                                            (32, 32, 32, 64, 2, 2)])
def test_eppa_tables_vs_oracle(cuda_device, ph, pw, eh, ew, V, m):
    """Bias tables == get_masks (utils.py:10-84) rearranged like modules.py:46,53; PE == SphericalPE(get_coords)."""
    from oracle import eppa as oe
    from panfusion_b200 import geometry as pg, ops
    cams = _cams(V, seed=ph + V)
    if ph == 32:  # the reference's own rig: horizon cameras
        cams = dict(FoV=torch.tensor([90.0, 90.0]), theta=torch.tensor([0.0, 180.0]), phi=torch.zeros(2))
    pm, em = oe.get_masks(ph, pw, eh, ew, cams)
    P, E = ph * pw, eh * ew
    ref1 = pm.reshape(V // m, m, E, P).permute(0, 2, 1, 3).reshape(V // m, E, m * P)
    ref2 = em.reshape(V // m, m * P, E)
    ce, _ = pg.camera_records("e2p", cams["FoV"], cams["theta"], cams["phi"], V, ph, pw, cuda_device)
    cp, _ = pg.camera_records("p2e", cams["FoV"], cams["theta"], cams["phi"], V, ph, pw, cuda_device)
    b1, b2 = ops.eppa_tables(ce, cp, m, ph, pw, eh, ew)
    torch.testing.assert_close(b1.cpu(), ref1, rtol=1e-5, atol=2e-6)
    torch.testing.assert_close(b2.cpu(), ref2, rtol=1e-5, atol=2e-6)
    for dim in (320, 640):
        pe_mod = oe.SphericalPE(dim // 4)
        pc, ec = oe.get_coords(ph, pw, eh, ew, cams)
        rp, re = pe_mod(pc).reshape(V * P, dim), pe_mod(ec).reshape(E, dim)
        gp, ge = ops.eppa_pe(ce, ph, pw, eh, ew, pe_mod.freq_bands)
        # sin/cos of arguments up to 2^79: both sides are correctly-rounded-ish fp32 libm results of the SAME fp32
        # argument; allow a few ulp
        torch.testing.assert_close(gp.cpu(), rp, rtol=0, atol=5e-6)
        torch.testing.assert_close(ge.cpu(), re, rtol=0, atol=5e-6)


def test_eppa_tables_vs_reference_goldens(cuda_device):
    """The CUDA bias tables against the goldens minted by executing the reference's get_masks (not the oracle):
    the 3-camera rig of tests/golden/eppa_geometry.npz and BASELINE config 4's geometry (ph != eh, icosahedron rings)."""
    from pathlib import Path
    import numpy as np
    from panfusion_b200 import geometry as pg, ops
    gdir = Path(__file__).parent / "golden"
    cases = [("eppa_geometry.npz", (8, 8, 8, 16), dict(FoV=torch.tensor([90.0, 75.0, 100.0]),
                                                       theta=torch.tensor([0.0, 45.0, 200.0]),
                                                       phi=torch.tensor([0.0, 30.0, -60.0]))),
             ("eppa_geometry_c4.npz", (8, 8, 16, 32), dict(FoV=torch.full((4,), 90.0),
                                                           theta=torch.tensor([-144.0, 72.0, -180.0, 36.0]),
                                                           phi=torch.tensor([52.6226, 10.8123, -10.8123, -52.6226])))]
    for fname, (ph, pw, eh, ew), cams in cases:
        gold = np.load(gdir / fname)
        V, P, E = len(cams["FoV"]), ph * pw, eh * ew
        pm, em = torch.from_numpy(gold["pers_masks"]), torch.from_numpy(gold["equi_masks"])
        ref1 = pm.reshape(1, V, E, P).permute(0, 2, 1, 3).reshape(1, E, V * P)   # modules.py:46
        ref2 = em.reshape(1, V * P, E)                                           # modules.py:53
        ce, _ = pg.camera_records("e2p", cams["FoV"], cams["theta"], cams["phi"], V, ph, pw, cuda_device)
        cp, _ = pg.camera_records("p2e", cams["FoV"], cams["theta"], cams["phi"], V, ph, pw, cuda_device)
        b1, b2 = ops.eppa_tables(ce, cp, V, ph, pw, eh, ew)
        torch.testing.assert_close(b1.cpu(), ref1, rtol=1e-5, atol=2e-6)
        torch.testing.assert_close(b2.cpu(), ref2, rtol=1e-5, atol=2e-6)


def test_eppa_tables_config4_level_size_vs_reference_golden(cuda_device):
    """pf_eppa_tables at config 4's real first EPPA level (32x32 views / 64x128 pano, icosahedron rings) against the
    reference-run golden: a strided subset of the query rows element-wise, the key-sum of EVERY row."""
    from pathlib import Path
    import numpy as np
    from oracle.make_golden import C4GEO_LEVEL, _cams_ico
    from panfusion_b200 import geometry as pg, ops
    gold = np.load(Path(__file__).parent / "golden" / "eppa_geometry_c4_level.npz")
    ph, pw, eh, ew = C4GEO_LEVEL
    cams = _cams_ico()
    V, P, E = len(cams["FoV"]), ph * pw, eh * ew
    ce, _ = pg.camera_records("e2p", cams["FoV"], cams["theta"], cams["phi"], V, ph, pw, cuda_device)
    cp, _ = pg.camera_records("p2e", cams["FoV"], cams["theta"], cams["phi"], V, ph, pw, cuda_device)
    b1, b2 = ops.eppa_tables(ce, cp, V, ph, pw, eh, ew)          # [1, E, V*P], [1, V*P, E]
    pm = b1.reshape(eh, ew, V, ph, pw).permute(2, 0, 1, 3, 4)     # -> pers_masks [V, eh, ew, ph, pw] (modules.py:46)
    em = b2.reshape(V, ph, pw, eh, ew)                            # -> equi_masks [V, ph, pw, eh, ew] (modules.py:53)
    torch.testing.assert_close(pm[:, ::7, ::9].cpu(), torch.from_numpy(gold["pers_rows"]), rtol=1e-5, atol=2e-6)
    torch.testing.assert_close(em[:, ::5, ::5].cpu(), torch.from_numpy(gold["equi_rows"]), rtol=1e-5, atol=2e-6)
    torch.testing.assert_close(pm.double().sum((-1, -2)).cpu(), torch.from_numpy(gold["pers_rowsum"]), rtol=0, atol=2e-3)
    torch.testing.assert_close(em.double().sum((-1, -2)).cpu(), torch.from_numpy(gold["equi_rowsum"]), rtol=0, atol=2e-3)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.uint8])
def test_pad_pano_bit_exact(cuda_device, dtype):
    """pad_pano / unpad_pano (utils/pano.py:74-105): 4-D and 5-D, every dtype width, against the oracle restatement
    (itself pinned to the reference in tests/test_oracle_golden.py)."""
    from oracle.eppa import pad_pano as ref_pad
    from panfusion_b200.pano import pad_pano, unpad_pano
    g = torch.Generator().manual_seed(3)
    for shape in ((2, 3, 5, 16), (2, 2, 3, 4, 12)):
        x = (torch.rand(shape, generator=g) * 200).to(dtype)
        for p in (1, 2, 8):
            got = pad_pano(x.to(cuda_device), p)
            ref = ref_pad(x.float(), p).to(dtype)
            assert got.shape == ref.shape and torch.equal(got.cpu(), ref)
            assert torch.equal(unpad_pano(got, p).cpu(), x)
    xd = x.to(cuda_device)
    assert pad_pano(xd, 0) is xd and unpad_pano(xd, 0) is xd
    with pytest.raises(NotImplementedError):
        pad_pano(torch.zeros(3, 4, 5, device=cuda_device), 1)
