"""-m gpu: GroupNorm (pf_gn_prep, pf_groupnorm_stats, pf_conv_prep), LayerNorm (pf_layernorm), the text tower's token
embedding (pf_embed_tokens) and the sampler's element-wise kernels (pf_cfg_ddim_step_dev, pf_timestep_embed) against
the fp64 restatements of tests/_contract.py, at the shapes and argument combinations the models pass.

Every output starts as NaN, so a store outside the contract (or a position never written) fails. The statistics
pf_gn_prep computes are checked directly, where the workspace keeps them, not only through the normalised output:
statistics errors scale like 1 / count and hide in the output at real image sizes. The inputs give every (image,
group) its own offset and scale and shift the seam columns, so a pixel, column, channel or image read from the wrong
place moves a statistic far past its bound. Each GroupNorm launch is also checked for its batch invariance (image n of
a batch is byte-identical to the same image launched alone), for counters that come back zero, and for a repeat launch
that is byte-identical. `_Recorder` logs the class of every call the models make;
`test_norm_call_table_covers_the_models` requires a case for each."""
import ctypes as C
import functools

import pytest
import torch

import _contract as ct

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]
ENTRIES = ("pf_gn_prep", "pf_groupnorm_stats", "pf_conv_prep", "pf_layernorm", "pf_embed_tokens",
           "pf_cfg_ddim_step_dev", "pf_timestep_embed")
GROUPS, EPS = 32, 1e-5
GN_MAX_SLABS = 64  # norm.cu: the workspace holds N * 64 * groups (sum, sum of squares) partials, then mean_rstd
SILU, NONE = ct.ACT_SILU, ct.ACT_NONE


def _nan(shape, dtype, dev):
    return torch.full(shape, float("nan"), dtype=dtype, device=dev)


def _vp(t):
    return C.c_void_p(0 if t is None else t.data_ptr())


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32)


def _same(a, b):
    return torch.equal(_bits(a), _bits(b))


@functools.lru_cache(maxsize=None)
def _ln_wave():
    """Tokens one pf_layernorm launch covers before a warp loops: 8 CTAs of 8 warps per SM."""
    return 64 * torch.cuda.get_device_properties(0).multi_processor_count


# ---- call classes ---------------------------------------------------------------------------------------------------

def _p(a):
    return a.value if isinstance(a, C.c_void_p) else a


def call_class(name, args):
    a = [_p(v) for v in args]
    if name == "pf_gn_prep":   # (x1, ld1, C1, x2, ld2, C2, cat, out, dt, N, H, W, groups, eps, g, b, act, cs, circ, up, ph, halo)
        C1, C2 = a[2], (a[5] if a[3] else 0)
        wide = a[1] > C1 or (bool(a[3]) and a[4] > C2)
        return (name, C1, C2, a[17], a[18], a[19], a[20], a[21], a[16], True, wide)
    if name == "pf_conv_prep":  # (x, out, dt, N, H, W, C, ld, mean_rstd, g, b, groups, act, circ, up, phases, halo)
        return (name, a[6], 0, None, a[13], a[14], a[15], a[16], a[12], bool(a[8]), a[7] > a[6])
    if name == "pf_groupnorm_stats":  # (x, dt, N, H, W, C, ld, groups, circ, ...)
        return (name, a[5], 0, a[8], None, None, None, None, None, True, a[6] > a[5])
    if name == "pf_layernorm":  # (x, ldx, out, ldo, dt, T, C, pe, pe_rows, ...)
        return (name, bool(a[7]), a[1] > a[6], a[5] > _ln_wave())
    if name == "pf_cfg_ddim_step_dev":  # (x, eps, out, count, W, roll, ...)
        return (name, a[5] != 0)
    return (name,)


class _Recorder:
    """Stands in for the library handle: logs the class of every normalisation / sampler call, then forwards it."""

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
    from panfusion_b200 import _lib
    rec = _Recorder(_lib.lib())
    monkeypatch.setattr(_lib, "lib", lambda: rec)
    return rec


# ---- GroupNorm ------------------------------------------------------------------------------------------------------

def gn(entry, N, H, W, C1, C2=0, cs=0, circ=0, up=1, phases=1, halo=1, act=SILU, ld_pad=0):
    """One GroupNorm call: entry "gn_prep" (pf_gn_prep), "stats+prep" (pf_groupnorm_stats then pf_conv_prep, as the
    VAE runs them) or "prep" (pf_conv_prep without statistics); cs = circ_stats; ld_pad widens the source rows."""
    return dict(entry=entry, N=N, H=H, W=W, C1=C1, C2=C2, cs=cs, circ=circ, up=up, phases=phases, halo=halo,
                act=act if entry != "prep" else NONE, ld_pad=ld_pad)


def _unet_level(N, H, W, C, pano):
    """ResnetBlock2D norm1 / norm2 and Transformer2DModel.norm at one level (engine.Branch): the panorama normalises
    pad_pano(2) (statistics and layout), its norm2 sees the padded width W + 4."""
    if pano:
        return [gn("gn_prep", N, H, W, C, cs=2, circ=2), gn("gn_prep", N, H, W + 4, C),
                gn("gn_prep", N, H, W, C, halo=0, act=NONE)]
    return [gn("gn_prep", N, H, W, C), gn("gn_prep", N, H, W, C, halo=0, act=NONE)]


def _conv_out(N, H, W, C, pano):
    """conv_norm_out + SiLU ahead of conv_out: statistics of the unpadded tensor, pad_pano(1) layout on the panorama."""
    return [gn("gn_prep", N, H, W, C, circ=1 if pano else 0)]


def _seams(pairs, pers, pano):
    """The decoder's torch.cat([hidden, skip], 1) at each (C1, C2), perspective and panorama."""
    out = []
    for (C1, C2), (Np, hp), (Ne, he, we) in zip(pairs, pers, pano):
        out += [gn("gn_prep", Np, hp, hp, C1, C2), gn("gn_prep", Ne, he, we, C1, C2, cs=2, circ=2)]
    return out


def _prep_layouts(C):
    """pf_conv_prep without statistics: Downsample2D's stride-2 phases (zero-padded and pad_pano(2)), Upsample2D's
    pad_pano(1) + halo input, the ControlNet's zero halo."""
    return [gn("prep", 2, 8, 16, C, phases=4), gn("prep", 2, 8, 12, C, circ=2, phases=4),
            gn("prep", 2, 8, 16, C, circ=1), gn("prep", 2, 8, 8, C)]


GN_CASES = {
    # the tiny config (block widths 64 / 128) the models' tests run: 2 views of 16 x 16 and a 16 x 32 panorama
    "unet_tiny": lambda: [x for C in (64, 128) for x in (_unet_level(4, 16, 16, C, False) + _unet_level(2, 16, 32, C, True)
                                                         + _conv_out(2, 16, 32, C, True) + _conv_out(4, 16, 16, C, False)
                                                         + _unet_level(2, 2, 4, C, True))]
                         + [gn("gn_prep", 2, 8, 8, 64, ld_pad=64), gn("gn_prep", 2, 8, 16, 64, 64, cs=2, circ=2, ld_pad=8)],
    # bench c2 at SD-2 widths: 16 views (8 per CFG element), a 64 x 128 panorama pair
    "unet_sd2_c2_pers": lambda: (_unet_level(16, 64, 64, 320, False) + _unet_level(16, 32, 32, 640, False)
                                 + _unet_level(16, 16, 16, 1280, False) + _unet_level(16, 8, 8, 1280, False)
                                 + _conv_out(16, 64, 64, 320, False)),
    "unet_sd2_c2_pano": lambda: (_unet_level(2, 64, 128, 320, True) + _unet_level(2, 32, 64, 640, True)
                                 + _unet_level(2, 16, 32, 1280, True) + _unet_level(2, 8, 16, 1280, True)
                                 + _conv_out(2, 64, 128, 320, True)),
    # bench c4: 40 views, a 128 x 256 panorama pair
    "unet_sd2_c4": lambda: (_unet_level(40, 64, 64, 320, False) + _unet_level(2, 128, 256, 320, True)
                            + _conv_out(2, 128, 256, 320, True)),
    "decoder_seams": lambda: (
        _seams([(1280, 1280), (1280, 640), (640, 640), (640, 320), (320, 320)],
               [(16, 8), (16, 32), (16, 32), (16, 64), (16, 64)],
               [(2, 8, 16), (2, 32, 64), (2, 32, 64), (2, 64, 128), (2, 64, 128)])
        + _seams([(128, 128), (128, 64), (64, 64)], [(4, 16)] * 3, [(2, 16, 32)] * 3)),
    # the VAE (stats+prep, zero padding): 512 x 1024 image levels at 128, 256 and 512 channels, the mid-block
    # attention's plain GroupNorm, and the tiny widths
    "vae": lambda: ([gn("stats+prep", 1, 512, 1024, C) for C in (128, 256, 512)]
                    + [gn("stats+prep", 2, 64, 128, 512), gn("stats+prep", 2, 64, 128, 512, halo=0, act=NONE)]
                    + [gn("stats+prep", 2, 16, 32, C, halo=h, act=a) for C in (64, 128, 256)
                       for h, a in ((1, SILU), (0, NONE))]),
    "prep_layouts": lambda: ([x for C in (64, 128, 256, 320, 512, 640, 1280) for x in _prep_layouts(C)]
                             + [gn("prep", 2, 6, 10, 128, circ=1, up=2), gn("prep", 2, 6, 10, 128, up=2)]  # nearest x2
                             + [gn("prep", 2, 8, 8, 64, ld_pad=64)]),
}


def _gn_operands(g, s, dt, dev):
    Cc = s["C1"] + s["C2"]
    x = ct.gn_operand(g, s["N"], s["H"], s["W"], Cc, GROUPS, dt).to(dev)
    gamma = (torch.randn(Cc, generator=g) * 0.5 + 1.0).to(dev)
    beta = (torch.randn(Cc, generator=g) * 0.5).to(dev)

    def src(lo, hi):  # channels [lo, hi) of x as a tensor of row stride hi - lo + ld_pad
        if hi == lo:
            return None
        buf = _nan((x.shape[0], hi - lo + s["ld_pad"]), dt, dev)
        buf[:, :hi - lo] = x[:, lo:hi]
        return buf[:, :hi - lo]
    return x, src(0, s["C1"]), src(s["C1"], Cc), gamma, beta


def _out_rows(s, N):
    Hu, Wu = s["H"] * s["up"], (s["W"] + 2 * s["circ"]) * s["up"]
    Ho, Wo = (Hu // 2 + 1, Wu // 2 + 1) if s["phases"] == 4 else (Hu + 2 * s["halo"], Wu + 2 * s["halo"])
    return s["phases"] * N * Ho * Wo, (s["phases"], N, Ho * Wo)


def _launch_gn(s, x1, x2, gamma, beta, N):
    """Run one spec on N images; -> (out, mean_rstd or None, cat_out or None, counters)."""
    from panfusion_b200 import _lib
    lib, dt, dev = _lib.lib(), x1.dtype, x1.device
    Cc = s["C1"] + s["C2"]
    rows, _ = _out_rows(s, N)
    out = _nan((rows, Cc), dt, dev)
    counters = torch.zeros(N, dtype=torch.int32, device=dev)
    args = (s["circ"], s["up"], s["phases"], s["halo"])
    if s["entry"] == "gn_prep":
        ws = _nan((lib.pf_gn_prep_ws_floats(N, GROUPS),), torch.float32, dev)
        cat = _nan((N * s["H"] * s["W"], Cc), dt, dev) if x2 is not None else None
        _lib.check(lib.pf_gn_prep(_vp(x1), x1.stride(0), s["C1"], _vp(x2), x2.stride(0) if x2 is not None else 0, s["C2"],
                                  _vp(cat), _vp(out), _lib.dtype_code(dt), N, s["H"], s["W"], GROUPS, C.c_float(EPS),
                                  _vp(gamma), _vp(beta), s["act"], s["cs"], *args, _vp(ws), _vp(counters), _st()))
        mr = ws[N * GN_MAX_SLABS * GROUPS * 2:].reshape(N, GROUPS, 2)
        return out, mr, cat, counters
    mr = None
    if s["entry"] == "stats+prep":
        ws = _nan((lib.pf_groupnorm_ws_floats(N, GROUPS),), torch.float32, dev)
        mr = _nan((N, GROUPS, 2), torch.float32, dev)
        _lib.check(lib.pf_groupnorm_stats(_vp(x1), _lib.dtype_code(dt), N, s["H"], s["W"], Cc, x1.stride(0), GROUPS,
                                          s["cs"], C.c_float(EPS), _vp(ws), _vp(counters), _vp(mr), _st()))
    _lib.check(lib.pf_conv_prep(_vp(x1), _vp(out), _lib.dtype_code(dt), N, s["H"], s["W"], Cc, x1.stride(0), _vp(mr),
                                _vp(gamma if mr is not None else None), _vp(beta if mr is not None else None), GROUPS,
                                s["act"], *args, _st()))
    return out, mr, None, counters


def _image(s, t, n, N, what):
    """Image n's part of an output: the layout [phases][N][Ho][Wo][C] or the tokens [N * H * W, C]."""
    if what == "out":
        _, shape = _out_rows(s, N)
        return t.reshape(*shape, -1)[:, n]
    hw = s["H"] * s["W"]
    return t[n * hw:(n + 1) * hw]


def _check_gn(s, g, dt, dev):
    """-> (worst stats err/bound, worst output err/bound) of one spec; asserts the exact properties."""
    N, H, W = s["N"], s["H"], s["W"]
    x, x1, x2, gamma, beta = _gn_operands(g, s, dt, dev)
    out, mr, cat, counters = _launch_gn(s, x1, x2, gamma, beta, N)
    out2, mr2, cat2, counters2 = _launch_gn(s, x1, x2, gamma, beta, N)
    torch.cuda.synchronize()
    label = f"{s['entry']} N={N} {H}x{W} C={s['C1']}+{s['C2']} cs={s['cs']} circ={s['circ']} up={s['up']} " \
            f"ph={s['phases']} halo={s['halo']} act={s['act']} ld+{s['ld_pad']} {dt}"
    assert (counters == 0).all() and (counters2 == 0).all(), label
    assert _same(out, out2) and (mr is None or _same(mr, mr2)), f"repeat launch differs: {label}"
    if cat is not None:
        assert _same(cat, x) and _same(cat2, x), label
    ws = 0.0
    if mr is not None:
        entry = "pf_gn_prep" if s["entry"] == "gn_prep" else "pf_groupnorm_stats"
        ref, bound = ct.gn_stats_ref(x, N, H, W, GROUPS, s["cs"], EPS, ct.gn_partition(entry, H, W, x.shape[1]))
        ws = ct.worst_ratio(mr, ref, bound)
    ref, bound = ct.gn_apply_ref(x, N, H, W, mr, gamma, beta, act=s["act"], circ=s["circ"], up=s["up"],
                                 phases=s["phases"], halo=s["halo"], out_dtype=dt)
    wo = ct.worst_ratio(out, ref, bound)
    del ref, bound
    if N > 1:  # the last image launched alone: the same bytes
        n, hw = N - 1, H * W
        sub = lambda t: None if t is None else t[n * hw:(n + 1) * hw]
        o1, m1, c1, k1 = _launch_gn(s, sub(x1), sub(x2), gamma, beta, 1)
        torch.cuda.synchronize()
        img = _image(s, out, n, N, "out")
        assert (k1 == 0).all() and _same(o1.reshape(img.shape), img), f"batch-variant output: {label}"
        assert m1 is None or _same(m1[0], mr[n]), f"batch-variant statistics: {label}"
        assert c1 is None or _same(c1, _image(s, cat, n, N, "tokens")), label
    print(f"[contract] groupnorm {label}: stats err/bound {ws:.3f}, output {wo:.3f}")
    return ws, wo


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", list(GN_CASES))
def test_groupnorm_contract(cuda_device, case, dtype):
    g = torch.Generator().manual_seed(sum(map(ord, case)))
    worst = [0.0, 0.0]
    for s in GN_CASES[case]():
        r = _check_gn(s, g, dtype, cuda_device)
        worst = [max(a, b) for a, b in zip(worst, r)]
    print(f"[contract] groupnorm {case} {dtype}: worst stats {worst[0]:.3f}, output {worst[1]:.3f}")
    assert max(worst) <= 1.0, worst


# ---- LayerNorm ------------------------------------------------------------------------------------------------------

def ln(T, C, pe_rows=0, ld_rows=0, label=""):
    """One pf_layernorm call: T tokens of width C, a PE table of pe_rows rows (0: none), x read as the first C columns
    of rows ld_rows * C wide (0: contiguous)."""
    return dict(T=T, C=C, pe_rows=pe_rows, ld_rows=ld_rows, label=label)


LN_CASES = {
    # EPPA norm1(x + PE) at bench c2's three levels: 16 views (pe of the 8-view rig, shared by the CFG pair) and the
    # 2 panoramas; level 0 runs 16 384 view tokens, past one wave of warps
    "eppa_c2": lambda: [ln(16 * 1024, 320, 8 * 1024, label="c2 views L0"), ln(2 * 2048, 320, 2048, label="c2 pano L0"),
                        ln(16 * 256, 640, 8 * 256, label="c2 views L1"), ln(2 * 512, 640, 512, label="c2 pano L1"),
                        ln(16 * 64, 1280, 8 * 64, label="c2 views L2"), ln(2 * 128, 1280, 128, label="c2 pano L2")],
    # bench c4: 40 icosahedron views of 32 x 32 and the 64 x 128 panorama level
    "eppa_c4": lambda: [ln(40 * 1024, 320, 20 * 1024, label="c4 views"), ln(2 * 8192, 320, 8192, label="c4 pano")],
    # MVDiffusion's LayerNorm(x + query_pe) (one PE row) at the SD-2-width levels of 16 views of 64 x 64 / 32 x 32
    "mvdiffusion_query_pe": lambda: [ln(16 * 4096, 320, 1, label="query_pe 64x64"), ln(16 * 1024, 640, 1, label="query_pe 32x32")],
    # the text tower's final LayerNorm (CFG pair of 77 tokens, SD-2 width) and the CLIP vision tower's post-LN of the
    # class-token rows, a strided view (ldx = 197 * 768)
    "towers": lambda: [ln(154, 1024, label="text final"), ln(20, 1024, label="text short"),
                       ln(4, 768, ld_rows=197, label="clip post-LN"), ln(9000, 768, ld_rows=2, label="strided, two waves")],
    "tiny": lambda: [ln(2 * 128, 64, 128, label="tiny views"), ln(2 * 64, 128, 32, label="tiny pano"),
                     ln(33, 64, label="33 tokens"), ln(100, 2048, 50, label="C = 2048")],
}


def _run_ln(s, g, dt, dev):
    from panfusion_b200 import _lib
    T, Cc = s["T"], s["C"]
    ld = s["ld_rows"] * Cc if s["ld_rows"] else Cc
    base = ((torch.randn(T, ld, generator=g) * 1.5 + 0.3)
            + 2 * torch.rand(T, 1, generator=g) - 1).to(dt).to(dev)  # each token its own offset
    x = base[:, :Cc]
    pe = torch.randn(s["pe_rows"], Cc, generator=g).to(dev) if s["pe_rows"] else None
    gamma, beta = torch.randn(Cc, generator=g).to(dev), torch.randn(Cc, generator=g).to(dev)
    out = _nan((T, Cc), dt, dev)
    _lib.check(_lib.lib().pf_layernorm(_vp(x), x.stride(0), _vp(out), out.stride(0), _lib.dtype_code(dt), T, Cc, _vp(pe),
                                       s["pe_rows"], _vp(gamma), _vp(beta), C.c_float(EPS), _st()))
    return x, pe, gamma, beta, out


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", list(LN_CASES))
def test_layernorm_contract(cuda_device, case, dtype):
    g = torch.Generator().manual_seed(sum(map(ord, case)))
    worst = 0.0
    for s in LN_CASES[case]():
        x, pe, gamma, beta, out = _run_ln(s, g, dtype, cuda_device)
        ref, bound = ct.layernorm_ref(x, pe, gamma, beta, EPS, dtype)
        r = ct.worst_ratio(out, ref, bound)
        print(f"[contract] layernorm {s['label']} T={s['T']} C={s['C']} pe_rows={s['pe_rows']} {dtype}: err/bound {r:.3f}")
        worst = max(worst, r)
    assert worst <= 1.0, worst


# ---- token embedding, CFG + DDIM, timestep embedding ----------------------------------------------------------------

@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("T,L,Cc", [(154, 77, 1024), (40, 20, 64), (77, 77, 768)])
def test_embed_tokens_contract(cuda_device, dtype, T, L, Cc):
    """pf_embed_tokens: the row is exactly fl16(tok[id] + pos[t % L]); (sum, sum of squares) of the stored row within
    row_stats_ref's bound; the two spare slots are zero."""
    from panfusion_b200 import _lib
    g = torch.Generator().manual_seed(T + Cc)
    vocab = 1000
    tok, pos = torch.randn(vocab, Cc, generator=g) * 0.5 + 0.2, torch.randn(L, Cc, generator=g) * 0.2
    ids = torch.randint(0, vocab, (T,), generator=g)
    dev = cuda_device
    tok_d, pos_d, ids_d = tok.to(dev), pos.to(dev), ids.to(dev)
    out = _nan((T, Cc), dtype, dev)
    st = torch.full((T, 2, 2), float("nan"), device=dev)
    _lib.check(_lib.lib().pf_embed_tokens(_vp(ids_d), _vp(tok_d), _vp(pos_d), _vp(out), _lib.dtype_code(dtype), _vp(st),
                                          T, L, Cc, vocab, _st()))
    row, ref, bound = ct.row_stats_ref(tok_d, pos_d, ids_d, L, dtype)
    assert _same(out, row)
    r = float(((st[:, 0].double() - ref).abs() / bound).max())
    print(f"[contract] embed_tokens T={T} L={L} C={Cc} {dtype}: stats err/bound {r:.3f}")
    assert (st[:, 1] == 0).all() and r <= 1.0, r


# (views per CFG element, view latent side, pano latent H x W): bench c2 and c4, and the tiny sampler test's rig
DDIM_SHAPES = {"c2": (8, 64, (64, 128)), "c4": (20, 64, (128, 256)), "tiny": (4, 16, (16, 32))}


@pytest.mark.parametrize("shape", list(DDIM_SHAPES))
def test_cfg_ddim_step_dev_contract(cuda_device, shape):
    """pf_cfg_ddim_step_dev as PanFusionSampler._step_body launches it: the views with no roll, the panorama rolled by
    a quarter turn, coefficients from the sampler's fp32 coef_table at three steps of the 50-step schedule."""
    from panfusion_b200 import _lib
    from panfusion_b200.sampler import DDIMSchedule
    m, h, (He, We) = DDIM_SHAPES[shape]
    sched = DDIMSchedule()
    sched.set_timesteps(50)
    table = torch.tensor([sched.coefficients(int(t)) for t in sched.timesteps], dtype=torch.float32)
    g = torch.Generator().manual_seed(m + h)
    dev = cuda_device
    worst = 0.0
    for step in (0, 25, 49):
        coef = table[step].to(dev)
        for lat, roll in (((1, m, 4, h, h), 0), ((1, 1, 4, He, We), We // 4)):
            x = torch.randn(lat, generator=g).to(dev)
            eps = torch.randn((2, *lat[1:]), generator=g).to(dev)
            out = torch.full_like(x, float("nan"))
            _lib.check(_lib.lib().pf_cfg_ddim_step_dev(_vp(x), _vp(eps), _vp(out), C.c_longlong(x.numel()), lat[-1], roll,
                                                      C.c_float(9.0), _vp(coef), _st()))
            ref, bound = ct.cfg_ddim_ref(x, eps, coef, 9.0, roll)
            worst = max(worst, ct.worst_ratio(out, ref, bound))
    print(f"[contract] cfg_ddim_step_dev {shape}: worst err/bound {worst:.3f}")
    assert worst <= 1.0, worst


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("dim", [320, 64])
def test_timestep_embed_contract(cuda_device, dtype, dim):
    """pf_timestep_embed at the schedule's ends (t = 999 and t = 1) and between, at SD-2's and the tiny config's width."""
    from panfusion_b200 import _lib
    t = torch.tensor([999.0, 1.0, 981.0, 21.0, 500.0], device=cuda_device)
    out = _nan((t.numel(), dim), dtype, cuda_device)
    _lib.check(_lib.lib().pf_timestep_embed(_vp(t), _vp(out), _lib.dtype_code(dtype), t.numel(), dim, _st()))
    ref, bound = ct.timestep_ref(t, dim, dtype)
    r = ct.worst_ratio(out, ref, bound)
    print(f"[contract] timestep_embed dim={dim} {dtype}: err/bound {r:.3f}")
    assert r <= 1.0, r


# ---- the table covers the models ------------------------------------------------------------------------------------

def _model_calls(dev):
    """The normalisation calls of: the tiny PanFusion forward (shared and per-batch cameras) and its 1 x 2 view-sharded
    ranks; the tiny MVDiffusion step; the CLIP text encoder; the CLIP image tower (all through the attention file's
    model runs); the tiny ControlNet forward; VAE encode and decode at the tiny and SD-2 widths; one sampler step."""
    from oracle import synth, unet as ou, vae as ov
    from panfusion_b200 import vae as pv
    from panfusion_b200.sampler import PanFusionSampler
    from test_gpu_attention_contract import _model_calls as attention_model_calls
    from test_gpu_mvgen import _build_cn_pair, _to_dev
    from test_gpu_sampler import _setup
    dt = torch.float16
    attention_model_calls(dev)
    cfg = ou.TINY_CONFIG
    _, cn = _build_cn_pair(dev, cfg, dt, True)
    inp = synth.step_inputs(2, (16, 32), (16, 16), cfg["cross_attention_dim"], seed=0)
    inp.update(synth.layout_conds(1, 2, (16, 32), (16, 16), seed=5, pers=True))
    cn(**_to_dev(inp, dev))
    g = torch.Generator().manual_seed(0)
    for vcfg in (ov.TINY_VAE_CONFIG, ov.SD2_VAE_CONFIG):
        orc = ov.build_vae(vcfg)
        pv.VAEEncoder(orc, compute_dtype=dt).prepare(dev, dt).moments((torch.rand(2, 3, 64, 64, generator=g) * 2 - 1).to(dev))
        pv.VAEDecoder(orc, compute_dtype=dt).prepare(dev, dt).decode(torch.randn(2, 4, 8, 16, generator=g).to(dev))
    _, mine, cams, pano, lat, prompt, pano_prompt = _setup(dev, dt)
    PanFusionSampler(mine, use_cuda_graph=False).denoise(lat.to(dev), pano.to(dev), prompt.to(dev), pano_prompt.to(dev),
                                                         cams, num_steps=1, rotate_back=False)
    torch.cuda.synchronize()


def test_norm_call_table_covers_the_models(recorder, cuda_device):
    """Every normalisation / sampler call class the models make is one a case above launches."""
    g = torch.Generator().manual_seed(0)
    dt, dev = torch.float16, cuda_device
    for build in GN_CASES.values():
        for s in build():
            _, x1, x2, gamma, beta = _gn_operands(g, s, dt, dev)
            _launch_gn(s, x1, x2, gamma, beta, s["N"])
    for build in LN_CASES.values():
        for s in build():
            _run_ln(s, g, dt, dev)
    test_embed_tokens_contract(dev, dt, 154, 77, 1024)
    for shape in DDIM_SHAPES:
        test_cfg_ddim_step_dev_contract(dev, shape)
    test_timestep_embed_contract(dev, dt, 320)
    torch.cuda.synchronize()
    covered = set(recorder.calls)
    recorder.calls.clear()
    _model_calls(dev)
    seen = set(recorder.calls)
    assert {c[0] for c in seen} == set(ENTRIES), "a model made no call of one of the entry points"
    for c in sorted(seen, key=str):
        print(f"[contract] norm call class {c}{'' if c in covered else '  <- no case'}")
    missing = sorted(seen - covered, key=str)
    assert not missing, f"call classes without a contract case: {missing}"
