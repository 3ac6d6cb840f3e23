"""-m gpu: the element-wise kernels of csrc/elementwise.cu at the shapes the models run them. pf_conv_in, pf_softmax_rows,
pf_gaussian_sample and pf_mse_loss are held to the fp64 contracts of tests/_contract.py; pf_add_noise and
pf_tensor_to_image must be bit-exact against the reference's eager fp32 ops.

Every output starts NaN-filled (uint8 outputs with a sentinel), with spare elements past the end or around the slice,
so a store outside the contract or a position never written fails. The last test runs the models through a recorder
of the library handle and requires every pf_* entry point they launch to be held by a named test file."""
import ctypes as C
import math
import re
from pathlib import Path

import pytest
import torch

import _contract as ct

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]
NONE, SILU = ct.ACT_NONE, ct.ACT_SILU
SPARE = 8  # rows past the end of an output that must stay untouched


def _nan(shape, dtype, dev):
    return torch.full(shape, float("nan"), dtype=dtype, device=dev)


def _vp(t):
    return C.c_void_p(0 if t is None else t.data_ptr())


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _spare(t):
    """t with SPARE NaN rows appended (what the contract leaves unwritten)."""
    return torch.cat([t, torch.full((SPARE, *t.shape[1:]), float("nan"), dtype=t.dtype, device=t.device)])


def _bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32)


# ---- pf_conv_in -----------------------------------------------------------------------------------------------------

def ci(N, Cin, H, W, Cout, circ=False, act=NONE, bias=True, real=None, fold=None, label=""):
    """One pf_conv_in call; `real` output channels carry weights (the rest are zero padding), `fold` takes the
    decoder's folded weights ("conv_in_w" or "conv_in_w_unscale") and a ones channel."""
    return dict(N=N, Cin=Cin, H=H, W=W, Cout=Cout, circ=circ, act=act, bias=bias, real=real or Cout, fold=fold,
                label=label)


CONV_IN_CASES = {
    # UNet conv_in at bench c2: 8 views per CFG element of 64 x 64 latents, the 64 x 128 panorama (circular)
    "unet_sd2": lambda: [ci(16, 4, 64, 64, 320, label="c2 views"), ci(2, 4, 64, 128, 320, circ=True, label="c2 pano")],
    "unet_tiny": lambda: [ci(4, 4, 16, 16, 64, label="tiny views"), ci(2, 4, 16, 32, 64, circ=True, label="tiny pano")],
    # ControlNet conditioning embedding: 3 -> 16 with SiLU at image resolution, padded to 64 output channels
    "controlnet": lambda: [ci(1, 3, 512, 1024, 64, act=SILU, real=16, label="cond 512x1024"),
                           ci(2, 3, 64, 126, 64, act=SILU, real=16, label="cond W % 4 != 0")],
    # VAE decoder conv_in over [z | ones] with post_quant_conv folded in (and decode_latent's 1 / scaling_factor)
    "vae_decoder": lambda: [ci(2, 5, 64, 64, 512, fold="conv_in_w_unscale", label="decode_latent 64x64"),
                            ci(1, 5, 64, 144, 512, fold="conv_in_w", label="decode_pano 64x144")],
    "vae_encoder": lambda: [ci(1, 3, 512, 512, 128, label="encode 512x512"), ci(1, 3, 512, 1024, 128, label="encode 512x1024")],
    # no bias, Cout = 8, both paths, and a W % 4 != 0 launch whose CTAs loop many times
    "edges": lambda: [ci(3, 4, 16, 20, 8, bias=False, label="Cout 8 no bias"), ci(3, 4, 16, 18, 8, bias=False, circ=True),
                      ci(2, 3, 256, 510, 128, label="W % 4 != 0, grid-stride"), ci(2, 4, 64, 126, 320, circ=True)],
}


def _conv_in_operands(s, g, dev, dt):
    N, Cin, H, W, Cout = s["N"], s["Cin"], s["H"], s["W"], s["Cout"]
    x = torch.randn(N, Cin, H, W, generator=g)
    x[..., 0] += 2.0   # the two sides of the seam differ
    x[..., -1] -= 2.0
    if s["fold"]:
        from oracle import vae as ov
        from panfusion_b200 import vae as pv
        p = pv.VAEDecoderPack(ov.build_vae(ov.SD2_VAE_CONFIG), dev, dt)
        x[:, 4] = 1.0
        return x.to(dev), getattr(p, s["fold"]), p.conv_in_b
    w = torch.zeros(Cout, Cin, 3, 3)
    w[:s["real"]] = torch.randn(s["real"], Cin, 3, 3, generator=g) * 0.3
    b = torch.zeros(Cout)
    b[:s["real"]] = torch.randn(s["real"], generator=g)
    return x.to(dev), w.to(dev), b.to(dev) if s["bias"] else None


def _launch_conv_in(x, w, b, dt, circ, act):
    from panfusion_b200 import _lib
    N, Cin, H, W = x.shape
    out = _nan((N * H * W + SPARE, w.shape[0]), dt, x.device)
    _lib.check(_lib.lib().pf_conv_in(_vp(x), _vp(w), _vp(b), _vp(out), _lib.dtype_code(dt), N, Cin, H, W, w.shape[0],
                                     int(circ), act, _st()))
    return out


def _grid_passes(s):
    """Grid-stride iterations of the busiest CTA: elementwise.cu launches min(ceil(total / 256), 4 SMs) CTAs."""
    total = s["N"] * s["H"] * (s["W"] // 4 if s["W"] % 4 == 0 else s["W"]) * (s["Cout"] // 8)
    ctas = min(-(-total // 256), 4 * torch.cuda.get_device_properties(0).multi_processor_count)
    return -(-total // (ctas * 256))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", list(CONV_IN_CASES))
def test_conv_in_contract(cuda_device, case, dtype):
    g = torch.Generator().manual_seed(sum(map(ord, case)))
    worst = 0.0
    for s in CONV_IN_CASES[case]():
        x, w, b = _conv_in_operands(s, g, cuda_device, dtype)
        out = _launch_conv_in(x, w, b, dtype, s["circ"], s["act"])
        ref, bound = ct.conv_in_ref(x, w, b, s["circ"], s["act"], dtype)
        r = ct.worst_ratio(out, _spare(ref), _spare(bound))
        if s["real"] < s["Cout"]:
            assert (out[:-SPARE, s["real"]:] == 0).all(), "zero-padded output channels are not exactly zero"
        print(f"[contract] conv_in {s['label']} N={s['N']} {s['Cin']}->{s['Cout']} {s['H']}x{s['W']} circ={s['circ']} "
              f"act={s['act']} bias={b is not None} passes={_grid_passes(s)} {dtype}: err/bound {r:.3f}")
        worst = max(worst, r)
        del out, ref, bound
    assert worst <= 1.0, worst


def test_conv_in_cases_reach_both_paths_and_loop(cuda_device):
    """The cases above run both code paths, and each path in a launch whose CTAs take several grid-stride passes."""
    specs = [s for build in CONV_IN_CASES.values() for s in build()]
    for quad in (True, False):
        assert max(_grid_passes(s) for s in specs if (s["W"] % 4 == 0) == quad) >= 4


# ---- pf_softmax_rows ------------------------------------------------------------------------------------------------

def sm(rows, cols, ld_pad=0, off=0, ldo_pad=0):
    """rows x cols logits read from rows ld_pad wider; probabilities written to columns [off, off + cols) of rows
    off + cols + ldo_pad wide (rounded up to even)."""
    return dict(rows=rows, cols=cols, ld_pad=ld_pad, off=off, ldo_pad=ldo_pad)


SCALE = 512 ** -0.5  # the VAE mid-block attention: one head of width 512
SOFTMAX_CASES = {
    "vae_64x64": [sm(4096, 4096)],                     # 64 x 64 latents
    "vae_64x144": [sm(9216, 9216)],                    # the padded 64 x 144 panorama latent
    "edges": [sm(7, 100, ld_pad=5, off=2, ldo_pad=3), sm(5, 777, off=4), sm(4, 1023, ld_pad=1, ldo_pad=1),
              sm(4, 1025, off=2, ldo_pad=2), sm(3, 511), sm(3, 513), sm(3, 4097, ld_pad=7, off=6, ldo_pad=1), sm(3, 1)],
}


def _logits(s, g, dev):
    """Each row its own offset in [-200, 200] and a spread of +-50 after scaling; row 0 has one dominant logit and
    row 1 is constant."""
    rows, cols = s["rows"], s["cols"]
    base = torch.empty(rows, cols + s["ld_pad"], device=dev)
    off = 400 * torch.rand(rows, 1, device=dev, generator=g) - 200
    base.copy_((off + 50 * (2 * torch.rand(rows, cols + s["ld_pad"], device=dev, generator=g) - 1)) / SCALE)
    x = base[:, :cols]
    if rows > 1:
        x[0, cols // 3] = x[0].max() + 60 / SCALE
        x[1] = 3.7
    return x


def _launch_softmax(x, dt, off, width):
    from panfusion_b200 import _lib
    buf = _nan((x.shape[0], width), dt, x.device)
    out = buf[:, off:off + x.shape[1]]
    _lib.check(_lib.lib().pf_softmax_rows(_vp(x), C.c_longlong(x.stride(0)), _vp(out), C.c_longlong(buf.stride(0)),
                                          _lib.dtype_code(dt), C.c_longlong(x.shape[0]), x.shape[1], C.c_float(SCALE),
                                          _st()))
    return buf


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", list(SOFTMAX_CASES))
def test_softmax_rows_contract(cuda_device, case, dtype):
    g = torch.Generator(device=cuda_device).manual_seed(sum(map(ord, case)))
    worst = 0.0
    for s in SOFTMAX_CASES[case]:
        x = _logits(s, g, cuda_device)
        width = s["off"] + s["cols"] + s["ldo_pad"]
        width += width % 2
        buf = _launch_softmax(x, dtype, s["off"], width)
        r = 0.0
        for r0 in range(0, s["rows"], 1024):  # the fp64 reference a block of rows at a time
            rows = slice(r0, min(s["rows"], r0 + 1024))
            ref, bound = ct.softmax_rows_ref(x[rows], SCALE, dtype)
            full = lambda t: torch.nn.functional.pad(t, (s["off"], width - s["off"] - s["cols"]), value=float("nan"))
            r = max(r, ct.worst_ratio(buf[rows], full(ref), full(bound)))
        print(f"[contract] softmax_rows {s['rows']}x{s['cols']} ld+{s['ld_pad']} out[{s['off']}:] ldo={width} {dtype}: "
              f"err/bound {r:.3f}")
        worst = max(worst, r)
    assert worst <= 1.0, worst


def _built_from_these_sources():
    from panfusion_b200 import _lib, build
    stamp = build.LIBDIR / "build.sha256"
    return _lib.LIB_PATH == build.LIB and stamp.exists() and stamp.read_text().strip() == build._digest()


def test_softmax_rows_refuses_a_misaligned_output(cuda_device):
    """An output slice that starts at an odd 16-bit column is refused on the host (the kernel stores column pairs as
    32-bit words). Only run against a library built from these sources: an older build would launch the store."""
    from panfusion_b200 import _lib
    if not _built_from_these_sources():
        pytest.skip("the loaded library was not built from this tree's sources")
    x = torch.randn(4, 64, device=cuda_device)
    buf = torch.zeros(4, 66, dtype=torch.float16, device=cuda_device)
    with pytest.raises(ValueError, match="aligned"):
        _lib.check(_lib.lib().pf_softmax_rows(_vp(x), C.c_longlong(64), _vp(buf[:, 1:65]), C.c_longlong(66),
                                              _lib.dtype_code(torch.float16), C.c_longlong(4), 64, C.c_float(1.0), _st()))
    torch.cuda.synchronize()
    assert not buf.any()


# ---- pf_gaussian_sample ---------------------------------------------------------------------------------------------

LOGVAR_EDGES = [-30.0, 20.0, math.nextafter(-30.0, 0.0), math.nextafter(20.0, 0.0), math.nextafter(-30.0, -100.0),
                math.nextafter(20.0, 100.0), -30.5, 20.5, -1e30, 1e30, -math.inf, math.inf]


def _launch_gaussian(mom, eps, L, scale, fill):
    from panfusion_b200 import _lib
    N, _, h, w = eps.shape
    out = torch.full((N * L * h * w + SPARE,), float("nan"), device=eps.device)
    out[:-SPARE] = fill
    _lib.check(_lib.lib().pf_gaussian_sample(_vp(mom), mom.stride(0), _vp(eps), _vp(out), N, L, h * w, C.c_float(scale),
                                             _st()))
    return out


def _check_gaussian(mom, eps, L, scale, fill=float("nan")):
    out = _launch_gaussian(mom, eps, L, scale, fill)
    ref, bound = ct.gaussian_sample_ref(mom, mom.stride(0), eps, L, scale)
    return ct.worst_ratio(out, torch.cat([ref.reshape(-1), torch.full((SPARE,), math.nan, device=ref.device,
                                                                      dtype=ref.dtype)]),
                          torch.cat([bound.reshape(-1), torch.full((SPARE,), 1.0, device=ref.device, dtype=ref.dtype)]))


@pytest.mark.parametrize("scale", [1.0, 0.18215])
def test_gaussian_sample_contract(cuda_device, scale):
    """The encoder's moments layout (rows of 64 floats, [mean | logvar] in the first 8, the rest NaN so a read past
    2L shows), two 512 x 512 images' latents, logvars across both clamp edges and exactly at, just inside and just
    beyond them; then the real moments of the tiny VAE encoder."""
    from oracle import vae as ov
    from panfusion_b200 import vae as pv
    g = torch.Generator().manual_seed(int(scale * 1000))
    N, L, h, w, ld = 2, 4, 64, 64, 64
    mom = torch.full((N * h * w, ld), float("nan"))
    mom[:, :L] = torch.randn(N * h * w, L, generator=g) * 3
    mom[:, L:2 * L] = torch.rand(N * h * w, L, generator=g) * 60 - 35
    mom[:len(LOGVAR_EDGES), L + 1] = torch.tensor(LOGVAR_EDGES)
    mom[h * w:h * w + len(LOGVAR_EDGES), 2 * L - 1] = torch.tensor(LOGVAR_EDGES)  # the second image, the last channel
    eps = torch.randn(N, L, h, w, generator=g).to(cuda_device)
    r = _check_gaussian(mom.to(cuda_device), eps, L, scale)
    enc = pv.VAEEncoder(ov.build_vae(ov.TINY_VAE_CONFIG), torch.float16).prepare(cuda_device, torch.float16)
    o, N2, h2, w2 = enc.moments((torch.rand(2, 3, 64, 64, generator=g) * 2 - 1).to(cuda_device))
    r2 = _check_gaussian(o, torch.randn(N2, L, h2, w2, generator=g).to(cuda_device), L, scale)
    print(f"[contract] gaussian_sample scale={scale}: err/bound {r:.3f} (synthetic), {r2:.3f} (encoder moments)")
    assert max(r, r2) <= 1.0, (r, r2)


def test_gaussian_sample_propagates_nan(cuda_device):
    """A NaN mean or a NaN logvar gives a NaN latent, as torch.clamp and the eager formula give; every other element
    holds its contract. The output starts finite here, so an element left unwritten fails too."""
    g = torch.Generator().manual_seed(7)
    N, L, h, w, ld = 2, 4, 8, 8, 64
    mom = torch.randn(N * h * w, ld, generator=g)
    mom[5, 1] = float("nan")              # a mean
    mom[9, L + 2] = float("nan")          # a logvar
    mom[h * w + 3, 2 * L - 1] = float("nan")
    eps = torch.randn(N, L, h, w, generator=g).to(cuda_device)
    r = _check_gaussian(mom.to(cuda_device), eps, L, 0.18215, fill=0.0)
    print(f"[contract] gaussian_sample with NaN moments: err/bound {r:.3f}")
    assert r <= 1.0, r


# ---- pf_mse_loss ----------------------------------------------------------------------------------------------------

# bench c2's training shapes for one sample: 8 views of 64 x 64 latents and the 64 x 128 panorama latent
MSE_SIZES = [1, 100, 295, 296 * 37 - 1, 296 * 37 + 1, 296 * 1000 + 1, 8 * 4 * 64 * 64, 4 * 64 * 128]


def _mse(a, b, ws, counter):
    from panfusion_b200 import _lib
    out = torch.full((2,), float("nan"), device=a.device)
    _lib.check(_lib.lib().pf_mse_loss(_vp(a), _vp(b), C.c_longlong(a.numel()), _vp(ws), _vp(counter), _vp(out), _st()))
    return out


@pytest.mark.parametrize("n", MSE_SIZES)
def test_mse_loss_contract(cuda_device, n):
    """Within mse_ref's bound; a repeat launch gives the same bits and the counter is back at zero each time."""
    from panfusion_b200 import _lib
    g = torch.Generator().manual_seed(n)
    a = (torch.randn(n, generator=g) * 2 + 0.5).to(cuda_device)
    b = torch.randn(n, generator=g).to(cuda_device)
    ws = _nan((_lib.lib().pf_mse_loss_ws_floats(),), torch.float32, cuda_device)
    counter = torch.zeros(1, dtype=torch.int32, device=cuda_device)
    o1 = _mse(a, b, ws, counter)
    torch.cuda.synchronize()
    assert counter.item() == 0
    o2 = _mse(a, b, ws, counter)
    torch.cuda.synchronize()
    assert counter.item() == 0 and torch.equal(_bits(o1), _bits(o2))
    ref, bound = ct.mse_ref(a, b)
    r = ct.worst_ratio(o1, torch.stack([ref, ref.new_tensor(math.nan)]), torch.stack([bound, bound]))
    print(f"[contract] mse_loss n={n}: err/bound {r:.3f}")
    assert r <= 1.0, r


def test_mse_loss_graph_replay_is_bit_identical(cuda_device):
    """pf_mse_loss captured in a CUDA graph and replayed gives the eager launch's bits, and re-arms its counter."""
    from panfusion_b200 import _lib
    n = 8 * 4 * 64 * 64
    g = torch.Generator().manual_seed(1)
    a, b = torch.randn(n, generator=g).to(cuda_device), torch.randn(n, generator=g).to(cuda_device)
    ws = _nan((_lib.lib().pf_mse_loss_ws_floats(),), torch.float32, cuda_device)
    counter = torch.zeros(1, dtype=torch.int32, device=cuda_device)
    eager = _mse(a, b, ws, counter)
    out = torch.full((2,), float("nan"), device=cuda_device)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        _lib.check(_lib.lib().pf_mse_loss(_vp(a), _vp(b), C.c_longlong(n), _vp(ws), _vp(counter), _vp(out), _st()))
    for _ in range(3):
        out.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        assert counter.item() == 0 and torch.equal(_bits(out[:1]), _bits(eager[:1])) and torch.isnan(out[1])


# ---- pf_add_noise, pf_tensor_to_image: bit-exact ----------------------------------------------------------------------

@pytest.mark.parametrize("shape", [(2, 20, 4, 64, 64), (2, 1, 4, 64, 128), (2, 8, 4, 64, 64)])
def test_add_noise_bit_exact(cuda_device, shape):
    """pf_add_noise at training shapes, the schedule's first and last timestep, against the eager fp32 ops of
    diffusers' add_noise. 20 views of 64 x 64 hold 327 680 elements per sample, past the 1184 x 256 threads of one
    grid row, so the grid-stride loop runs twice. Only in-range timesteps: the kernel traps on any other."""
    from oracle import sampler as osamp, training as otr
    from panfusion_b200 import _lib
    g = torch.Generator().manual_seed(shape[1])
    abar = osamp.DDIM().alphas_cumprod.float()
    x0, noise = torch.randn(*shape, generator=g), torch.randn(*shape, generator=g)
    t = torch.tensor([0, abar.numel() - 1])
    dev = cuda_device
    x0d, nd, td, ad = x0.to(dev), noise.to(dev), t.to(dev), abar.to(dev)
    per = x0[0].numel()
    out = _nan((x0.numel() + SPARE,), torch.float32, dev)
    _lib.check(_lib.lib().pf_add_noise(_vp(x0d), _vp(nd), _vp(out), _vp(td), _vp(ad), abar.numel(), shape[0],
                                       C.c_longlong(per), _st()))
    want = otr.add_noise(x0, noise, t, abar).reshape(-1)
    assert torch.equal(out[:-SPARE].cpu(), want) and torch.isnan(out[-SPARE:]).all()


@pytest.mark.parametrize("shape", [(1, 3, 512, 1024), (8, 3, 512, 512)])
def test_tensor_to_image_bit_exact(cuda_device, shape):
    """pf_tensor_to_image on a 512 x 1024 panorama and a batch of 8 views, with exact rounding ties and values past
    [-1, 1], against the reference's eager ops; the bytes past the end keep their sentinel."""
    from oracle import vae as ov
    from panfusion_b200 import _lib
    g = torch.Generator().manual_seed(shape[0])
    x = torch.randn(*shape, generator=g) * 0.8
    x.view(-1)[:255] = (torch.arange(0, 255, dtype=torch.float32) + 0.5) / 255 * 2 - 1
    x.view(-1)[255:259] = torch.tensor([-1.5, 1.5, -1.0, 1.0])
    n, Cc, H, W = shape
    out = torch.full((x.numel() + 64,), 0xAB, dtype=torch.uint8, device=cuda_device)
    _lib.check(_lib.lib().pf_tensor_to_image(_vp(x.to(cuda_device)), _vp(out), C.c_longlong(n), Cc, H, W, _st()))
    want = torch.from_numpy(ov.tensor_to_image(x)).reshape(-1)
    assert torch.equal(out[:-64].cpu(), want) and (out[-64:] == 0xAB).all()


# ---- census: every entry point the models launch is held by a test file -------------------------------------------

# entry point -> the test file that holds it. pf_cfg_ddim_step (host coefficients) is absent on purpose: no model
# calls it, the sampler launches pf_cfg_ddim_step_dev.
REGISTRY = {
    "pf_check_device": "conftest.py",
    "pf_last_error": "test_cabi.py",
    "pf_gemm_taps": "test_gpu_contracts.py",
    "pf_gemm_pick_block_n": "test_cabi.py",
    "pf_gemm_splitk_plan": "test_gpu_contracts.py",
    "pf_gemm_row_stats_slots": "test_cabi.py",
    "pf_fmha_fwd": "test_gpu_attention_contract.py",
    "pf_bias_tile_flags": "test_gpu_attention_contract.py",
    "pf_bias_tile_scan": "test_gpu_attention_contract.py",
    "pf_bias_tile_pack": "test_gpu_attention_contract.py",
    "pf_cpattn_tables": "test_gpu_attention_contract.py",
    "pf_cpattn_gather": "test_gpu_attention_contract.py",
    "pf_cpattn_attn": "test_gpu_attention_contract.py",
    "pf_groupnorm_ws_floats": "test_gpu_norm_contract.py",
    "pf_groupnorm_stats": "test_gpu_norm_contract.py",
    "pf_gn_prep_ws_floats": "test_gpu_norm_contract.py",
    "pf_gn_prep": "test_gpu_norm_contract.py",
    "pf_conv_prep": "test_gpu_norm_contract.py",
    "pf_layernorm": "test_gpu_norm_contract.py",
    "pf_embed_tokens": "test_gpu_norm_contract.py",
    "pf_timestep_embed": "test_gpu_norm_contract.py",
    "pf_cfg_ddim_step_dev": "test_gpu_norm_contract.py",
    "pf_eppa_tables": "test_gpu_kernels.py",   # against the oracle and the reference-run goldens
    "pf_eppa_pe": "test_gpu_kernels.py",
    "pf_pad_pano": "test_gpu_kernels.py",
    "pf_copy2d": "test_gpu_kernels.py",
    "pf_e2p": "test_gpu_resample.py",
    "pf_e2p_shared": "test_gpu_resample.py",
    "pf_p2e": "test_gpu_resample.py",
    "pf_mp2e": "test_gpu_mvdiffusion.py",
    "pf_allgather_views": "test_gpu_multi.py",
    "pf_clip_prep_taps_ints": "test_gpu_clip_score.py",
    "pf_clip_prep_taps": "test_gpu_clip_score.py",
    "pf_clip_prep": "test_gpu_clip_score.py",
    "pf_clip_embed": "test_gpu_clip_score.py",
    "pf_layout_condition": "test_gpu_layout.py",
    "pf_conv_in": "test_gpu_elementwise_contract.py",
    "pf_softmax_rows": "test_gpu_elementwise_contract.py",
    "pf_gaussian_sample": "test_gpu_elementwise_contract.py",
    "pf_mse_loss_ws_floats": "test_gpu_elementwise_contract.py",
    "pf_mse_loss": "test_gpu_elementwise_contract.py",
    "pf_add_noise": "test_gpu_elementwise_contract.py",
    "pf_tensor_to_image": "test_gpu_elementwise_contract.py",
}


class _NameRecorder:
    """Stands in for the library handle: records the name of every pf_* symbol called, then forwards the call."""

    def __init__(self, lib):
        self._lib, self.names = lib, set()

    def __getattr__(self, name):
        f = getattr(self._lib, name)
        if not name.startswith("pf_"):
            return f

        def rec(*args):
            self.names.add(name)
            return f(*args)
        return rec


def _training_forward(dev):
    """One TrainingStep.loss forward of the tiny two-branch model (add_noise twice, both MSE terms), the latents
    drawn through the VAE encoder, and the uint8 conversion of a decoded panorama."""
    from oracle import synth, unet as ou, vae as ov
    from panfusion_b200 import vae as pv
    from panfusion_b200.training import TrainingStep
    from test_gpu_mvgen import _build_mine
    dt, cfg = torch.float16, ou.TINY_CONFIG
    _, mine = _build_mine(dev, cfg, dt)
    inp = synth.step_inputs(2, (16, 32), (16, 16), cfg["cross_attention_dim"], seed=3, batch=2)
    g = torch.Generator().manual_seed(5)
    orc = ov.build_vae(ov.TINY_VAE_CONFIG)
    enc = pv.VAEEncoder(orc, dt).prepare(dev, dt)
    lat, plat = TrainingStep.encode((torch.rand(2, 2, 3, 128, 128, generator=g) * 2 - 1).to(dev),
                                    (torch.rand(2, 1, 3, 128, 256, generator=g) * 2 - 1).to(dev), enc, 8,
                                    generator=torch.Generator(device=dev).manual_seed(1))
    cams = {k: v.to(dev) for k, v in inp["cameras"].items()}
    TrainingStep(mine).loss(lat, plat, inp["prompt_embd"].to(dev), inp["pano_prompt_embd"].to(dev), cams,
                            t=torch.tensor([0, 999], device=dev))
    pv.tensor_to_image(pv.VAEDecoder(orc, dt).prepare(dev, dt).decode(plat[:, 0]))
    torch.cuda.synchronize()


def test_every_entry_point_the_models_launch_is_held(monkeypatch, cuda_device):
    """Record the pf_* entry points of the model runs of test_gpu_norm_contract._model_calls (tiny PanFusion and its
    sharded ranks, MVDiffusion, the text and CLIP towers, ControlNet, VAE encode / decode, one sampler step) and of one
    training-step forward; each must be in REGISTRY, and its registered test file must exist and name it."""
    from panfusion_b200 import _lib
    from test_gpu_norm_contract import _model_calls
    rec = _NameRecorder(_lib.lib())
    monkeypatch.setattr(_lib, "lib", lambda: rec)
    _model_calls(cuda_device)
    _training_forward(cuda_device)
    here = Path(__file__).resolve().parent
    problems = []
    for name in sorted(rec.names):
        f = REGISTRY.get(name)
        text = (here / f).read_text() if f and (here / f).exists() else None
        state = ("NOT REGISTERED" if f is None else "file missing" if text is None else
                 "ok" if re.search(rf"\b{name}\b", text) else "file does not name it")
        print(f"[census] {name:28s} -> {f}: {state}")
        if state != "ok":
            problems.append((name, f, state))
    assert not problems, problems
