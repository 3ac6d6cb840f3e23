"""CPU: the error bounds of tests/_contract.py (used by test_gpu_contracts.py) are tight enough to fail.

Each case computes the exact fp64 result of a small tap-GEMM or attention, rounds it to the output type as a correct
kernel would, and checks that it passes the bound; then it emulates one subtle kernel bug (a dropped tap, a shifted
row-bias group, a halo row in the output, a residual read one row off, swapped GEGLU halves, an unmasked ragged key, a
bias read from the wrong batch) and checks that the bound catches it on at least one element. The convolution cases
(conv_ref, the contract of csrc/conv_mma.cuh) first pin conv_ref to F.conv2d, then emulate a seam column wrapped to
zero, a neighbouring column's bias, a dropped K chunk, the residual on the wrong side of the ReLU, a tile row reading the
previous image, a store past Cout and a shifted output slice. The normalisation and sampler references (GroupNorm,
LayerNorm, the token embedding's row statistics, CFG + DDIM, the timestep embedding) are pinned to F.group_norm on
pad_pano, F.layer_norm, the oracle's DDIM step and Timesteps, then shown to catch a dropped pixel, a one-sided seam
weight, a count over the unpadded width, the next group's or another image's statistics, a block-indexed PE, a skipped
token, a reversed roll, swapped CFG halves, swapped sin / cos halves and statistics of the unrounded row. The conv_in,
VAE softmax, latent sampling and MSE references are pinned to F.conv2d (on pad_pano for the circular case),
torch.softmax, the DiagonalGaussianDistribution.sample formula and F.mse_loss, then shown to catch a seam wrapped to
zero, a tap reading the previous image, a missing bias, SiLU before the bias, the decoder fold's ones channel padded
with ones, logits scaled before the maximum is subtracted, a dropped last odd column, a clamp at 30, swapped mean and
logvar, an NHWC output and a mean over the padded element count."""
import pytest
import torch

import _contract as ct
from panfusion_b200.packing import pack_conv3x3, pack_geglu

DTYPES = [torch.float16, torch.bfloat16]


def _kernel_like(ref, dtype):
    """What a correct kernel stores: the exact value rounded once to the output type (NaN stays NaN)."""
    return ref.to(dtype).double() if dtype != torch.float32 else ref.float().double()


def _caught(exact, mutated, dtype):
    ref, bound = exact
    ok = ct.worst_ratio(_kernel_like(ref, dtype), ref, bound)
    bad = ct.worst_ratio(_kernel_like(mutated, dtype), ref, bound)
    assert ok <= 1.0, ok
    assert bad > 1.0, bad


def _conv_setup(dtype, N=2, H=5, W=6, C=16, Co=24, seed=0):
    """A 3x3 / pad 1 convolution in the padded-flat layout the engine uses (zero halo of one pixel)."""
    g = torch.Generator().manual_seed(seed)
    Hp, Wp = H + 2, W + 2
    x = torch.zeros(N, Hp, Wp, C)
    x[:, 1:-1, 1:-1] = torch.randn(N, H, W, C, generator=g)
    A = x.reshape(N * Hp * Wp, C).to(dtype)
    w = torch.randn(Co, C, 3, 3, generator=g) / (9 * C) ** 0.5
    B = pack_conv3x3(w).to(dtype)
    taps = [(dy - 1) * Wp + (dx - 1) for dy in range(3) for dx in range(3)]
    kw = dict(M=N * Hp * Wp, Kc=C, taps=taps, bias=torch.randn(Co, generator=g), image_map=(Hp, Wp, 1, 1, H, W))
    return g, A, B, kw, N * H * W


@pytest.mark.parametrize("dtype", DTYPES)
def test_dropped_tap_is_caught(dtype):
    g, A, B, kw, rows = _conv_setup(dtype)
    exact = ct.tap_gemm_ref(A, B, rows, dtype, **kw)
    C = kw["Kc"]
    keep = [t for t in range(9) if t != 5]
    Bd = torch.cat([B[:, t * C:(t + 1) * C] for t in keep], 1)
    mutated, _ = ct.tap_gemm_ref(A, Bd, rows, dtype, **dict(kw, taps=[kw["taps"][t] for t in keep]))
    _caught(exact, mutated, dtype)


@pytest.mark.parametrize("dtype", DTYPES)
def test_shifted_rowbias_group_is_caught(dtype):
    g, A, B, kw, rows = _conv_setup(dtype)
    temb = torch.randn(2, B.shape[0], generator=g)
    exact = ct.tap_gemm_ref(A, B, rows, dtype, rowbias=temb, **kw)
    mutated, _ = ct.tap_gemm_ref(A, B, rows, dtype, rowbias=temb.roll(1, 0), **kw)
    _caught(exact, mutated, dtype)


@pytest.mark.parametrize("dtype", DTYPES)
def test_halo_row_in_the_output_is_caught(dtype):
    g, A, B, kw, rows = _conv_setup(dtype)
    exact = ct.tap_gemm_ref(A, B, rows, dtype, **kw)
    Hp, Wp, i0, j0, H, W = kw["image_map"]
    shifted, _ = ct.tap_gemm_ref(A, B, rows, dtype, **dict(kw, image_map=(Hp, Wp, i0, j0 - 1, H, W)))
    mutated = exact[0].clone()
    mutated[0] = shifted[0]  # output pixel (0, 0) of image 0 takes the M-row of the halo pixel to its left
    _caught(exact, mutated, dtype)


@pytest.mark.parametrize("dtype", DTYPES)
def test_residual_one_row_off_is_caught(dtype):
    g, A, B, kw, rows = _conv_setup(dtype)
    res = torch.randn(rows, B.shape[0], generator=g).to(dtype)
    exact = ct.tap_gemm_ref(A, B, rows, dtype, residual=res, **kw)
    mutated, _ = ct.tap_gemm_ref(A, B, rows, dtype, residual=res.roll(1, 0), **kw)
    _caught(exact, mutated, dtype)


@pytest.mark.parametrize("dtype", DTYPES)
def test_swapped_geglu_halves_are_caught(dtype):
    g = torch.Generator().manual_seed(1)
    M, K, inner, bn = 40, 64, 128, 64
    A = torch.randn(M, K, generator=g).to(dtype)
    W = torch.randn(2 * inner, K, generator=g) / K ** 0.5
    b = torch.randn(2 * inner, generator=g)
    Wp, bp = pack_geglu(W, b, bn)
    exact = ct.tap_gemm_ref(A, Wp.to(dtype), M, dtype, M=M, Kc=K, bias=bp, act=ct.ACT_GEGLU, geglu_bn=bn)
    sw = lambda t: torch.cat([t[inner:], t[:inner]])
    Ws, bs = pack_geglu(sw(W), sw(b), bn)
    mutated, _ = ct.tap_gemm_ref(A, Ws.to(dtype), M, dtype, M=M, Kc=K, bias=bs, act=ct.ACT_GEGLU, geglu_bn=bn)
    _caught(exact, mutated, dtype)


def _attention(dtype, B, Lq, Lk, heads=2, d=32, seed=2):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(B, Lq, heads * d, generator=g).to(dtype)
    k = torch.randn(B, Lk + 1, heads * d, generator=g).to(dtype)  # one row past Lk: what an unmasked key would read
    v = torch.randn(B, Lk + 1, heads * d, generator=g).to(dtype)
    return g, q, k, v


@pytest.mark.parametrize("dtype", DTYPES)
def test_unmasked_ragged_key_is_caught(dtype):
    g, q, k, v = _attention(dtype, 1, 7, 5)
    ref, pv = ct.fmha_ref(q, k[:, :5], v[:, :5], heads=2, head_dim=32, scale=32 ** -0.5)
    mutated, _ = ct.fmha_ref(q, k, v, heads=2, head_dim=32, scale=32 ** -0.5)
    _caught((ref, ct.fmha_bound(ref, pv, dtype)), mutated, dtype)


@pytest.mark.parametrize("dtype", DTYPES)
def test_bias_of_the_wrong_batch_is_caught(dtype):
    g, q, k, v = _attention(dtype, 2, 9, 6)
    k, v = k[:, :6], v[:, :6]
    bias = torch.rand(2, 9, 6, generator=g) * 2 - 1
    ref, pv = ct.fmha_ref(q, k, v, heads=2, head_dim=32, scale=32 ** -0.5, bias=bias)
    mutated, _ = ct.fmha_ref(q, k, v, heads=2, head_dim=32, scale=32 ** -0.5, bias=bias[[1, 0]])
    _caught((ref, ct.fmha_bound(ref, pv, dtype)), mutated, dtype)


def test_rows_outside_the_contract_must_stay_untouched():
    """A kernel that writes a row the contract leaves alone fails even when every due value is right."""
    ref = torch.tensor([[1.0], [float("nan")]], dtype=torch.float64)
    bound = torch.tensor([[1e-3], [float("nan")]], dtype=torch.float64)
    assert ct.worst_ratio(torch.tensor([[1.0], [float("nan")]]), ref, bound) == 0.0
    with pytest.raises(AssertionError):
        ct.worst_ratio(torch.tensor([[1.0], [0.0]]), ref, bound)
    assert ct.worst_ratio(torch.tensor([[float("nan")], [float("nan")]]), ref, bound) == float("inf")


# ---- implicit-GEMM convolution (conv_mma.cuh) -----------------------------------------------------------------------

def _conv_operands(seed, B=2, H=5, W=6, cin=32, cin_pad=32, cout=6, cw=32, k=3, res=False, offset=0.0):
    """fp16 channels-last input (channels past cin zero), the packed fp16 weight [k*k][cin_pad][cw] (zero past cin and
    cout), an fp32 bias over cw columns and an optional fp16 residual for the stride-1 'same' output."""
    g = torch.Generator().manual_seed(seed)
    x = torch.zeros(B, H, W, cin_pad)
    x[..., :cin] = torch.randn(B, H, W, cin, generator=g) + offset
    w = torch.randn(cout, cin, k, k, generator=g, dtype=torch.float64) / (cin * k * k) ** 0.5
    wp = torch.zeros(k * k, cin_pad, cw, dtype=torch.float64)
    wp[:, :cin, :cout] = w.permute(2, 3, 1, 0).reshape(k * k, cin, cout)
    bias = torch.randn(cw, generator=g) * 0.5
    r = torch.randn(B * H * W, cout, generator=g).half() if res else None
    return x.half(), wp.half(), bias, r


def _conv_kw(cout, k, s=1, circ=False, relu=False, dtype=torch.float16, **kw):
    return dict(Cout=cout, kh=k, kw=k, stride_h=s, stride_w=s, ph=k // 2, pw=k // 2, circ=circ, relu=relu,
                out_dtype=dtype, **kw)


def _caught_or_stray(exact, mutated, dtype):
    """Like _caught, but a mutation that writes outside the contract's elements counts as caught too."""
    ref, bound = exact
    assert ct.worst_ratio(_kernel_like(ref, dtype), ref, bound) <= 1.0
    try:
        bad = ct.worst_ratio(_kernel_like(mutated, dtype), ref, bound)
    except AssertionError:
        return
    assert bad > 1.0, bad


@pytest.mark.parametrize("k,s,ph,pw", [(3, 1, 1, 1), (1, 2, 0, 0), (4, 2, 1, 1), (7, 2, 3, 3), (1, 1, 0, 0),
                                       (3, 2, 0, 0), (5, 1, 2, 2)])
@pytest.mark.parametrize("circ", [False, True])
def test_conv_ref_matches_torch(k, s, ph, pw, circ):
    """conv_ref against F.conv2d with explicit zero padding, or oracle.faed.circular_pad (rows zero, columns wrapped)."""
    import torch.nn.functional as F
    from oracle import faed as of
    x, wp, bias, _ = _conv_operands(3 + k, B=2, H=9, W=8, cin=24, cout=10, k=k)
    ref, bound = ct.conv_ref(x, wp, bias, Cout=10, kh=k, kw=k, stride_h=s, stride_w=s, ph=ph, pw=pw, circ=circ,
                             relu=False, out_dtype=torch.float32)
    w = wp.double()[:, :, :10].reshape(k, k, 32, 10).permute(3, 2, 0, 1)
    xd = x.double().permute(0, 3, 1, 2)
    y = F.conv2d(of.circular_pad(xd, ph) if circ else F.pad(xd, (pw, pw, ph, ph)), w, bias[:10].double(), stride=s)
    assert torch.allclose(ref, y.permute(0, 2, 3, 1).reshape(-1, 10), rtol=1e-12, atol=1e-12)
    assert (bound > 0).all()


def test_conv_ref_stride_2_1_and_asymmetric_phase_pads():
    """HorizonNet's (2, 1) stride, and a stride-2 data-gradient phase (2x2 kernel, pads (1 - r, 1 - c), Ho = H,
    Wo = W given): both against F.conv2d on an explicitly padded input."""
    import torch.nn.functional as F
    from oracle import horizonnet as oh
    x, wp, bias, _ = _conv_operands(11, H=8, W=6, cin=16, cin_pad=16, cout=8, k=3)
    ref, _ = ct.conv_ref(x, wp, bias, Cout=8, kh=3, kw=3, stride_h=2, stride_w=1, ph=1, pw=1, circ=True, relu=False,
                         out_dtype=torch.float32)
    w = wp.double()[:, :, :8].reshape(3, 3, 16, 8).permute(3, 2, 0, 1)
    y = oh.conv(x.double().permute(0, 3, 1, 2), w, bias[:8].double(), 3, (2, 1))
    assert torch.allclose(ref, y.permute(0, 2, 3, 1).reshape(-1, 8), rtol=1e-12, atol=1e-12)
    x, wp, bias, _ = _conv_operands(12, H=4, W=5, cin=16, cin_pad=16, cout=8, k=2)
    w = wp.double()[:, :, :8].reshape(2, 2, 16, 8).permute(3, 2, 0, 1)
    xd = x.double().permute(0, 3, 1, 2)
    for r in (0, 1):
        for c in (0, 1):
            ref, _ = ct.conv_ref(x, wp, bias, Cout=8, kh=2, kw=2, stride_h=1, stride_w=1, ph=1 - r, pw=1 - c, circ=True,
                                 relu=False, out_dtype=torch.float32, Ho=4, Wo=5)
            xp = F.pad(torch.cat([xd[..., 5 - (1 - c):], xd, xd[..., :c]], -1), (0, 0, 1 - r, r))
            y = F.conv2d(xp, w, bias[:8].double())
            assert y.shape[-2:] == (4, 5)
            assert torch.allclose(ref, y.permute(0, 2, 3, 1).reshape(-1, 8), rtol=1e-12, atol=1e-12), (r, c)


def test_conv_ref_leaves_rows_past_m_and_columns_outside_the_slice_nan():
    x, wp, bias, _ = _conv_operands(4, cout=6)
    ref, bound = ct.conv_ref(x, wp, bias, **_conv_kw(6, 3, out_rows=70, out_ld=12, out_off=4))
    M = 2 * 5 * 6
    assert torch.isnan(ref[M:]).all() and torch.isnan(ref[:, :4]).all() and torch.isnan(ref[:, 10:]).all()
    assert not torch.isnan(ref[:M, 4:10]).any() and torch.equal(torch.isnan(ref), torch.isnan(bound))


CONV_DTYPES = [torch.float16, torch.float32]


@pytest.mark.parametrize("dtype", CONV_DTYPES)
def test_conv_seam_wrapped_to_zero_is_caught(dtype):
    x, wp, bias, _ = _conv_operands(5, W=7, k=3, offset=0.5)
    exact = ct.conv_ref(x, wp, bias, **_conv_kw(6, 3, circ=True, dtype=dtype))
    mutated, _ = ct.conv_ref(x, wp, bias, **_conv_kw(6, 3, circ=False, dtype=dtype))
    _caught(exact, mutated, dtype)


@pytest.mark.parametrize("dtype", CONV_DTYPES)
def test_conv_bias_of_the_neighbouring_column_is_caught(dtype):
    x, wp, bias, _ = _conv_operands(6)
    exact = ct.conv_ref(x, wp, bias, **_conv_kw(6, 3, relu=True, dtype=dtype))
    b2 = bias.clone()
    b2[1::2] = bias[0::2]  # the epilogue's column pair (c, c + 1) both take bias[c]
    mutated, _ = ct.conv_ref(x, wp, b2, **_conv_kw(6, 3, relu=True, dtype=dtype))
    _caught(exact, mutated, dtype)


@pytest.mark.parametrize("dtype", CONV_DTYPES)
def test_conv_dropped_last_k_chunk_of_a_tap_is_caught(dtype):
    """Cin = 32 in two 16-channel k-steps per tap: the second chunk of tap 8 (the last k-step) is lost."""
    x, wp, bias, _ = _conv_operands(7, cin=32, cin_pad=32)
    exact = ct.conv_ref(x, wp, bias, **_conv_kw(6, 3, dtype=dtype))
    w2 = wp.clone()
    w2[8, 16:] = 0
    mutated, _ = ct.conv_ref(x, w2, bias, **_conv_kw(6, 3, dtype=dtype))
    _caught(exact, mutated, dtype)


@pytest.mark.parametrize("dtype", CONV_DTYPES)
def test_conv_residual_after_the_relu_is_caught(dtype):
    x, wp, bias, res = _conv_operands(8, res=True)
    exact = ct.conv_ref(x, wp, bias, **_conv_kw(6, 3, circ=True, relu=True, dtype=dtype, residual=res,
                                                res_before_relu=True))
    mutated, _ = ct.conv_ref(x, wp, bias, **_conv_kw(6, 3, circ=True, relu=True, dtype=dtype, residual=res))
    _caught(exact, mutated, dtype)


@pytest.mark.parametrize("dtype", CONV_DTYPES)
def test_conv_tile_row_reading_the_previous_image_is_caught(dtype):
    """The first output row of image 1 takes image 0's last input row for its top tap instead of zero padding: the
    same convolution over the images stacked along H."""
    x, wp, bias, _ = _conv_operands(9, B=3, H=4, W=6)
    exact = ct.conv_ref(x, wp, bias, **_conv_kw(6, 3, circ=True, dtype=dtype))
    mutated, _ = ct.conv_ref(x.reshape(1, 12, 6, 32), wp, bias, **_conv_kw(6, 3, circ=True, dtype=dtype))
    assert torch.equal(mutated[:18], exact[0][:18])  # image 0's first three output rows are unchanged
    _caught(exact, mutated, dtype)


@pytest.mark.parametrize("dtype", CONV_DTYPES)
def test_conv_column_past_cout_is_caught(dtype):
    """FAED's last layer: Cout = 4 of a 32-wide packed weight; a store of column 4 (the next pair) fails."""
    x, wp, bias, _ = _conv_operands(10, cout=3, cw=32, k=9, W=10)
    exact = ct.conv_ref(x, wp, bias, **_conv_kw(4, 9, circ=True, dtype=dtype, out_ld=8))
    assert torch.equal(exact[0][:, 3], bias[3].double().expand(exact[0].shape[0]))  # the zero weight column: bias only
    mutated = exact[0].clone()
    mutated[:, 4] = bias[4].double()
    _caught_or_stray(exact, mutated, dtype)
    with pytest.raises(AssertionError):
        ct.worst_ratio(_kernel_like(mutated, dtype), *exact)


@pytest.mark.parametrize("dtype", CONV_DTYPES)
def test_conv_output_slice_shifted_by_two_columns_is_caught(dtype):
    """An Inception branch written at out_off + 2 of its concat buffer."""
    x, wp, bias, _ = _conv_operands(11, cout=10, cw=32)
    exact = ct.conv_ref(x, wp, bias, **_conv_kw(10, 3, relu=True, dtype=dtype, out_ld=24, out_off=6))
    mutated = torch.full_like(exact[0], float("nan"))
    mutated[:, 8:18] = exact[0][:, 6:16]
    _caught_or_stray(exact, mutated, dtype)


@pytest.mark.parametrize("dtype", DTYPES)
def test_causal_mask_shifted_by_one_key_is_caught(dtype):
    """The text tower's causal bias (finfo(float32).min above the diagonal): one row that also sees the next key."""
    g, q, k, v = _attention(dtype, 2, 9, 9, heads=2, d=64)
    k, v = k[:, :9], v[:, :9]
    causal = torch.full((9, 9), torch.finfo(torch.float32).min).triu(1)
    ref, pv = ct.fmha_ref(q, k, v, heads=2, head_dim=64, scale=64 ** -0.5, bias=causal)
    shifted = causal.clone()
    shifted[4, 5] = 0.0
    mutated, _ = ct.fmha_ref(q, k, v, heads=2, head_dim=64, scale=64 ** -0.5, bias=shifted)
    _caught((ref, ct.fmha_bound(ref, pv, dtype)), mutated, dtype)


# ---- correspondence-aware attention (cpattn.cu) ---------------------------------------------------------------------

def _cp_rigs(B, m, img, G):
    """K, R [B, m, 3, 3] of horizon rigs (FoV 120, so neighbouring views overlap): every element the same rig, or
    (G = B) element b turned by 20 b degrees."""
    import numpy as np
    from oracle import mvdiffusion as omv
    if G == 1:
        return omv.horizon_cameras(m, batch=B, fov=120.0, size=img)
    theta = np.rad2deg(np.linspace(0, 2 * np.pi, m, endpoint=False))
    KR = [[omv.get_K_R(120.0, t + 20.0 * b, 0.0, img) for t in theta] for b in range(B)]
    K = torch.stack([torch.from_numpy(np.stack([k for k, _ in row])) for row in KR])
    R = torch.stack([torch.from_numpy(np.stack([r for _, r in row])) for row in KR])
    return K, R


def _cp_gather_setup(dtype, G=1, B=2, m=3, h=5, C=32, img=40, seed=12):
    """Tokens [B * m * h * h, C] in the 16-bit type, the oracle's tables in pf_cpattn_tables' layout (pos | xy_rel) and
    MVDiffusion's frequency table."""
    from oracle import mvdiffusion as omv
    from panfusion_b200.mvdiffusion import _PosEmbedding
    K, R = _cp_rigs(B, m, img, G)
    pos, mask, rel = omv.tables(K, R, h, img)
    table = torch.cat([pos, rel], -1).float()[:G].contiguous()
    x = torch.randn(B * m * h * h, C, generator=torch.Generator().manual_seed(seed)).to(dtype)
    freq = _PosEmbedding(C // 4).freq_bands.reshape(-1).float()
    return dict(x=x, B=B, m=m, h=h, w=h, C=C, G=G, pos=table, mask=mask[:G].to(torch.uint8), freq=freq), (pos, mask, rel)


def test_cpattn_gather_ref_matches_the_oracle():
    """cpattn_gather_ref equals oracle.mvdiffusion.gather_keys (F.grid_sample of the normalised grid + PosEmbedding,
    times the mask) on the oracle's own tables, per batch element with its own cameras."""
    from oracle import mvdiffusion as omv
    kw, (pos, mask, rel) = _cp_gather_setup(torch.float16, G=2)
    ref, bound = ct.cpattn_gather_ref(**kw, out_dtype=torch.float16)
    B, m, h, C = kw["B"], kw["m"], kw["h"], kw["C"]
    x5 = kw["x"].float().reshape(B, m, h, h, C).permute(0, 1, 4, 2, 3)
    want = omv.gather_keys(x5, pos, mask, rel, kw["freq"]).reshape(-1, C)
    assert mask.any() and not mask.all()
    assert torch.allclose(ref, want.double(), rtol=0, atol=2e-5), (ref - want).abs().max()
    assert (ref[~mask.reshape(-1)] == 0).all() and (bound > 0).all()


def _gather_caught(kw, mutated, dtype):
    ref, bound = ct.cpattn_gather_ref(**kw, out_dtype=dtype)
    _caught((ref, bound), mutated, dtype)


@pytest.mark.parametrize("dtype", DTYPES)
def test_cpattn_swapped_neighbours_are_caught(dtype):
    kw, _ = _cp_gather_setup(dtype)
    _gather_caught(kw, ct.cpattn_gather_ref(**kw, out_dtype=dtype, neighbours=(1, -1))[0], dtype)


@pytest.mark.parametrize("dtype", DTYPES)
def test_cpattn_swapped_bilinear_weights_are_caught(dtype):
    """The x fraction weighting the y taps and vice versa: the same taps at (floor x + frac y, floor y + frac x)."""
    kw, _ = _cp_gather_setup(dtype)
    p = kw["pos"].clone()
    fx, fy = p[..., 0].floor(), p[..., 1].floor()
    p[..., 0], p[..., 1] = fx + (kw["pos"][..., 1] - fy), fy + (kw["pos"][..., 0] - fx)
    _gather_caught(kw, ct.cpattn_gather_ref(**dict(kw, pos=p), out_dtype=dtype)[0], dtype)


@pytest.mark.parametrize("dtype", DTYPES)
def test_cpattn_swapped_pe_halves_are_caught(dtype):
    kw, _ = _cp_gather_setup(dtype)
    ref, _ = ct.cpattn_gather_ref(**kw, out_dtype=dtype)
    N = kw["C"] // 4
    arg = (kw["pos"][..., 2:, None] * kw["freq"]).double()            # [G, m, P, 18, 2, N]
    sin, cos = arg.sin().flatten(-2), arg.cos().flatten(-2)
    live = kw["mask"].bool().expand(kw["B"], -1, -1, -1).reshape(-1)
    d = (torch.cat([cos - sin, sin - cos], -1)).expand(kw["B"], -1, -1, -1, -1).reshape(-1, 4 * N)
    mutated = ref.clone()
    mutated[live] += d[live]
    _caught(ct.cpattn_gather_ref(**kw, out_dtype=dtype), mutated, dtype)


@pytest.mark.parametrize("dtype", DTYPES)
def test_cpattn_unmasked_key_is_caught(dtype):
    kw, _ = _cp_gather_setup(dtype)
    ones = torch.ones_like(kw["mask"])
    _gather_caught(kw, ct.cpattn_gather_ref(**dict(kw, mask=ones), out_dtype=dtype)[0], dtype)


@pytest.mark.parametrize("dtype", DTYPES)
def test_cpattn_per_batch_tables_read_with_g0_are_caught(dtype):
    kw, _ = _cp_gather_setup(dtype, G=2)
    shared = dict(kw, G=1, pos=kw["pos"][:1], mask=kw["mask"][:1])
    _gather_caught(kw, ct.cpattn_gather_ref(**shared, out_dtype=dtype)[0], dtype)


def test_cpattn_stats_bound_accepts_fp32_sums_of_the_stored_keys():
    kw, _ = _cp_gather_setup(torch.bfloat16, C=64)
    ref, _ = ct.cpattn_gather_ref(**kw, out_dtype=torch.bfloat16)
    keys = ref.to(torch.bfloat16)
    k32 = keys.float()
    got = torch.stack([k32.sum(1), (k32 * k32).sum(1)], 1).double()
    want, bound = ct.cpattn_stats_ref(keys, 64)
    assert ((got - want).abs() <= bound).all()
    unrounded = torch.stack([ref.sum(1), (ref * ref).sum(1)], 1)      # statistics of the values before the store
    assert ((unrounded - want).abs() > bound).any()


def _cp_attn_setup(dtype, T=37, C=96, seed=13):
    g = torch.Generator().manual_seed(seed)
    q = (torch.randn(T, C, generator=g) * 2).to(dtype)
    kv = torch.randn(T * 18, 2 * C, generator=g).to(dtype)
    return q, kv


def test_cpattn_attn_ref_matches_softmax_attention():
    """cpattn_attn_ref equals the reference's attention (oracle.eppa's softmax(q k^T * scale) v per head) over the
    18 keys of each query; below the output rounding its bound is at least four times tighter than fmha_bound."""
    q, kv = _cp_attn_setup(torch.float16)
    T, C = q.shape
    ref, bound = ct.cpattn_attn_ref(q, kv, C, 32 ** -0.5, torch.float16)
    sc = float(torch.tensor(32 ** -0.5, dtype=torch.float32))  # the kernel's float argument
    qh = q.double().reshape(T, 1, C // 32, 32).transpose(1, 2)
    k = kv[:, :C].double().reshape(T, 18, C // 32, 32).transpose(1, 2)
    v = kv[:, C:].double().reshape(T, 18, C // 32, 32).transpose(1, 2)
    want = (torch.softmax(qh @ k.transpose(-1, -2) * sc, -1) @ v).transpose(1, 2).reshape(T, C)
    assert torch.allclose(ref, want, rtol=1e-12, atol=1e-12)
    pv = (torch.softmax(qh @ k.transpose(-1, -2) * sc, -1) @ v.abs()).transpose(1, 2).reshape(T, C)
    loose = ct.fmha_bound(ref, pv, torch.float16)
    assert (bound - ct.ulp_out(ref, torch.float16) < loose / 4).all()


@pytest.mark.parametrize("dtype", DTYPES)
def test_cpattn_dropped_key_slot_is_caught(dtype):
    """The softmax over 17 of the 18 slots (the last one never read)."""
    q, kv = _cp_attn_setup(dtype)
    T, C = q.shape
    exact = ct.cpattn_attn_ref(q, kv, C, 32 ** -0.5, dtype)
    qh = q.double().reshape(T, 1, C // 32, 32).transpose(1, 2)
    k = kv[:, :C].double().reshape(T, 18, C // 32, 32).transpose(1, 2)[:, :, :17]
    v = kv[:, C:].double().reshape(T, 18, C // 32, 32).transpose(1, 2)[:, :, :17]
    mutated = (torch.softmax(qh @ k.transpose(-1, -2) * 32 ** -0.5, -1) @ v).transpose(1, 2).reshape(T, C)
    _caught(exact, mutated, dtype)


@pytest.mark.parametrize("dtype", DTYPES)
def test_cpattn_head_reading_the_next_heads_v_is_caught(dtype):
    q, kv = _cp_attn_setup(dtype)
    C = q.shape[1]
    exact = ct.cpattn_attn_ref(q, kv, C, 32 ** -0.5, dtype)
    kv2 = kv.clone()
    kv2[:, C:] = kv[:, C:].roll(-32, 1)  # head h's V columns hold head h + 1's
    _caught(exact, ct.cpattn_attn_ref(q, kv2, C, 32 ** -0.5, dtype)[0], dtype)


# ---- normalisation and sampler kernels (norm.cu, elementwise.cu) ---------------------------------------------------

def _nchw(x, N, H, W):
    return x.double().reshape(N, H, W, -1).permute(0, 3, 1, 2)


def _gn_setup(dtype, N=2, H=4, W=12, C=64, groups=32, seed=20):
    g = torch.Generator().manual_seed(seed)
    x = ct.gn_operand(g, N, H, W, C, groups, dtype)
    return x, torch.randn(C, generator=g), torch.randn(C, generator=g)


@pytest.mark.parametrize("circ_stats,circ,phases,up,halo,act", [
    (2, 2, 1, 1, 1, ct.ACT_SILU),   # panorama norm1: pad_pano(2) statistics and layout
    (0, 1, 1, 1, 1, ct.ACT_SILU),   # conv_out: statistics of the unpadded tensor, pad_pano(1) layout
    (0, 0, 1, 1, 0, ct.ACT_NONE),   # the transformer's plain GroupNorm
    (2, 2, 4, 1, 1, ct.ACT_SILU),   # stride-2 phases
    (1, 1, 1, 2, 1, ct.ACT_SILU),   # nearest x2
])
def test_gn_refs_match_torch_group_norm(circ_stats, circ, phases, up, halo, act):
    """gn_stats_ref and gn_apply_ref equal F.group_norm of pad_pano(x, circ_stats) applied to pad_pano(x, circ), then
    SiLU, nearest x2, the zero halo and the stride-2 phase split (the composition of the reference's modules)."""
    import torch.nn.functional as F
    from oracle.eppa import pad_pano
    N, H, W, C, G = 2, 4, 12, 64, 32
    x, gamma, beta = _gn_setup(torch.float16, N, H, W, C, G)
    xs = pad_pano(_nchw(x, N, H, W), circ_stats)
    mean = xs.reshape(N, G, -1).mean(-1)
    rstd = (xs.reshape(N, G, -1).var(-1, unbiased=False) + ct._f32(1e-5)).rsqrt()
    stats, sb = ct.gn_stats_ref(x, N, H, W, G, circ_stats, 1e-5, ct.gn_partition("pf_gn_prep", H, W, C))
    assert torch.allclose(stats[..., 0], mean, rtol=1e-12, atol=1e-12)
    assert torch.allclose(stats[..., 1], rstd, rtol=1e-12, atol=1e-12)
    assert (sb > 0).all()
    full = F.group_norm(pad_pano(_nchw(x, N, H, W), circ), G, gamma.double(), beta.double(), 1e-5)
    if circ_stats != circ:  # the statistics come from the other width: apply them by hand
        cpg = C // G
        full = ((pad_pano(_nchw(x, N, H, W), circ) - mean.repeat_interleave(cpg, 1)[..., None, None])
                * rstd.repeat_interleave(cpg, 1)[..., None, None] * gamma.double()[:, None, None] + beta.double()[:, None, None])
    if act == ct.ACT_SILU:
        full = F.silu(full)
    if up == 2:
        full = F.interpolate(full, scale_factor=2.0, mode="nearest")
    full = F.pad(full, [1, 1, 1, 1]) if (halo or phases == 4) else full
    if phases == 4:
        want = torch.stack([full[:, :, py::2, px::2] for py in (0, 1) for px in (0, 1)]).permute(0, 1, 3, 4, 2)
    else:
        want = full.permute(0, 2, 3, 1)
    ref, bound = ct.gn_apply_ref(x, N, H, W, stats.float(), gamma, beta, act=act, circ=circ, up=up, phases=phases,
                                 halo=halo, out_dtype=torch.float16)
    # the reference applies fp64 statistics, the contract the fp32 ones the launch reads
    assert torch.allclose(ref, want.reshape(ref.shape), rtol=1e-6, atol=1e-6)
    pad = (want.reshape(ref.shape) == 0).all(1)
    assert pad.any() == bool(halo or phases == 4) and (bound[pad] == ct.EXACT).all() and (ref[pad] == 0).all()


def _stats(x, N, H, W, G, weights, count, eps=1e-5):
    """fp64 (mean, rstd) of x with per-column weights and an explicit count: the emulated statistics bugs."""
    cpg = x.shape[1] // G
    xb = x.double().reshape(N, H, W, G, cpg)
    w = weights.double()[None, None, :, None, None]
    mean = (w * xb).sum((1, 2, 4)) / count
    var = (w * xb * xb).sum((1, 2, 4)) / count - mean * mean
    return torch.stack([mean, 1.0 / torch.sqrt(var + ct._f32(eps))], -1)


def _seam_weights(W, circ, left=True, right=True):
    col = torch.arange(W)
    return 1.0 + left * (col < circ).double() + right * (col >= W - circ).double()


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("bug", ["dropped pixel", "one-sided seam", "unpadded count"])
def test_gn_stats_bugs_are_caught(dtype, bug):
    """One pixel of a slab never added; the duplicated seam columns weighted on the left side only; the count taken
    over the unpadded width. Shapes as the UNet's panorama norm1 at a small level (pad_pano(2) statistics)."""
    N, H, W, C, G, circ = 2, 8, 16, 128, 32, 2
    x, _, _ = _gn_setup(dtype, N, H, W, C, G, seed=21)
    exact = ct.gn_stats_ref(x, N, H, W, G, circ, 1e-5, ct.gn_partition("pf_gn_prep", H, W, C))
    count = H * (W + 2 * circ) * (C // G)
    if bug == "dropped pixel":
        xd = x.clone()
        xd[(H * W) // 2 + 3] = 0  # a pixel inside a slab of image 0
        mutated = _stats(xd, N, H, W, G, _seam_weights(W, circ), count)
    elif bug == "one-sided seam":
        mutated = _stats(x, N, H, W, G, _seam_weights(W, circ, right=False), count)
    else:
        mutated = _stats(x, N, H, W, G, _seam_weights(W, circ), H * W * (C // G))
    assert torch.allclose(_stats(x, N, H, W, G, _seam_weights(W, circ), count), exact[0], rtol=1e-9, atol=1e-9)
    _caught(exact, mutated, torch.float32)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("bug", ["next group", "other image"])
def test_gn_apply_bugs_are_caught(dtype, bug):
    """A group-edge channel normalised with the next group's statistics; an image normalised with another's."""
    N, H, W, C, G = 2, 4, 8, 128, 32
    x, gamma, beta = _gn_setup(dtype, N, H, W, C, G, seed=22)
    st = ct.gn_stats_ref(x, N, H, W, G, 0, 1e-5, ct.gn_partition("pf_gn_prep", H, W, C))[0].float()
    kw = dict(act=ct.ACT_SILU, circ=0, up=1, phases=1, halo=1, out_dtype=dtype)
    exact = ct.gn_apply_ref(x, N, H, W, st, gamma, beta, **kw)
    if bug == "next group":
        mutated = exact[0].clone()
        edge = C // G - 1  # the last channel of group 0
        mutated[:, edge] = ct.gn_apply_ref(x, N, H, W, st.roll(-1, 1), gamma, beta, **kw)[0][:, edge]
    else:
        mutated = ct.gn_apply_ref(x, N, H, W, st.roll(1, 0), gamma, beta, **kw)[0]
    _caught(exact, mutated, dtype)


def _ln_setup(dtype, T=64, C=320, pe_rows=16, seed=23):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(T, C, generator=g) * 2 + 0.5).to(dtype)
    pe = torch.randn(pe_rows, C, generator=g)
    return x, pe, torch.randn(C, generator=g), torch.randn(C, generator=g)


def test_layernorm_ref_matches_torch_layer_norm():
    import torch.nn.functional as F
    x, pe, gamma, beta = _ln_setup(torch.bfloat16)
    ref, bound = ct.layernorm_ref(x, pe, gamma, beta, 1e-5, torch.bfloat16)
    f = (x.float() + pe.repeat(x.shape[0] // pe.shape[0], 1)).double()
    want = F.layer_norm(f, (x.shape[1],), gamma.double(), beta.double(), ct._f32(1e-5))
    assert torch.allclose(ref, want, rtol=1e-12, atol=1e-12) and (bound > 0).all()
    ref0, _ = ct.layernorm_ref(x[::2], None, gamma, beta, 1e-5, torch.bfloat16)  # a strided view, no PE
    assert torch.allclose(ref0, F.layer_norm(x[::2].double(), (x.shape[1],), gamma.double(), beta.double(), ct._f32(1e-5)))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("bug", ["pe by block", "skipped token"])
def test_layernorm_bugs_are_caught(dtype, bug):
    """pe[t // (T / pe_rows)] instead of pe[t % pe_rows]; the second token of a warp never written (NaN-filled)."""
    x, pe, gamma, beta = _ln_setup(dtype)
    exact = ct.layernorm_ref(x, pe, gamma, beta, 1e-5, dtype)
    T, rows = x.shape[0], pe.shape[0]
    if bug == "pe by block":
        mutated, _ = ct.layernorm_ref(x, pe[torch.arange(T) // (T // rows)], gamma, beta, 1e-5, dtype)
    else:
        mutated = exact[0].clone()
        mutated[1] = float("nan")
    _caught(exact, mutated, dtype)


def _embed_setup(T=154, L=77, C=192, vocab=50, seed=24):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(vocab, C, generator=g) * 0.5 + 0.1, torch.randn(L, C, generator=g) * 0.3,
            torch.randint(0, vocab, (T,), generator=g), L)


@pytest.mark.parametrize("dtype", DTYPES)
def test_row_stats_of_the_fp32_row_are_caught(dtype):
    """The statistics must be those of the stored 16-bit row: fp32 sums of it pass, the unrounded row's fail."""
    tok, pos, ids, L = _embed_setup()
    row, ref, bound = ct.row_stats_ref(tok, pos, ids, L, dtype)
    assert torch.equal(row, (tok[ids] + pos.repeat(2, 1)).to(dtype))
    r32 = row.float()
    got = torch.stack([r32.sum(1), (r32 * r32).sum(1)], 1).double()
    assert ((got - ref).abs() <= bound).all()
    f = (tok[ids] + pos.repeat(2, 1)).double()
    assert ((torch.stack([f.sum(1), (f * f).sum(1)], 1) - ref).abs() > bound).any()


def _ddim_setup(seed=25, W=32):
    from panfusion_b200.sampler import DDIMSchedule
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(2, 4, 16, W, generator=g)
    eps = torch.randn(2, 2, 4, 16, W, generator=g)
    sched = DDIMSchedule()
    sched.set_timesteps(50)
    t = int(sched.timesteps[3])
    return x, eps, t, torch.tensor(sched.coefficients(t), dtype=torch.float32)


def test_cfg_ddim_ref_matches_the_oracle_step():
    """cfg_ddim_ref with the sampler's fp32 coefficients equals the oracle's CFG combine + DDIM step, rolled."""
    from oracle.sampler import DDIM
    x, eps, t, coef = _ddim_setup()
    sched = DDIM()
    sched.set_timesteps(50)
    e = eps[0].double() + 9.0 * (eps[1].double() - eps[0].double())
    want = torch.roll(sched.step(e, t, x.double()), 8, dims=-1)
    ref, bound = ct.cfg_ddim_ref(x, eps, coef, 9.0, 8)
    assert torch.allclose(ref, want, rtol=0, atol=2e-6)  # the coefficients are fp32
    assert (bound > 0).all()


@pytest.mark.parametrize("bug", ["roll direction", "swapped halves"])
def test_cfg_ddim_bugs_are_caught(bug):
    x, eps, _, coef = _ddim_setup()
    exact = ct.cfg_ddim_ref(x, eps, coef, 9.0, 8)
    if bug == "roll direction":
        mutated, _ = ct.cfg_ddim_ref(x, eps, coef, 9.0, -8)
    else:
        mutated, _ = ct.cfg_ddim_ref(x, eps.flip(0), coef, 9.0, 8)
    _caught(exact, mutated, torch.float32)


@pytest.mark.parametrize("dtype", DTYPES)
def test_timestep_ref_matches_the_oracle_and_swapped_halves_are_caught(dtype):
    from oracle.unet import Timesteps
    t = torch.tensor([999.0, 1.0, 500.0, 21.0])
    ref, bound = ct.timestep_ref(t, 320, dtype)
    want = Timesteps(320)(t).double()  # fp32 frequencies and products: within the bound of the exact value
    assert ((want - ref).abs() <= bound).all()
    mutated = torch.cat([ref[:, 160:], ref[:, :160]], 1)
    _caught((ref, bound), mutated, dtype)


# ---- FAED training kernels (faed_train.cu) --------------------------------------------------------------------------

def _ratio(got, ref, bound):
    return float(torch.nan_to_num((got.double() - ref).abs() / bound, nan=float("inf")).max())


def _wgrad_setup(B=2, H=6, W=9, cin=16, cdy=16, k=3, s=1, seed=30):
    g = torch.Generator().manual_seed(seed)
    p = 1 if s == 2 else k // 2
    Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    x = torch.randn(B, H, W, cin, generator=g).half()
    dy = torch.randn(B, Ho, Wo, cdy, generator=g).half()
    return x, dy, dict(Ho=Ho, Wo=Wo, k=k, stride=s, pad=p)


@pytest.mark.parametrize("k,s", [(3, 1), (9, 1), (4, 2)])
def test_wgrad_ref_matches_autograd(k, s):
    """wgrad_ref's dw / db (Cin_w < Cin, Cout < Cdy) equal autograd's weight gradient of conv2d on circular_pad."""
    import torch.nn.functional as F
    from panfusion_b200.faed_train import circular_pad
    x, dy, kw = _wgrad_setup(W=12, k=k, s=s)
    cin_w, cout = 3, 6
    r = ct.wgrad_ref(x, dy, **kw)
    w = torch.zeros(cout, cin_w, k, k, dtype=torch.float64, requires_grad=True)
    b = torch.zeros(cout, dtype=torch.float64, requires_grad=True)
    y = F.conv2d(circular_pad(x[..., :cin_w].permute(0, 3, 1, 2).double(), kw["pad"]), w, b, stride=s)
    y.backward(dy[..., :cout].permute(0, 3, 1, 2).double())
    assert torch.allclose(ct.wgrad_layout(r["w"], cin_w, cout, k), w.grad, rtol=1e-12, atol=1e-12)
    assert torch.allclose(r["b"][:cout], b.grad, rtol=1e-12, atol=1e-12)
    assert torch.allclose(r["part"].sum(0), r["w"]) and r["part"].shape[0] == r["nch"] > 1 or r["nch"] == 1


def test_wgrad_chunk_restates_the_workspace_size():
    """wgrad_chunk is the kernel's: 200 chunks of 1312 pixels for 32 -> 32 k9 at 256 x 1024 (the 2^24-float cap),
    403 of 5216 for the first layer at 4 x 512 x 1024 (the largest chunk the trainer makes)."""
    assert ct.wgrad_chunk(256 * 1024, 81, 32, 32) == 1312 and -(-256 * 1024 // 1312) == 200
    assert ct.wgrad_chunk(4 * 512 * 1024, 81, 16, 32) == 5216 and -(-4 * 512 * 1024 // 5216) == 403
    assert ct.wgrad_chunk(960, 9, 32, 32) == 960


def _wgrad_bug(bug, chunk):
    """(exact, mutated) partials / reduction / end-to-end for one emulated wgrad bug at the given chunk size."""
    x, dy, kw = _wgrad_setup(B=1, H=2 * chunk // 32 if chunk > 1000 else 6, W=32 if chunk > 1000 else 9, cin=8, cdy=8,
                             k=3, seed=31)
    exact = ct.wgrad_ref(x, dy, chunk=chunk, **kw)
    return x, dy, kw, exact


@pytest.mark.parametrize("chunk", [64, 5216])
@pytest.mark.parametrize("bug", ["seam read as zero", "last stage of a chunk dropped"])
def test_wgrad_partial_bugs_are_caught(bug, chunk):
    x, dy, kw, exact = _wgrad_bug(bug, chunk)
    ok = _ratio(exact["part"].float(), exact["part"], exact["part_bound"])
    if bug == "seam read as zero":
        # taps kx = 0 read column W - 1 only through the wrap (ox = 0): zeroing it there is the bug
        xo = x.clone()
        xo[:, :, -1] = 0
        mutated = exact["part"].clone()
        mutated[:, 0::3] = ct.wgrad_ref(xo, dy, chunk=chunk, **kw)["part"][:, 0::3]
    else:
        dyd = dy.clone().reshape(-1, dy.shape[-1])
        P = dyd.shape[0]
        for c0 in range(0, P, chunk):
            end = min(P, c0 + chunk)
            last = (end - c0 - 1) // 32 * 32 + c0
            dyd[last:end] = 0
        mutated = ct.wgrad_ref(x, dyd.reshape(dy.shape), chunk=chunk, **kw)["part"]
    bad = _ratio(mutated.float(), exact["part"], exact["part_bound"])
    assert ok <= 1.0 < bad, (ok, bad)


@pytest.mark.parametrize("bug", ["column sum added twice", "f applied as inv_n * S", "transposed tap"])
def test_wgrad_reduction_bugs_are_caught(bug):
    """The reduction of the kernel's partials (one chunk's dY column sum added twice, the factor inv_n * S) and the
    end-to-end dw (dw[co][ci][kx][ky]); S = 2^10 with the trainer's inv_n of a 64 x 128 pair."""
    x, dy, kw = _wgrad_setup(B=2, H=8, W=20, k=3, seed=32)
    r = ct.wgrad_ref(x, dy, chunk=64, **kw)
    inv_n, S = 1.0 / (3 * 2 * 64 * 128), 2.0 ** 10
    f = ct.faedt_factor(inv_n, S)
    part, dbpart = r["part"].float(), r["dbpart"].float()
    ref, bound = ct.wgrad_reduce_ref(part, f)
    dref, dbound = ct.wgrad_reduce_ref(dbpart, f)
    good = (part.sum(0) * f, dbpart.sum(0) * f)
    assert _ratio(good[0], ref, bound) <= 1.0 and _ratio(good[1], dref, dbound) <= 1.0
    e2e_ok = _ratio(good[0], f * r["w"], f * r["w_bound"] + ct.U * f * r["w"].abs())
    assert e2e_ok <= 1.0, e2e_ok
    if bug == "column sum added twice":
        bad = _ratio((dbpart.sum(0) + dbpart[1]) * f, dref, dbound)
    elif bug == "f applied as inv_n * S":
        bad = _ratio(part.sum(0) * ct._f32(inv_n * S), ref, bound)
    else:
        k = kw["k"]
        t = part.sum(0) * f
        tt = t.reshape(k, k, *t.shape[1:]).transpose(0, 1).reshape(t.shape)
        bad = _ratio(tt, f * r["w"], f * r["w_bound"] + ct.U * f * r["w"].abs())
    assert bad > 1.0, bad


def _bn_operand(P, C, seed, mean=40.0, spread=0.5):
    """A conv output before BN: each channel's bias (mean ~ 40) large against its spread."""
    g = torch.Generator().manual_seed(seed)
    return (mean + 5 * torch.randn(C, generator=g) + spread * torch.randn(P, C, generator=g)).half()


@pytest.mark.parametrize("P,C", [(3007, 32), (257, 64), (16, 128)])
def test_bn_refs_match_torch_batch_norm(P, C):
    """bn_stats_ref / bn_apply_ref / bn_bwd_ref equal F.batch_norm(training=True), its running-statistic inputs and
    its autograd (through ReLU, the mask from the output)."""
    import torch.nn.functional as F
    z = _bn_operand(P, C, seed=P + C)
    g = torch.Generator().manual_seed(1)
    gamma, beta = 0.5 + torch.rand(C, generator=g), 0.2 * torch.randn(C, generator=g)
    st = ct.bn_stats_ref(z)
    zd = z.double()
    assert torch.equal(st["count"].sum(0), torch.full((C,), float(P), dtype=torch.float64))
    assert torch.allclose(st["stats"][0], zd.mean(0), rtol=1e-12)
    assert torch.allclose(st["stats"][1], 1 / torch.sqrt(zd.var(0, unbiased=False) + ct._f32(1e-5)), rtol=1e-10)
    assert torch.allclose(st["stats"][2], zd.var(0, unbiased=True), rtol=1e-10)
    assert (st["stats_bound"] > 0).all() and (st["m2_bound"] > 0).all()
    stats = st["stats"]  # fp64 statistics: the references then equal torch's to fp64 rounding
    zr = zd.clone().requires_grad_(True)
    gr, br = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    out = F.batch_norm(zr, None, None, gr, br, True, 0.1, ct._f32(1e-5)).relu()
    ref, _ = ct.bn_apply_ref(z, stats, gamma, beta, True)
    assert torch.allclose(ref, out.detach(), rtol=1e-10, atol=1e-10)
    gup = torch.randn(P, C, generator=g).half()
    out.backward(gup.double())
    bw = ct.bn_bwd_ref(gup, out.detach(), z, stats, gamma, 1.0)
    assert torch.allclose(bw["dgamma"], gr.grad, rtol=1e-10, atol=1e-10)
    assert torch.allclose(bw["dbeta"], br.grad, rtol=1e-12, atol=1e-12)
    dz, _ = bw["dz_ref"](bw["sums"])
    assert torch.allclose(dz, zr.grad, rtol=1e-8, atol=1e-8)


def _bn_kernel_like_stats(z):
    """Welford per lane, Chan merges, all in fp32: the kernel's own algorithm on the CPU (chunk counts as floats)."""
    P, C = z.shape
    L, chunk = 256 // C, ct.bn_row_chunk(z.shape[0])
    zf = z.float()

    def merge(a, b):
        n, mean, m2 = a
        nb, mb, m2b = b
        live = nb > 0
        nab = n + nb
        delta = mb - mean
        w = torch.where(live, nb / torch.where(live, nab, torch.ones_like(nab)), torch.zeros_like(nb))
        mean2 = mean + delta * w
        m22 = m2 + (m2b + delta * delta * (n * w))
        return (torch.where(live, nab, n), torch.where(live, mean2, mean), torch.where(live, m22, m2))
    parts, acc = [], None
    for r0 in range(0, P, chunk):
        lanes = []
        for lane in range(L):
            rows = zf[r0 + lane:min(P, r0 + chunk):L]
            n, mean, m2 = torch.zeros(C), torch.zeros(C), torch.zeros(C)
            for v in rows:
                n = n + 1
                d = v - mean
                mean = mean + d / n
                m2 = m2 + d * (v - mean)
            lanes.append((n, mean, m2))
        c = lanes[0]
        for b in lanes[1:]:
            c = merge(c, b)
        parts.append(c)
        acc = c if acc is None else merge(acc, c)
    n, mean, m2 = acc
    stats = torch.stack([mean, 1 / torch.sqrt(m2 / n + ct._f32(1e-5)), m2 / (n - 1)])
    return parts, stats


@pytest.mark.parametrize("P,C", [(257, 32), (600, 128)])
def test_bn_stats_bound_accepts_fp32_welford(P, C):
    """The kernel's algorithm run in fp32 on the CPU passes every per-chunk and merged bound; counts are exact."""
    z = _bn_operand(P, C, seed=40)
    st = ct.bn_stats_ref(z)
    parts, stats = _bn_kernel_like_stats(z)
    assert torch.equal(torch.stack([p[0] for p in parts]).double(), st["count"])
    assert _ratio(torch.stack([p[1] for p in parts]), st["mean"], st["mean_bound"]) <= 1.0
    assert _ratio(torch.stack([p[2] for p in parts]), st["m2"], st["m2_bound"]) <= 1.0
    assert _ratio(stats, st["stats"], st["stats_bound"]) <= 1.0


@pytest.mark.parametrize("P,C", [(257, 32), (16, 128)])
def test_bn_stats_bugs_are_caught(P, C):
    """A chunk's count off by one row (the last chunk of P = 257 has one); invstd from the unbiased variance."""
    z = _bn_operand(P, C, seed=41)
    st = ct.bn_stats_ref(z)
    if P > 256:
        short = ct.bn_stats_ref(z[:P - 1])
        assert not torch.equal(short["count"].sum(0), st["count"].sum(0))
    var_u = st["stats"][2]
    mutated = st["stats"].clone()
    mutated[1] = 1 / torch.sqrt(var_u + ct._f32(1e-5))
    assert _ratio(st["stats"].float(), st["stats"], st["stats_bound"]) <= 1.0
    assert _ratio(mutated.float(), st["stats"], st["stats_bound"]) > 1.0


@pytest.mark.parametrize("bug", ["mask from pre-ReLU z", "dz without the xhat term"])
def test_bn_bwd_bugs_are_caught(bug):
    """At the trainer's deepest level (P = 16, C = 128) and at P = 3007, C = 32."""
    for P, C in ((16, 128), (3007, 32)):
        z = _bn_operand(P, C, seed=42, mean=0.3, spread=1.0)
        g = torch.Generator().manual_seed(2)
        gamma, beta = 0.5 + torch.rand(C, generator=g), 0.2 * torch.randn(C, generator=g)
        stats = ct.bn_stats_ref(z)["stats"].float()
        out = ct.bn_apply_ref(z, stats, gamma, beta, True)[0].half()
        gup = torch.randn(P, C, generator=g).half()
        bw = ct.bn_bwd_ref(gup, out, z, stats, gamma, 1.0)
        ref, bound = bw["dz_ref"](bw["sums"].float())
        assert _ratio(ref.half(), ref, bound) <= 1.0
        if bug == "mask from pre-ReLU z":
            mut = ct.bn_bwd_ref(gup, z, z, stats, gamma, 1.0)
            bad = max(_ratio(mut["dbeta"].float(), bw["dbeta"], bw["dbeta_bound"]),
                      _ratio(mut["dz_ref"](bw["sums"].float())[0].half(), ref, bound))
        else:
            s = bw["sums"].float().double()
            bad = _ratio((gamma.double() * stats[1].double() * (gup.double() * (out.double() > 0) - s[0])).half(),
                         ref, bound)
        assert bad > 1.0, (P, C, bad)


@pytest.mark.parametrize("H,W", [(1, 5), (5, 1), (3, 7), (4, 8)])
def test_upsample_refs_match_interpolate_and_catch_bugs(H, W):
    """upsample_ref is F.interpolate (bilinear, align_corners=False) and upsample_bwd_ref its autograd; align_corners
    =True, a wrapped far edge and a backward gather missing output 2i - 1 are caught."""
    import torch.nn.functional as F
    g = torch.Generator().manual_seed(H * 10 + W)
    x = torch.randn(2, H, W, 8, generator=g).half()
    gy = torch.randn(2, 2 * H, 2 * W, 8, generator=g).half()
    ref, bound = ct.upsample_ref(x)
    xr = x.permute(0, 3, 1, 2).double().requires_grad_(True)
    y = F.interpolate(xr, scale_factor=2, mode="bilinear", align_corners=False)
    assert torch.allclose(ref, y.detach().permute(0, 2, 3, 1), rtol=1e-14, atol=1e-14)
    y.backward(gy.permute(0, 3, 1, 2).double())
    bref, bbound = ct.upsample_bwd_ref(gy, H, W)
    assert torch.allclose(bref, xr.grad.permute(0, 2, 3, 1), rtol=1e-14, atol=1e-14)
    assert _ratio(ref.half(), ref, bound) <= 1.0 and _ratio(bref.half(), bref, bbound) <= 1.0
    xd = x.double().permute(0, 3, 1, 2)
    bad = [_ratio(F.interpolate(xd, scale_factor=2, mode="bilinear", align_corners=True).permute(0, 2, 3, 1).half(),
                  ref, bound)]
    if W > 1:  # the far edge wrapped to column 0 instead of clamped
        wrapped = F.interpolate(torch.cat([xd, xd[..., :1]], -1), size=(2 * H, 2 * W + 2), mode="bilinear",
                                align_corners=False)
        wrapped = F.interpolate(torch.cat([xd, xd[..., :1]], -1), scale_factor=2, mode="bilinear",
                                align_corners=False)[..., :2 * W]
        bad.append(_ratio(wrapped.permute(0, 2, 3, 1).half(), ref, bound))
    # the gather over outputs 2i .. 2i + 2 only (output 2i - 1 dropped)
    gd = gy.double().permute(0, 3, 1, 2)
    miss = torch.zeros_like(gd)
    miss[..., 0::2, :] = 1
    miss[..., 0, :] = 1
    keep_y = torch.ones(2 * H, dtype=torch.float64)
    keep_y[1::2] = 0
    keep_y[2 * H - 1] = 1 if H == 1 else 0
    xr2 = torch.zeros_like(xr).requires_grad_(True)
    yy = F.interpolate(xr2, scale_factor=2, mode="bilinear", align_corners=False)
    # an input row iy keeps outputs 2 iy, 2 iy + 1, 2 iy + 2 and loses 2 iy - 1: emulate on a per-input basis
    rows = []
    for iy in range(H):
        (gi,) = torch.autograd.grad(yy, xr2, gd * _drop_row_mask(H, W, iy), retain_graph=True)
        rows.append(gi[..., iy, :])
    missing = torch.stack(rows, -2).permute(0, 2, 3, 1)
    if H > 1:
        bad.append(_ratio(missing.half(), bref, bbound))
    assert all(b > 1.0 for b in bad), bad


def _drop_row_mask(H, W, iy):
    """The outputs input row iy gathers from, without output row 2 iy - 1."""
    m = torch.ones(2 * H, 2 * W, dtype=torch.float64)
    if iy > 0:
        m[2 * iy - 1] = 0
    return m


def _loss_setup(B=2, H=4, W=8, seed=50):
    g = torch.Generator().manual_seed(seed)
    o = torch.randn(B, H, W, 4, generator=g) * 2
    t = torch.rand(B, 3, H, W, generator=g) * 2 - 1
    o[0, 0, :3, :3] = 0
    t[0, :, 0, :3] = 0  # d = 0 exactly: sign(0) = 0
    return o, t


def test_loss_ref_matches_torch_and_catches_bugs():
    """pred = tanh, the L1 mean and autograd's seed direction; sign(0) = 1, a seed without (1 - pred^2) and the mean
    over 4 channels are caught."""
    B, H, W = 2, 4, 8
    o, t = _loss_setup(B, H, W)
    r = ct.loss_ref(o, t, B, H, W)
    orr = o[..., :3].permute(0, 3, 1, 2).double().requires_grad_(True)
    loss = (torch.tanh(orr) - t.double()).abs().mean()
    loss.backward()
    assert torch.allclose(r["loss"], loss.detach(), rtol=1e-14)
    pred = r["pred"].float()
    assert _ratio(pred, r["pred"], r["pred_bound"]) <= 1.0
    S = 2.0 ** 15
    # autograd's gradient is sign(d) (1 - tanh^2) / count: the seed is that times S * count
    want = (orr.grad * 3 * B * H * W * S)
    seed = torch.zeros(B, H, W, 16, dtype=torch.float16)
    seed[..., :3] = want.permute(0, 2, 3, 1).half()
    ok, n_clear = ct.seed_check(seed, pred, r["d"], r["pred_bound"], S)
    assert ok <= 1.0 and n_clear > 0, ok
    assert _ratio(torch.tensor(float(r["loss"])), r["loss"], r["loss_bound"]) <= 1.0
    sign1 = torch.where(r["d"] == 0, torch.ones_like(r["d"]), torch.sign(r["d"]))
    bad_seed = seed.clone()
    bad_seed[..., :3] = (sign1 * (1 - pred.double() ** 2) * S).permute(0, 2, 3, 1).half()
    assert ct.seed_check(bad_seed, pred, r["d"], r["pred_bound"], S)[0] > 1.0
    bad_seed[..., :3] = (torch.sign(r["d"]) * S).permute(0, 2, 3, 1).half()
    assert ct.seed_check(bad_seed, pred, r["d"], r["pred_bound"], S)[0] > 1.0
    four = (r["d"].abs().sum() + (torch.tanh(o[..., 3].double())).abs().sum()) / (4 * B * H * W)
    assert _ratio(four, r["loss"], r["loss_bound"]) > 1.0


def test_pack_ref_adjoints_match_autograd():
    """pack_ref's stride-1 flipped kernel and stride-2 phase kernels, convolved as FAEDTrainer._dgrad does, give
    autograd's input gradient of the circular convolution (fp64, before the fp16 rounding)."""
    import torch.nn.functional as F
    from panfusion_b200.faed_train import circular_pad
    g = torch.Generator().manual_seed(60)
    for k, s in ((3, 1), (4, 2)):
        cin, cout, B, H, W = 5, 6, 1, 6, 8
        p = 1 if s == 2 else k // 2
        w = torch.randn(cout, cin, k, k, generator=g, dtype=torch.float64)
        x = torch.randn(B, cin, H, W, generator=g, dtype=torch.float64, requires_grad=True)
        y = F.conv2d(circular_pad(x, p), w, stride=s)
        gy = torch.randn(y.shape, generator=g, dtype=torch.float64)
        y.backward(gy)
        fwd, dg = pack_ref_fp64(w, k, s)
        assert torch.equal(fwd[:, :cin, :cout], w.permute(2, 3, 1, 0).reshape(k * k, cin, cout))
        if s == 1:
            wt = dg.reshape(k, k, cout, cin).permute(3, 2, 0, 1)
            dx = F.conv2d(circular_pad(gy, p), wt)
        else:
            dx = torch.zeros_like(x)
            for r in (0, 1):
                for c in (0, 1):
                    wt = dg[4 * (2 * r + c):4 * (2 * r + c) + 4].reshape(2, 2, cout, cin).permute(3, 2, 0, 1)
                    gp = F.pad(gy, (0, 0, 1 - r, r))
                    gp = torch.cat([gp[..., gp.shape[-1] - (1 - c):], gp, gp[..., :c]], -1)
                    dx[..., r::2, c::2] = F.conv2d(gp, wt)
        assert torch.allclose(dx, x.grad, rtol=1e-12, atol=1e-12), (k, s)


def pack_ref_fp64(w, k, s):
    """pack_ref applied to the weights' flat indices (exact in fp16 below 2048), then to the fp64 weights."""
    Cout, Cin = w.shape[:2]
    idx = torch.arange(w.numel(), dtype=torch.float32).reshape(w.shape)
    fi, di = ct.pack_ref(idx, k, s, Cin, Cout, Cout, Cin)
    flat = w.reshape(-1)
    return flat[fi.long()], flat[di.long()]


# ---- conv_in, VAE softmax, latent sampling, training loss (elementwise.cu) ------------------------------------------

def _conv_in_setup(N=2, Cin=4, H=5, W=8, Cout=16, seed=70):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, Cin, H, W, generator=g)
    x[..., 0] += 2.0   # the seam columns differ from their wrapped neighbours
    x[..., -1] -= 2.0
    w = torch.randn(Cout, Cin, 3, 3, generator=g) * 0.3
    return g, x, w, torch.randn(Cout, generator=g)


def _tokens(t):
    return t.double().permute(0, 2, 3, 1).reshape(-1, t.shape[1])


@pytest.mark.parametrize("circ", [False, True])
@pytest.mark.parametrize("act", [ct.ACT_NONE, ct.ACT_SILU])
def test_conv_in_ref_matches_torch(circ, act):
    """conv_in_ref equals F.conv2d (on pad_pano(x, 1) for the circular case, rows zero-padded), then SiLU."""
    import torch.nn.functional as F
    from oracle.eppa import pad_pano, unpad_pano
    _, x, w, b = _conv_in_setup()
    xd, wd, bd = x.double(), w.double(), b.double()
    want = unpad_pano(F.conv2d(pad_pano(xd, 1), wd, bd, padding=1), 1) if circ else F.conv2d(xd, wd, bd, padding=1)
    if act == ct.ACT_SILU:
        want = F.silu(want)
    ref, bound = ct.conv_in_ref(x, w, b, circ, act, torch.float16)
    assert torch.allclose(ref, _tokens(want), rtol=1e-12, atol=1e-12) and (bound > 0).all()


def test_conv_in_ref_of_the_decoder_fold_matches_post_quant_then_conv_in():
    """VAEDecoderPack's fold: conv_in over [z | ones] with the composed weights equals post_quant_conv (1 x 1) followed
    by conv_in with zero padding; zero output channels (the ControlNet's padding to 64) must be exact zeros."""
    import torch.nn.functional as F
    g, z, wi, b = _conv_in_setup(Cin=4, Cout=16, seed=71)
    wq, bq = torch.randn(4, 4, generator=g).double(), torch.randn(4, generator=g).double()
    w5 = torch.cat([torch.einsum("octs,ci->oits", wi.double(), wq), torch.einsum("octs,c->ots", wi.double(), bq)[:, None]], 1)
    x5 = torch.cat([z, torch.ones_like(z[:, :1])], 1)
    ref, _ = ct.conv_in_ref(x5, w5, b, False, ct.ACT_NONE, torch.float16)
    want = F.conv2d(F.conv2d(z.double(), wq[..., None, None], bq), wi.double(), b.double(), padding=1)
    assert torch.allclose(ref, _tokens(want), rtol=1e-12, atol=1e-12)
    wp, bp = torch.zeros(64, 4, 3, 3), torch.zeros(64)
    wp[:16], bp[:16] = wi, b
    _, bound = ct.conv_in_ref(z, wp, bp, False, ct.ACT_SILU, torch.float16)
    assert (bound[:, 16:] == ct.EXACT).all() and (bound[:, :16] > ct.EXACT).all()


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("bug", ["seam wrapped to zero", "previous image's last row", "missing bias",
                                 "silu before the bias", "ones channel padded as data"])
def test_conv_in_bugs_are_caught(dtype, bug):
    """The seam column read as zero padding; row 0 of image n reading image n - 1's last row (the images stacked
    without a border); the bias never seeded; SiLU applied before the bias; the decoder fold's ones channel padded
    with ones (post_quant_conv's bias folded into conv_in's bias), which changes only the border pixels."""
    g, x, w, b = _conv_in_setup(Cin=5 if bug == "ones channel padded as data" else 4)
    circ = bug == "seam wrapped to zero"
    act = ct.ACT_SILU if bug == "silu before the bias" else ct.ACT_NONE
    if bug == "ones channel padded as data":
        x[:, 4] = 1.0
    exact = ct.conv_in_ref(x, w, b, circ, act, dtype)
    N, Cin, H, W = x.shape
    if bug == "seam wrapped to zero":
        mutated, _ = ct.conv_in_ref(x, w, b, False, act, dtype)
    elif bug == "previous image's last row":
        stacked = x.permute(1, 0, 2, 3).reshape(1, Cin, N * H, W)
        mutated, _ = ct.conv_in_ref(stacked, w, b, circ, act, dtype)
    elif bug == "missing bias":
        mutated, _ = ct.conv_in_ref(x, w, None, circ, act, dtype)
    elif bug == "silu before the bias":
        mutated = ct.conv_in_ref(x, w, None, circ, act, dtype)[0] + b.double()
    else:
        mutated, _ = ct.conv_in_ref(x[:, :4], w[:, :4], b + w[:, 4].sum((1, 2)), circ, act, dtype)
    _caught(exact, mutated, dtype)


def _softmax_logits(rows, cols, scale, seed=72):
    """Logits as the VAE attention makes them: each row its own offset, a spread of +-50 after scaling."""
    g = torch.Generator().manual_seed(seed)
    off = 400 * torch.rand(rows, 1, generator=g) - 200
    return (off + 50 * (2 * torch.rand(rows, cols, generator=g) - 1)) / scale


def test_softmax_rows_ref_matches_torch_softmax():
    scale = 512 ** -0.5
    s = _softmax_logits(6, 777, scale)
    ref, bound = ct.softmax_rows_ref(s[:, :700], scale, torch.float16)  # a view with ld > cols
    want = torch.softmax(ct._f32(scale) * s[:, :700].double(), -1)
    assert torch.allclose(ref, want, rtol=1e-12, atol=0) and (bound > 0).all()


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("bug", ["scaled before the max", "dropped last odd column"])
def test_softmax_rows_bugs_are_caught(dtype, bug):
    """exp(scale x - max x): the logits scaled before the unscaled maximum is subtracted, which overflows fp32 on a
    negative-going row; the last column of an odd-width row never stored."""
    scale, cols = 512 ** -0.5, 1025
    s = _softmax_logits(4, cols, scale)
    s[1] -= 3000.0  # a row far below zero
    exact = ct.softmax_rows_ref(s, scale, dtype)
    if bug == "scaled before the max":
        e = torch.exp(s * ct._f32(scale) - s.amax(1, keepdim=True))  # fp32, as the kernel would compute it
        mutated = (e / e.sum(1, keepdim=True)).double()
    else:
        mutated = exact[0].clone()
        mutated[:, -1] = float("nan")
    _caught(exact, mutated, dtype)


def _moments(N=2, L=4, h=3, w=5, ld=64, seed=73):
    g = torch.Generator().manual_seed(seed)
    mom = torch.full((N * h * w, ld), float("nan"))
    mom[:, :L] = torch.randn(N * h * w, L, generator=g) * 3
    mom[:, L:2 * L] = torch.rand(N * h * w, L, generator=g) * 60 - 35  # logvar in [-35, 25): both clamp edges
    return mom, torch.randn(N, L, h, w, generator=g)


def test_gaussian_sample_ref_matches_diagonal_gaussian_sample():
    """The diffusers formula (oracle DiagonalGaussianDistribution.sample with the given noise) times the scale, and
    NaN in from either the mean or the logvar gives NaN out."""
    from oracle.vae import DiagonalGaussianDistribution
    mom, eps = _moments()
    mom[3, 1], mom[7, 4 + 2] = float("nan"), float("nan")
    N, L, h, w = eps.shape
    params = mom[:, :2 * L].double().reshape(N, h, w, 2 * L).permute(0, 3, 1, 2)
    want = DiagonalGaussianDistribution(params).sample(noise=eps.double()) * ct._f32(0.18215)
    ref, bound = ct.gaussian_sample_ref(mom, mom.stride(0), eps, L, 0.18215)
    assert torch.allclose(ref, want, rtol=1e-12, atol=0, equal_nan=True)
    assert torch.isnan(ref).sum() == 2 and torch.equal(torch.isnan(ref), torch.isnan(bound))


@pytest.mark.parametrize("bug", ["clamp at 30", "mean and logvar swapped", "NHWC output"])
def test_gaussian_sample_bugs_are_caught(bug):
    mom, eps = _moments()
    N, L, h, w = eps.shape
    exact = ct.gaussian_sample_ref(mom, mom.stride(0), eps, L, 0.18215)
    if bug == "clamp at 30":
        m4 = mom[:, :2 * L].double().reshape(N, h, w, 2 * L).permute(0, 3, 1, 2)
        mutated = (m4[:, :L] + torch.exp(0.5 * m4[:, L:].clamp(-30.0, 30.0)) * eps.double()) * ct._f32(0.18215)
    elif bug == "mean and logvar swapped":
        sw = mom.clone()
        sw[:, :L], sw[:, L:2 * L] = mom[:, L:2 * L], mom[:, :L]
        mutated, _ = ct.gaussian_sample_ref(sw, sw.stride(0), eps, L, 0.18215)
    else:
        mutated = exact[0].permute(0, 2, 3, 1).reshape(exact[0].shape)
    _caught(exact, mutated, torch.float32)


def _mse_like_the_kernel(a, b):
    """pf_mse_loss in fp32: 296 chunks, 256 thread-strided chains each, a shuffle tree, 8 warp partials in series,
    then the fp64 sum of the partials and the fp64 mean rounded to fp32."""
    n = a.numel()
    chunk = -(-n // ct.MSE_CTAS)
    k = -(-chunk // 256)
    d = torch.zeros(ct.MSE_CTAS * chunk)
    d[:n] = a.reshape(-1) - b.reshape(-1)
    d = torch.nn.functional.pad(d.reshape(ct.MSE_CTAS, chunk), (0, k * 256 - chunk)).reshape(ct.MSE_CTAS, k, 256)
    acc = torch.zeros(ct.MSE_CTAS, 256)
    for i in range(k):
        acc = acc + d[:, i] * d[:, i]
    acc = acc.reshape(ct.MSE_CTAS, 8, 32)
    for o in (16, 8, 4, 2, 1):
        acc = acc[..., :o] + acc[..., o:2 * o]
    s = torch.zeros(ct.MSE_CTAS)
    for wi in range(8):
        s = s + acc[:, wi, 0]
    return torch.tensor(float(s.double().sum() / n), dtype=torch.float32)


@pytest.mark.parametrize("n", [100, 296 * 37 - 1, 296 * 443 + 1])
def test_mse_ref_matches_torch_and_catches_the_padded_count(n):
    """mse_ref equals F.mse_loss; the kernel's fp32 summation order passes its bound; a mean over the padded count
    296 * ceil(n / 296) fails it."""
    g = torch.Generator().manual_seed(n)
    a, b = torch.randn(n, generator=g) * 2 + 0.5, torch.randn(n, generator=g)
    ref, bound = ct.mse_ref(a, b)
    assert torch.allclose(ref, torch.nn.functional.mse_loss(a.double(), b.double()), rtol=1e-13, atol=0)
    assert abs(_mse_like_the_kernel(a, b).double() - ref) <= bound
    assert abs(ref.float().double() - ref) <= bound
    padded = (a.double() - b.double()).pow(2).sum() / (ct.MSE_CTAS * -(-n // ct.MSE_CTAS))
    assert abs(padded.float().double() - ref) > bound
