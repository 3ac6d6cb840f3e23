"""CPU: the error bounds of tests/_contract.py (used by test_gpu_contracts.py) are tight enough to fail.

Each case computes the exact fp64 result of a small tap-GEMM or attention, rounds it to the output type as a correct
kernel would, and checks that it passes the bound; then it emulates one subtle kernel bug (a dropped tap, a shifted
row-bias group, a halo row in the output, a residual read one row off, swapped GEGLU halves, an unmasked ragged key, a
bias read from the wrong batch) and checks that the bound catches it on at least one element."""
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
