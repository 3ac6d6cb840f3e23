"""-m gpu: pf_gemm_taps' A windows against the fp64 restatement of the header contract (tests/_contract.py).

Taps whose offsets lie within 8 rows of each other share one A window of 136 rows, and each tap's wgmma operand starts
1..8 rows into it. These cases put taps at every shift inside a window, windows that start before row 0 and end past
a_rows (zero-filled by the TMA), groups of 1, 2, 3 and 9 taps in one call, taps passed out of offset order, and spans
exactly at the limit and one past it, at every tile width, with fp32 and 16-bit direct stores and split-K.
M = 1000 is not a multiple of 128, so the first and the last, partial, M-tile both read clipped windows."""
import pytest
import torch

import _contract as ct

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]

# name -> taps (row offsets, in the caller's order)
TAP_SETS = {
    "shift_0_1_2": [0, 1, 2],
    "shift_2_1_0_before_row_0": [-2, -1, 0],
    "every_shift_1_to_8": [0, 1, 2, 3, 4, 5, 6, 7, 8],
    "groups_3_2_1_unsorted": [40, -3, 20, 21, -5, -4],
    "span_at_limit_and_past": [3, -5, 11, 12, 19, 27, 36],
    "3x3_row_pitch_5": [(dy - 1) * 5 + (dx - 1) for dy in range(3) for dx in range(3)],
    "3x3_row_pitch_3_one_window": [(dy - 1) * 3 + (dx - 1) for dy in range(3) for dx in range(3)],
    "downsample_phases": [((dy % 2) * 2 + (dx % 2)) * 300 + (dy // 2) * 12 + (dx // 2)
                          for dy in range(3) for dx in range(3)],
}


def _operands(taps, dt, dev, M=1000, Kc=128, N=160, seed=0):
    g = torch.Generator().manual_seed(seed)
    A = torch.randn((M, Kc), generator=g).to(dt).to(dev)  # a_rows = M: windows of the last tile end past it
    B = (torch.randn((N, len(taps) * Kc), generator=g) * (len(taps) * Kc) ** -0.5).to(dt).to(dev)
    bias = (torch.randn(N, generator=g) * 0.1).to(dev)
    return A, B, bias


def _check(name, got, ref, bound):
    rows = ~torch.isnan(ref[:, 0])
    assert not torch.isnan(got.double()[rows]).any(), f"{name}: NaN in a written row"
    err = (got.double()[rows] - ref[rows]).abs()
    bad = err > bound[rows]
    assert not bad.any(), (f"{name}: {int(bad.sum())} elements over the bound, worst "
                           f"{(err / bound[rows]).max().item():.3g} x bound")


@pytest.mark.parametrize("dtype", DTYPES, ids=["f16", "bf16"])
@pytest.mark.parametrize("block_n", [64, 128, 160])
@pytest.mark.parametrize("taps", list(TAP_SETS), ids=list(TAP_SETS))
def test_tap_windows_direct_store(cuda_device, taps, block_n, dtype):
    """fp32 output: the direct-store epilogue at every co-resident tile width."""
    from panfusion_b200 import ops
    tp = TAP_SETS[taps]
    A, B, bias = _operands(tp, dtype, cuda_device, N=2 * block_n)
    M = A.shape[0]
    out = torch.full((M, B.shape[0]), float("nan"), dtype=torch.float32, device=cuda_device)
    ops.gemm_taps(A, B, out, M=M, Kc=A.shape[1], taps=tp, bias=bias, block_n=block_n, k_splits=1)
    ref, bound = ct.tap_gemm_ref(A, B, M, torch.float32, M=M, Kc=A.shape[1], taps=tp, bias=bias)
    _check(f"{taps} block_n={block_n}", out, ref, bound)


@pytest.mark.parametrize("dtype", DTYPES, ids=["f16", "bf16"])
@pytest.mark.parametrize("taps", list(TAP_SETS), ids=list(TAP_SETS))
def test_tap_windows_tma_store(cuda_device, taps, dtype):
    """16-bit output with a 16-bit residual: the direct-store epilogue's 16-bit path."""
    from panfusion_b200 import ops
    tp = TAP_SETS[taps]
    A, B, bias = _operands(tp, dtype, cuda_device, seed=1)
    M, N = A.shape[0], B.shape[0]
    res = torch.randn((M, N), generator=torch.Generator().manual_seed(2)).to(dtype).to(cuda_device)
    out = torch.full((M, N), float("nan"), dtype=dtype, device=cuda_device)
    ops.gemm_taps(A, B, out, M=M, Kc=A.shape[1], taps=tp, bias=bias, residual=res, k_splits=1)
    ref, bound = ct.tap_gemm_ref(A, B, M, dtype, M=M, Kc=A.shape[1], taps=tp, bias=bias, residual=res)
    _check(taps, out, ref, bound)


@pytest.mark.parametrize("dtype", DTYPES, ids=["f16", "bf16"])
@pytest.mark.parametrize("k_splits", [2, 3, 5])
@pytest.mark.parametrize("taps", ["groups_3_2_1_unsorted", "3x3_row_pitch_5", "downsample_phases"])
def test_tap_windows_split_k(cuda_device, taps, k_splits, dtype):
    """Split-K cuts K between (window group, channel slab) units, also inside a group's channel slabs (Kc = 320)."""
    from panfusion_b200 import ops
    tp = TAP_SETS[taps]
    A, B, bias = _operands(tp, dtype, cuda_device, M=300, Kc=320, seed=3)
    M = A.shape[0]
    out = torch.full((M, B.shape[0]), float("nan"), dtype=dtype, device=cuda_device)
    ops.gemm_taps(A, B, out, M=M, Kc=A.shape[1], taps=tp, bias=bias, k_splits=k_splits)
    ref, bound = ct.tap_gemm_ref(A, B, M, dtype, M=M, Kc=A.shape[1], taps=tp, bias=bias)
    _check(f"{taps} k_splits={k_splits}", out, ref, bound)


@pytest.mark.parametrize("dtype", DTYPES, ids=["f16", "bf16"])
def test_tap_windows_conv_image_map(cuda_device, dtype):
    """A 3x3 convolution through the halo-dropping row map: 2 images of 9 x 13 pixels (M = 2 * 11 * 15 = 330)."""
    from panfusion_b200 import ops
    from panfusion_b200.engine import taps3x3
    N, H, W, C, CO = 2, 9, 13, 64, 320
    g = torch.Generator().manual_seed(4)
    x = torch.randn((N * H * W, C), generator=g).to(dtype).to(cuda_device)
    A = ops.conv_prep(x, N, H, W, halo=1)
    Hp, Wp = H + 2, W + 2
    tp = taps3x3(Wp)
    B = (torch.randn((CO, 9 * C), generator=g) * (9 * C) ** -0.5).to(dtype).to(cuda_device)
    out = torch.full((N * H * W, CO), float("nan"), dtype=dtype, device=cuda_device)
    kw = dict(M=N * Hp * Wp, Kc=C, taps=tp, image_map=(Hp, Wp, 1, 1, H, W))
    ops.gemm_taps(A, B, out, k_splits=1, **kw)
    ref, bound = ct.tap_gemm_ref(A, B, out.shape[0], dtype, **kw)
    _check("conv 9x13", out, ref, bound)


@pytest.mark.parametrize("dtype", DTYPES, ids=["f16", "bf16"])
def test_tap_windows_repeatable_and_order_free(cuda_device, dtype):
    """The K order depends on the tap offsets alone: the same taps in another caller order, with B's tap blocks
    permuted to match, give bit-identical results, and so do repeated launches."""
    from panfusion_b200 import ops
    tp = TAP_SETS["groups_3_2_1_unsorted"]
    A, B, bias = _operands(tp, dtype, cuda_device, seed=5)
    M, N, Kc = A.shape[0], B.shape[0], A.shape[1]
    perm = [3, 0, 5, 1, 4, 2]
    Bp = torch.cat([B[:, p * Kc:(p + 1) * Kc] for p in perm], 1).contiguous()
    outs = []
    for taps, w in ((tp, B), (tp, B), ([tp[p] for p in perm], Bp)):
        o = torch.empty((M, N), dtype=torch.float32, device=cuda_device)
        ops.gemm_taps(A, w, o, M=M, Kc=Kc, taps=taps, bias=bias, k_splits=1)
        outs.append(o)
    assert torch.equal(outs[0], outs[1])
    assert torch.equal(outs[0], outs[2])
