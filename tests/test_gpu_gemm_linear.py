"""-m gpu: the persistent linear GEMM behind pf_gemm_taps (one tap, plain row map, 16-bit output) against the fp64
restatement of the header contract (tests/_contract.py), at what persistence adds to the tap-GEMM:

- M of 1, 127, 129, 1000 and 65 600: a partial last m-tile, whose rows past M are neither written nor read as residual;
- grids with fewer tiles than SMs, one tile per SM, one tile more, and many tiles per CTA;
- K of 64 (fewer K-slabs than ring slots), 320, 640 and 1600 (the ring wraps inside a tile and across tiles);
- every tile width with each epilogue: bias, GELU / SiLU, LayerNorm consumer, residual with row statistics, GEGLU into
  a column slice;
- a row-statistics producer feeding a LayerNorm consumer;
- byte-identical repeats (direct and replayed from a CUDA graph), and row statistics that do not depend on M.
Outputs are pre-filled with NaN (a missed element fails) and column slices keep their NaN neighbours (an element
written outside the slice fails)."""
import pytest
import torch

import _contract as ct

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]
SILU, GELU, GEGLU = 1, 2, 3


def _rand(g, shape, dev, dtype, scale=1.0):
    return (torch.randn(shape, generator=g) * scale).to(dtype).to(dev)


def _nan(shape, dtype, dev):
    return torch.full(shape, float("nan"), dtype=dtype, device=dev)


def _lin_ln(g, n, k, dev, dtype, geglu_bn=0):
    from panfusion_b200.engine import _LinLN
    norm = torch.nn.LayerNorm(k)
    with torch.no_grad():
        norm.weight.copy_(1 + 0.3 * torch.randn(k, generator=g))
        norm.bias.copy_(0.2 * torch.randn(k, generator=g))
    return _LinLN(torch.randn(n, k, generator=g) / k ** 0.5, torch.randn(n, generator=g) * 0.5, norm, dev, dtype,
                  geglu_bn=geglu_bn)


def _ln_stats(x):
    """(sum, sum of squares) of every stored 16-bit row in slot 0, zeros in slot 1."""
    x64 = x.double()
    st = torch.zeros((x.shape[0], 2, 2), dtype=torch.float64, device=x.device)
    st[:, 0, 0], st[:, 0, 1] = x64.sum(1), (x64 * x64).sum(1)
    return st.float().contiguous()


def _check(name, got, ref, bound):
    got = got.double()
    rows = ~torch.isnan(ref[:, 0])
    assert torch.isnan(got[~rows]).all(), f"{name}: a row past M was written"
    assert not torch.isnan(got[rows]).any(), f"{name}: NaN in a written row"
    err = (got[rows] - ref[rows]).abs()
    bad = err > bound[rows]
    assert not bad.any(), (f"{name}: {int(bad.sum())} elements over the bound, worst "
                           f"{(err / bound[rows]).max().item():.3g} x bound")


def _stats_ref(out):
    """fp64 (sum, sum of squares) per row of the fp32 values the statistics sum; checked on the stored outputs."""
    o = out.double()
    return o.sum(1), (o * o).sum(1)


def _check_stats(name, stats, out, rows):
    s, q = _stats_ref(out[:rows])
    ks, kq = stats[:rows, :, 0].double().sum(1), stats[:rows, :, 1].double().sum(1)
    n = out.shape[1]
    # the statistics sum fp32 values before the 16-bit rounding of the stored outputs
    u = 2.0 ** -7 if out.dtype == torch.bfloat16 else 2.0 ** -10
    mag = out[:rows].double().abs().sum(1)
    assert ((ks - s).abs() <= u * mag + 1e-3 * n ** 0.5).all(), f"{name}: row sums"
    assert ((kq - q).abs() <= 3 * u * (out[:rows].double() ** 2).sum(1) + 1e-3).all(), f"{name}: row sums of squares"


EPILOGUES = ["bias", "gelu", "silu", "ln", "res_stats"]
MK = [(1, 64), (127, 320), (129, 640), (1000, 1600), (65600, 320)]


def _linear_case(g, dev, dt, M, K, N, epi, bn, res_cols=None):
    from panfusion_b200 import ops
    A = _rand(g, (M, K), dev, dt)
    kw = dict(M=M, Kc=K, block_n=bn)
    ref_kw = dict(M=M, Kc=K)
    if epi == "ln":
        p = _lin_ln(g, N, K, dev, dt)
        B = p.w
        kw.update(bias=p.b, ln=(_ln_stats(A), p.colsum, p.eps))
        ref_kw.update(bias=p.b, ln_eps=p.eps)
    else:
        B = _rand(g, (N, K), dev, dt, scale=K ** -0.5)
        bias = (torch.randn(N, generator=g) * 0.5).to(dev)
        kw["bias"] = bias
        ref_kw["bias"] = bias
        if epi in ("gelu", "silu"):
            kw["act"] = ref_kw["act"] = GELU if epi == "gelu" else SILU
    if epi == "res_stats":
        # the residual is a column slice of a wider tensor: a read past the slice adds the wrong values
        wide = _rand(g, (M, N + (res_cols or 0)), dev, dt)
        res = wide[:, :N]
        kw.update(residual=res, row_stats=True)
        ref_kw["residual"] = res
    out = _nan((M, N), dt, dev)
    ref, bound = ct.tap_gemm_ref(A, B, M, dt, **ref_kw)
    r = ops.gemm_taps(A, B, out, **kw)
    return out, ref, bound, (r[1] if epi == "res_stats" else None)


@pytest.mark.parametrize("dtype", DTYPES, ids=["f16", "bf16"])
@pytest.mark.parametrize("block_n", [64, 128, 160])
@pytest.mark.parametrize("epi", EPILOGUES)
@pytest.mark.parametrize("mk", MK, ids=[f"M{m}_K{k}" for m, k in MK])
def test_linear_epilogues(cuda_device, mk, epi, block_n, dtype):
    M, K = mk
    if M == 65600 and dtype == torch.float16:
        pytest.skip("many-wave case: bf16 only")
    g = torch.Generator().manual_seed(M + K + block_n)
    N = 2 * block_n if block_n != 160 else 320
    out, ref, bound, stats = _linear_case(g, cuda_device, dtype, M, K, N, epi, block_n, res_cols=24)
    name = f"M={M} K={K} {epi} block_n={block_n}"
    _check(name, out, ref, bound)
    if stats is not None:
        from panfusion_b200 import ops
        assert stats.shape == (M, 2 * N // ops.pick_block_n(N), 2)  # a producer's width comes from N alone
        _check_stats(name, stats, out, M)


SMS_GRIDS = ["below_sms", "one_per_sm", "one_more", "many_waves"]


@pytest.mark.parametrize("grid", SMS_GRIDS)
@pytest.mark.parametrize("epi", ["res_stats", "ln"])
def test_linear_grid_sizes(cuda_device, grid, epi):
    """Tiles below, at and one above the SM count, and many tiles per CTA, at the 160-wide tile and K = 640."""
    sms = torch.cuda.get_device_properties(cuda_device).multi_processor_count
    M = {"below_sms": 128 * (sms // 2) - 5, "one_per_sm": 128 * sms, "one_more": 128 * sms + 1,
         "many_waves": 65600}[grid]
    g = torch.Generator().manual_seed(7)
    out, ref, bound, stats = _linear_case(g, cuda_device, torch.bfloat16, M, 640, 160, epi, 160, res_cols=8)
    _check(f"{grid} {epi}", out, ref, bound)
    if stats is not None:
        _check_stats(f"{grid} {epi}", stats, out, M)


@pytest.mark.parametrize("dtype", DTYPES, ids=["f16", "bf16"])
@pytest.mark.parametrize("mk", [(1, 320), (129, 64), (1000, 1280), (65600, 320)],
                         ids=["M1_K320", "M129_K64", "M1000_K1280", "M65600_K320"])
def test_geglu_column_slice(cuda_device, mk, dtype):
    """LayerNorm consumer with GEGLU at the packed 256-wide tile, written into fh[:, :Fk] of fh = [M, Fk + C]."""
    from panfusion_b200 import ops
    M, C = mk
    if M == 65600 and dtype == torch.float16:
        pytest.skip("many-wave case: bf16 only")
    Fk = 4 * C if C >= 320 else 640
    g = torch.Generator().manual_seed(M + C)
    dev = cuda_device
    h = _rand(g, (M, C), dev, dtype)
    p = _lin_ln(g, 2 * Fk, C, dev, dtype, geglu_bn=256)
    fh = _nan((M, Fk + C), dtype, dev)
    out = fh[:, :Fk]
    ref, bound = ct.tap_gemm_ref(h, p.w, M, dtype, M=M, Kc=C, bias=p.b, act=GEGLU, ln_eps=p.eps, geglu_bn=256)
    ops.gemm_taps(h, p.w, out, M=M, Kc=C, bias=p.b, act=GEGLU, block_n=256, ln=(_ln_stats(h), p.colsum, p.eps))
    _check(f"GEGLU M={M} C={C}", out, ref, bound)
    assert torch.isnan(fh[:, Fk:].double()).all(), "GEGLU wrote outside its column slice"


@pytest.mark.parametrize("block_n", [128, 160])
def test_producer_to_ln_consumer(cuda_device, block_n):
    """to_out-like GEMM with residual and row statistics, then a q|k|v-like LayerNorm consumer reading those statistics."""
    from panfusion_b200 import ops
    dev, dt = cuda_device, torch.bfloat16
    g = torch.Generator().manual_seed(11)
    M, C = 1000, 320 if block_n == 160 else 256
    x = _rand(g, (M, C), dev, dt)
    w1 = _rand(g, (C, C), dev, dt, scale=C ** -0.5)
    b1 = (torch.randn(C, generator=g) * 0.5).to(dev)
    res = _rand(g, (M, C), dev, dt)
    h = _nan((M, C), dt, dev)
    _, st = ops.gemm_taps(x, w1, h, M=M, Kc=C, bias=b1, residual=res, row_stats=True)
    ref, bound = ct.tap_gemm_ref(x, w1, M, dt, M=M, Kc=C, bias=b1, residual=res)
    _check("producer", h, ref, bound)
    p = _lin_ln(g, 3 * C, C, dev, dt)
    q = _nan((M, 3 * C), dt, dev)
    ops.gemm_taps(h, p.w, q, M=M, Kc=C, bias=p.b, ln=(st, p.colsum, p.eps), block_n=block_n)
    ref, bound = ct.tap_gemm_ref(h, p.w, M, dt, M=M, Kc=C, bias=p.b, ln_eps=p.eps)
    _check("LN consumer of the producer's statistics", q, ref, bound)


def test_repeat_and_graph_replay_byte_identical(cuda_device):
    from panfusion_b200 import ops
    dev, dt = cuda_device, torch.bfloat16
    g = torch.Generator().manual_seed(5)
    M, K, N = 20000, 1600, 320
    A = _rand(g, (M, K), dev, dt)
    B = _rand(g, (N, K), dev, dt, scale=K ** -0.5)
    bias = (torch.randn(N, generator=g) * 0.5).to(dev)
    res = _rand(g, (M, N), dev, dt)
    Fk = 1280
    p = _lin_ln(g, 2 * Fk, N, dev, dt, geglu_bn=256)
    outs = [torch.empty((M, N), dtype=dt, device=dev) for _ in range(2)]
    fhs = [torch.empty((M, Fk), dtype=dt, device=dev) for _ in range(2)]
    stats = [None, None]

    def run(i):
        _, stats[i] = ops.gemm_taps(A, B, outs[i], M=M, Kc=K, bias=bias, residual=res, row_stats=True)
        ops.gemm_taps(outs[i], p.w, fhs[i], M=M, Kc=N, bias=p.b, act=GEGLU, block_n=256,
                      ln=(stats[i], p.colsum, p.eps))

    run(0)
    run(1)
    torch.cuda.synchronize()
    for a, b in ((outs[0], outs[1]), (stats[0], stats[1]), (fhs[0], fhs[1])):
        assert torch.equal(a.view(torch.uint8) if a.dtype != torch.float32 else a.view(torch.int32),
                           b.view(torch.uint8) if b.dtype != torch.float32 else b.view(torch.int32))
    first = [t.clone() for t in (outs[0], stats[0], fhs[0])]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            run(0)
    torch.cuda.current_stream().wait_stream(s)
    for _ in range(2):
        for t in (outs[0], stats[0], fhs[0]):
            t.zero_()
        graph.replay()
        torch.cuda.synchronize()
        for want, got in zip(first, (outs[0], stats[0], fhs[0])):
            assert torch.equal(want.view(torch.int16) if want.dtype != torch.float32 else want.view(torch.int32),
                               got.view(torch.int16) if got.dtype != torch.float32 else got.view(torch.int32))


@pytest.mark.parametrize("block_n", [64, 128, 160])
def test_row_stats_independent_of_m(cuda_device, block_n):
    """Rows [0, M1) of the statistics (and the outputs) are byte-identical for M = M1 and M = 2 M1."""
    from panfusion_b200 import ops
    dev, dt = cuda_device, torch.bfloat16
    g = torch.Generator().manual_seed(3)
    M1, K, N = 4100, 320, 2 * block_n
    A = _rand(g, (2 * M1, K), dev, dt)
    B = _rand(g, (N, K), dev, dt, scale=K ** -0.5)
    res = _rand(g, (2 * M1, N), dev, dt)
    o1, o2 = torch.empty((M1, N), dtype=dt, device=dev), torch.empty((2 * M1, N), dtype=dt, device=dev)
    _, s1 = ops.gemm_taps(A[:M1], B, o1, M=M1, Kc=K, residual=res[:M1], row_stats=True, block_n=block_n)
    _, s2 = ops.gemm_taps(A, B, o2, M=2 * M1, Kc=K, residual=res, row_stats=True, block_n=block_n)
    assert torch.equal(s1.view(torch.int32), s2[:M1].view(torch.int32))
    assert torch.equal(o1.view(torch.int16), o2[:M1].view(torch.int16))
