"""-m gpu: wgmma tap-GEMM (pf_gemm_taps) against a plain PyTorch fp32 reference of the same contraction.

Inputs are rounded to the 16-bit compute type first, so the only differences are fp32 accumulation order and the
final rounding of the output: tolerance rtol 1e-3 / atol 1e-4 for fp32 outputs (north_star), and one output ulp
(2^-8 bf16, 2^-11 fp16 relative) for 16-bit outputs.
"""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _tol(dtype):
    return dict(rtol=1e-3, atol=1e-4) if dtype == torch.float32 else (
        dict(rtol=2 ** -7, atol=2e-2) if dtype == torch.bfloat16 else dict(rtol=2 ** -10, atol=2e-3))


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("M,N,K,bn", [(300, 320, 640, 0), (128, 64, 64, 64), (1000, 1280, 320, 128),
                                      (257, 640, 1024, 160), (4096, 960, 320, 0)])
def test_linear_plain(cuda_device, dtype, M, N, K, bn):
    from panfusion_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(M + N + K)
    A = torch.randn(M, K, generator=g).to(dtype).to(cuda_device)
    B = (torch.randn(N, K, generator=g) / K ** 0.5).to(dtype).to(cuda_device)
    ref = A.float() @ B.float().T
    out = torch.empty(M, N, dtype=torch.float32, device=cuda_device)
    ops.gemm_taps(A, B, out, M=M, Kc=K, block_n=bn)
    torch.testing.assert_close(out, ref, rtol=1e-3, atol=1e-4)
    out16 = torch.empty(M, N, dtype=dtype, device=cuda_device)
    ops.gemm_taps(A, B, out16, M=M, Kc=K, block_n=bn)
    torch.testing.assert_close(out16.float(), ref, **_tol(dtype))


@pytest.mark.parametrize("act", ["none", "silu", "gelu"])
@pytest.mark.parametrize("res_dtype", [None, torch.float32, torch.bfloat16])
def test_linear_epilogue(cuda_device, act, res_dtype):
    from panfusion_b200 import ops
    M, N, K = 777, 640, 320
    g = torch.Generator(device="cpu").manual_seed(7)
    A = torch.randn(M, K, generator=g).bfloat16().to(cuda_device)
    B = (torch.randn(N, K, generator=g) / K ** 0.5).bfloat16().to(cuda_device)
    bias = torch.randn(N, generator=g).to(cuda_device)
    rowbias = torch.randn(4, N, generator=g).to(cuda_device)
    rpg = 200
    res = None if res_dtype is None else torch.randn(M, N, generator=g).to(res_dtype).to(cuda_device)
    ref = A.float() @ B.float().T + bias + rowbias[(torch.arange(M, device=cuda_device) // rpg)]
    ref = {"none": lambda x: x, "silu": F.silu, "gelu": F.gelu}[act](ref)
    if res is not None:
        ref = ref + res.float()
    out = torch.empty(M, N, dtype=torch.float32, device=cuda_device)
    ops.gemm_taps(A, B, out, M=M, Kc=K, bias=bias, rowbias=rowbias, rows_per_group=rpg, residual=res,
                  act={"none": ops.PF_ACT_NONE, "silu": ops.PF_ACT_SILU, "gelu": ops.PF_ACT_GELU}[act])
    torch.testing.assert_close(out, ref, rtol=1e-3, atol=2e-4)


@pytest.mark.parametrize("bn", [64, 128, 160])
def test_linear_rowbias_direct_store(cuda_device, bn):
    """16-bit output of a row-bias GEMM, which the tap-GEMM's direct-store epilogue writes, at every tile width: bias,
    per-group row bias, SiLU and a 16-bit residual."""
    from panfusion_b200 import ops
    M, N, K = 777, 640, 320
    g = torch.Generator(device="cpu").manual_seed(11)
    A = torch.randn(M, K, generator=g).bfloat16().to(cuda_device)
    B = (torch.randn(N, K, generator=g) / K ** 0.5).bfloat16().to(cuda_device)
    bias = torch.randn(N, generator=g).to(cuda_device)
    rowbias = torch.randn(4, N, generator=g).to(cuda_device)
    rpg = 200
    res = torch.randn(M, N, generator=g).bfloat16().to(cuda_device)
    ref = F.silu(A.float() @ B.float().T + bias + rowbias[(torch.arange(M, device=cuda_device) // rpg)]) + res.float()
    out = torch.empty(M, N, dtype=torch.bfloat16, device=cuda_device)
    ops.gemm_taps(A, B, out, M=M, Kc=K, bias=bias, rowbias=rowbias, rows_per_group=rpg, residual=res,
                  act=ops.PF_ACT_SILU, block_n=bn)
    torch.testing.assert_close(out.float(), ref, **_tol(torch.bfloat16))


@pytest.mark.parametrize("N2", [1280, 2560, 5120])
def test_geglu(cuda_device, N2):
    """GEGLU (models/modules/transformer.py:8-16): proj -> chunk(2) -> x * gelu(gate), at its one tile width (256)
    with a 16-bit output."""
    from panfusion_b200 import ops
    from panfusion_b200.packing import pack_geglu
    M, K = 500, 320
    g = torch.Generator(device="cpu").manual_seed(3)
    A = torch.randn(M, K, generator=g).bfloat16().to(cuda_device)
    W = (torch.randn(N2, K, generator=g) / K ** 0.5).bfloat16()
    b = torch.randn(N2, generator=g)
    y = A.float() @ W.float().T.to(cuda_device) + b.to(cuda_device)
    x, gate = y.chunk(2, dim=-1)
    ref = x * F.gelu(gate)
    assert ops.pick_block_n(N2, ops.PF_ACT_GEGLU) == 256
    Wp, bp = pack_geglu(W, b, 256)
    out = torch.empty(M, N2 // 2, dtype=torch.bfloat16, device=cuda_device)
    ops.gemm_taps(A, Wp.to(cuda_device), out, M=M, Kc=K, bias=bp.to(cuda_device), act=ops.PF_ACT_GEGLU, block_n=256)
    torch.testing.assert_close(out.float(), ref, **_tol(torch.bfloat16))


@pytest.mark.parametrize("n,H,W,Cin,Cout", [(2, 8, 12, 64, 128), (3, 16, 16, 320, 320), (1, 8, 20, 128, 64),
                                            (2, 64, 64, 64, 160)])
def test_conv3x3_taps(cuda_device, n, H, W, Cin, Cout):
    """3x3 / pad 1 convolution as 9 taps over the zero-haloed channels-last image."""
    from panfusion_b200 import ops
    from panfusion_b200.packing import pack_conv3x3
    g = torch.Generator(device="cpu").manual_seed(11)
    x = torch.randn(n, Cin, H, W, generator=g).bfloat16()
    w = (torch.randn(Cout, Cin, 3, 3, generator=g) / (9 * Cin) ** 0.5).bfloat16()
    b = torch.randn(Cout, generator=g)
    ref = F.conv2d(x.float(), w.float(), b, padding=1).to(cuda_device)
    Hp, Wp = H + 2, W + 2
    xp = torch.zeros(n, Hp, Wp, Cin, dtype=torch.bfloat16)
    xp[:, 1:-1, 1:-1] = x.permute(0, 2, 3, 1)
    A = xp.reshape(n * Hp * Wp, Cin).to(cuda_device)
    Bw = pack_conv3x3(w).to(cuda_device)
    taps = [(dy - 1) * Wp + (dx - 1) for dy in range(3) for dx in range(3)]
    out = torch.empty(n * H * W, Cout, dtype=torch.float32, device=cuda_device)
    ops.gemm_taps(A, Bw, out, M=n * Hp * Wp, Kc=Cin, taps=taps, bias=b.to(cuda_device),
                  image_map=(Hp, Wp, 1, 1, H, W))
    got = out.reshape(n, H, W, Cout).permute(0, 3, 1, 2)
    torch.testing.assert_close(got, ref, rtol=1e-3, atol=2e-4)


def test_bad_args_raise(cuda_device):
    from panfusion_b200 import ops
    A = torch.zeros(128, 72, dtype=torch.bfloat16, device=cuda_device)
    B = torch.zeros(64, 72, dtype=torch.bfloat16, device=cuda_device)
    out = torch.zeros(128, 64, dtype=torch.float32, device=cuda_device)
    with pytest.raises(ValueError):
        ops.gemm_taps(A, B, out, M=128, Kc=72)  # Kc not a multiple of 64


@pytest.mark.parametrize("k_splits", [None, 3, 9])
def test_conv3x3_split_k(cuda_device, k_splits):
    """Long-K / few-tile convolution (the 8x8-level shapes): split-K partials + fixed-order reduce == plain path."""
    from panfusion_b200 import ops
    from panfusion_b200.packing import pack_conv3x3
    n, H, W, Cin, Cout = 4, 8, 8, 640, 320
    g = torch.Generator(device="cpu").manual_seed(5)
    x = torch.randn(n, Cin, H, W, generator=g).bfloat16()
    w = (torch.randn(Cout, Cin, 3, 3, generator=g) / (9 * Cin) ** 0.5).bfloat16()
    b = torch.randn(Cout, generator=g)
    temb = torch.randn(n, Cout, generator=g)
    res = torch.randn(n, Cout, H, W, generator=g).bfloat16()
    ref = (F.conv2d(x.float(), w.float(), b, padding=1) + temb[:, :, None, None] + res.float()).to(cuda_device)
    Hp, Wp = H + 2, W + 2
    xp = torch.zeros(n, Hp, Wp, Cin, dtype=torch.bfloat16)
    xp[:, 1:-1, 1:-1] = x.permute(0, 2, 3, 1)
    A = xp.reshape(n * Hp * Wp, Cin).to(cuda_device)
    taps = [(dy - 1) * Wp + (dx - 1) for dy in range(3) for dx in range(3)]
    out = torch.empty(n * H * W, Cout, dtype=torch.float32, device=cuda_device)
    ops.gemm_taps(A, pack_conv3x3(w).to(cuda_device), out, M=n * Hp * Wp, Kc=Cin, taps=taps, bias=b.to(cuda_device),
                  rowbias=temb.to(cuda_device), residual=res.permute(0, 2, 3, 1).reshape(n * H * W, Cout).contiguous().to(cuda_device),
                  image_map=(Hp, Wp, 1, 1, H, W), k_splits=k_splits)
    got = out.reshape(n, H, W, Cout).permute(0, 3, 1, 2)
    torch.testing.assert_close(got, ref, rtol=1e-3, atol=2e-4)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("M,C,N", [(4096 * 10, 320, 960), (300, 640, 640), (130, 1280, 3840), (4096 * 10, 320, 320),
                                   (777, 640, 1920)])
def test_layernorm_fused_into_gemm_pair(cuda_device, dtype, M, C, N):
    """LayerNorm folded around two GEMMs (pf_gemm_args row_stats_out / ln_stats): the producer `x = A W0^T + b0 + res`
    emits per-row (sum, sum^2) partials, the consumer runs on the UN-normalised x with gamma-scaled weights and
    normalises in its epilogue. Reference: fp32 torch LayerNorm(x_16bit) -> Linear, i.e. what the stand-alone
    pf_layernorm + pf_gemm_taps pair computes (diffusers BasicTransformerBlock norm -> to_q|k|v, MVGenModel.py:104)."""
    from panfusion_b200 import ops
    from panfusion_b200.engine import _LinLN
    g = torch.Generator(device="cpu").manual_seed(M + C + N)
    A = torch.randn(M, C, generator=g).to(dtype).to(cuda_device)
    W0 = (torch.randn(C, C, generator=g) / C ** 0.5).to(dtype).to(cuda_device)
    b0 = torch.randn(C, generator=g).to(cuda_device) + 3.0                     # a DC offset: mean >> 0
    res = (torch.randn(M, C, generator=g) * 2).to(dtype).to(cuda_device)
    norm = torch.nn.LayerNorm(C)
    lin = torch.nn.Linear(C, N)
    with torch.no_grad():
        norm.weight.copy_(1 + 0.3 * torch.randn(C, generator=g))
        norm.bias.copy_(0.2 * torch.randn(C, generator=g))
    x = torch.empty(M, C, dtype=dtype, device=cuda_device)
    x, st = ops.gemm_taps(A, W0, x, M=M, Kc=C, bias=b0, residual=res, row_stats=True)
    xf = x.float()
    # producer statistics == sums of the (fp32, pre-rounding) rows: compare with the stored 16-bit rows
    s = st.sum(1)
    eps16 = 2 ** -8 if dtype == torch.bfloat16 else 2 ** -11
    torch.testing.assert_close(s[:, 0], xf.sum(1), rtol=0, atol=eps16 * xf.abs().sum(1).max().item())
    torch.testing.assert_close(s[:, 1], (xf * xf).sum(1), rtol=4 * eps16, atol=1e-3)
    p = _LinLN(lin.weight, lin.bias, norm, cuda_device, dtype)
    out = torch.empty(M, N, dtype=dtype, device=cuda_device)
    ops.gemm_taps(x, p.w, out, M=M, Kc=C, bias=p.b, ln=(st, p.colsum, p.eps))
    ref = F.linear(F.layer_norm(xf, (C,), norm.weight.to(cuda_device), norm.bias.to(cuda_device), norm.eps),
                   lin.weight.to(cuda_device), lin.bias.to(cuda_device))
    # the un-fused path rounds LN(x) to 16 bit before the GEMM; the fused one does not: same error budget
    err = (out.float() - ref).abs().max().item() / ref.abs().max().item()
    print(f"[parity] fused LN->linear {dtype} M={M} C={C} N={N}: max err {err:.2e} of max|ref|")
    assert err < (1.5e-2 if dtype == torch.bfloat16 else 2e-3)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("M,C", [(4096 * 10, 320), (500, 640), (200, 1280)])
def test_layernorm_fused_into_geglu(cuda_device, dtype, M, C):
    """norm3 -> GEGLU projection (diffusers FeedForward; models/modules/transformer.py:8-16,159-160) with the LayerNorm
    folded into the GEGLU epilogue."""
    from panfusion_b200 import ops
    from panfusion_b200.engine import _LinLN
    g = torch.Generator(device="cpu").manual_seed(M + C)
    x = (torch.randn(M, C, generator=g) * 1.5 + 0.7).to(dtype).to(cuda_device)
    W0 = torch.eye(C).to(dtype).to(cuda_device)
    norm = torch.nn.LayerNorm(C)
    lin = torch.nn.Linear(C, 8 * C)
    with torch.no_grad():
        norm.weight.copy_(1 + 0.3 * torch.randn(C, generator=g))
        norm.bias.copy_(0.2 * torch.randn(C, generator=g))
    y = torch.empty(M, C, dtype=dtype, device=cuda_device)
    y, st = ops.gemm_taps(x, W0, y, M=M, Kc=C, row_stats=True)                 # identity producer: y == x
    assert torch.equal(y, x)
    bn = ops.pick_block_n(8 * C, ops.PF_ACT_GEGLU)
    p = _LinLN(lin.weight, lin.bias, norm, cuda_device, dtype, geglu_bn=bn)
    out = torch.empty(M, 4 * C, dtype=dtype, device=cuda_device)
    ops.gemm_taps(y, p.w, out, M=M, Kc=C, bias=p.b, act=ops.PF_ACT_GEGLU, block_n=bn,
                  ln=(st, p.colsum, p.eps))
    h = F.linear(F.layer_norm(x.float(), (C,), norm.weight.to(cuda_device), norm.bias.to(cuda_device), norm.eps),
                 lin.weight.to(cuda_device), lin.bias.to(cuda_device))
    a, gate = h.chunk(2, dim=-1)
    ref = a * F.gelu(gate)
    err = (out.float() - ref).abs().max().item() / ref.abs().max().item()
    print(f"[parity] fused LN->GEGLU {dtype} M={M} C={C}: max err {err:.2e} of max|ref|")
    assert err < (1.5e-2 if dtype == torch.bfloat16 else 2e-3)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("circ", [False, True])
def test_upsample_phase_convolutions(cuda_device, dtype, circ):
    """Upsample2D (nearest x2 -> conv3x3, MVGenModel.py:272-277; panorama: pad_pano(1) -> up -> unpad_pano(2)) as four
    2x2 phase convolutions with scattered output (pf_gemm_args.out_sy/out_sx) == the torch composition, up to the
    rounding of the pre-summed weights."""
    from oracle.eppa import pad_pano
    from panfusion_b200 import engine
    N, C, Co, H, W = 3, 128, 192, 8, 12
    g = torch.Generator().manual_seed(9)
    x = torch.randn(N, C, H, W, generator=g).to(dtype)
    conv = torch.nn.Conv2d(C, Co, 3, padding=1)
    with torch.no_grad():
        conv.weight.copy_(torch.randn(Co, C, 3, 3, generator=g) / (9 * C) ** 0.5)
        conv.bias.copy_(torch.randn(Co, generator=g))
    xs = pad_pano(x.float(), 1) if circ else x.float()
    ref = F.conv2d(F.interpolate(xs, scale_factor=2.0, mode="nearest"), conv.weight, conv.bias, padding=1)
    ref = ref[..., 2:-2] if circ else ref

    class _P:  # the two attributes Branch.upsample reads from its pack
        dt = dtype
    br = engine.Branch.__new__(engine.Branch)
    br.p, br.circ, br.dt = _P(), circ, dtype
    u = engine._Up(conv, cuda_device, dtype)
    o = br.upsample(engine.img_from_nchw(x.to(cuda_device), dtype), u)
    assert (o.N, o.H, o.W) == (N, 2 * H, 2 * W)
    tol = dict(rtol=2 ** -7, atol=3e-2) if dtype == torch.bfloat16 else dict(rtol=2 ** -10, atol=4e-3)
    torch.testing.assert_close(o.nchw().float().cpu(), ref, **tol)
