"""-m gpu: pf_gemm_taps and pf_fmha_fwd at the argument combinations the models pass, against fp64 restatements of the
header contract (tests/_contract.py) with a bound scaled by each element's magnitude.

Every case builds its operands the way the cited call site does (same slicing, image map, scatter, tile width, packers,
`ln=` tuple) at SD-2 widths, with the batch trimmed to 1-2 images. The reference is computed on the device in fp64
from the same 16-bit values the kernel reads. Outputs are pre-filled with NaN, so a write outside the contract's rows
(or columns, for column-slice outputs) fails as well. `test_call_table_covers_the_models` keeps the table honest: a call
class a model forward makes must have a case here."""
import pytest
import torch

import _contract as ct

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]


def _nan(shape, dtype, dev):
    return torch.full(shape, float("nan"), dtype=dtype, device=dev)


def _rand(g, shape, dev, dtype=torch.float32, scale=1.0, offset=0.0):
    return (torch.randn(shape, generator=g) * scale + offset).to(dtype).to(dev)


def _w(g, n, k, dev, dtype):
    return _rand(g, (n, k), dev, dtype, scale=k ** -0.5)


def _ln_stats(x):
    """(sum, sum of squares) of every stored 16-bit row in slot 0, zeros in slot 1: the ln_stats operand the text tower's
    token embedding writes (pf_embed_tokens)."""
    x64 = x.double()
    st = torch.zeros((x.shape[0], 2, 2), dtype=torch.float64, device=x.device)
    st[:, 0, 0], st[:, 0, 1] = x64.sum(1), (x64 * x64).sum(1)
    return st.float().contiguous()


def _lin_ln(g, n, k, dev, dtype, geglu_bn=0):
    from panfusion_b200.engine import _LinLN
    norm = torch.nn.LayerNorm(k)
    with torch.no_grad():
        norm.weight.copy_(1 + 0.3 * torch.randn(k, generator=g))
        norm.bias.copy_(0.2 * torch.randn(k, generator=g))
    return _LinLN(torch.randn(n, k, generator=g) / k ** 0.5, torch.randn(n, generator=g) * 0.5, norm, dev, dtype,
                  geglu_bn=geglu_bn)


def _gemm(checks, name, A, B, out, launches=1, **kw):
    """ops.gemm_taps(A, B, out, **kw) on a NaN-filled `out`, its fp64 reference and bound -> checks[name].
    `launches`: kernels the call must launch (2 = split-K partials + reduce)."""
    from panfusion_b200 import ops
    ref_kw = {k: v for k, v in kw.items() if k not in ("block_n", "ln", "row_stats")}
    if "ln" in kw:
        ref_kw["ln_eps"] = kw["ln"][2]
    if kw.get("act") == ops.PF_ACT_GEGLU:
        ref_kw["geglu_bn"] = kw["block_n"]
    ref, bound = ct.tap_gemm_ref(A, B, out.shape[0], out.dtype, **ref_kw)
    l0 = ops.LAUNCHES
    r = ops.gemm_taps(A, B, out, **kw)
    assert ops.LAUNCHES - l0 == launches, f"{name}: {ops.LAUNCHES - l0} launches, expected {launches}"
    checks.append((name, out, ref, bound))
    return r


# ---- tap-GEMM call table ------------------------------------------------------------------------------------------
# Each case: (call classes it makes, builder). A class is (num_taps, act, image_map given, residual given, fp32 out), the
# key ops.GEMM_LOG records; builders return [(label, got, ref, bound)].

def _conv_operand(g, dev, dt, N, H, W, C, circ=0, phases=1):
    """The tap-GEMM A operand of a convolution, made by pf_conv_prep from random channels-last tokens."""
    from panfusion_b200 import ops
    return ops.conv_prep(_rand(g, (N * H * W, C), dev, dt), N, H, W, circ=circ, phases=phases, halo=1)


def case_temb_mlp(g, dev, dt):
    """Branch.set_timesteps (engine.py:225-229): M = number of images, one partial tile; SiLU 16-bit, then fp32 out."""
    from panfusion_b200 import ops
    n, checks = 2, []
    e0 = _rand(g, (n, 320), dev, dt)
    e1 = _gemm(checks, "te1 silu", e0, _w(g, 1280, 320, dev, dt), _nan((n, 1280), dt, dev), M=n, Kc=320,
               bias=_rand(g, 1280, dev, scale=0.5), act=ops.PF_ACT_SILU)
    e2 = _gemm(checks, "te2 silu", e1, _w(g, 1280, 1280, dev, dt), _nan((n, 1280), dt, dev), M=n, Kc=1280,
               bias=_rand(g, 1280, dev, scale=0.5), act=ops.PF_ACT_SILU)
    _gemm(checks, "temb_all fp32", e2, _w(g, 17600, 1280, dev, dt), _nan((n, 17600), torch.float32, dev), M=n, Kc=1280,
          bias=_rand(g, 17600, dev, scale=0.5))
    return checks


def case_linear_edge_m(g, dev, dt):
    """map_mode 0 at M = 1, 127, 129 (a partial first / last tile), one tile width each: fp32 out + GELU (64),
    16-bit residual + SiLU through the persistent linear GEMM (128), per-group row bias through the tap-GEMM's direct
    stores (160)."""
    from panfusion_b200 import ops
    checks = []
    A = _rand(g, (129, 640), dev, dt)
    B = _w(g, 640, 640, dev, dt)
    bias = _rand(g, 640, dev, scale=0.5)
    _gemm(checks, "M=1 bn64 gelu fp32", A[:1], B, _nan((1, 640), torch.float32, dev), M=1, Kc=640, bias=bias,
          act=ops.PF_ACT_GELU, block_n=64)
    _gemm(checks, "M=127 bn128 silu res16", A[:127], B, _nan((127, 640), dt, dev), M=127, Kc=640, bias=bias,
          residual=_rand(g, (127, 640), dev, dt), act=ops.PF_ACT_SILU, block_n=128)
    _gemm(checks, "M=129 bn160 rowbias", A, B, _nan((129, 640), dt, dev), M=129, Kc=640, bias=bias,
          rowbias=_rand(g, (3, 640), dev, scale=0.5), rows_per_group=64, block_n=160)
    return checks


def _resnet_conv1(checks, g, dev, dt, N, H, W, cin, cout, circ, name, launches=1):
    """Branch.resnet conv1 (engine.py:294): per-image row bias = a column slice of the [N, sum(Cout)] temb table,
    16-bit output over the padded width We."""
    from panfusion_b200.engine import taps3x3
    We = W + 2 * circ
    Hp, Wp = H + 2, We + 2
    a1 = _conv_operand(g, dev, dt, N, H, W, cin, circ=circ)
    temb = _rand(g, (N, 17600), dev, scale=0.5)
    _gemm(checks, name, a1, _w(g, cout, 9 * cin, dev, dt), _nan((N * H * We, cout), dt, dev), launches, M=N * Hp * Wp,
          Kc=cin, taps=taps3x3(Wp), bias=_rand(g, cout, dev, scale=0.5), rowbias=temb[:, 640:640 + cout],
          image_map=(Hp, Wp, 1, 1, H, We))


def _resnet_conv2(checks, g, dev, dt, N, H, W, c, circ, name, launches=1):
    """Branch.resnet / _DecoderBranch.resnet conv2 (engine.py:304, vae.py:101): row map with the panorama crop j0 = 1 + circ,
    16-bit output, 16-bit residual (direct-store epilogue)."""
    from panfusion_b200.engine import taps3x3
    We = W + 2 * circ
    Hp, Wp = H + 2, We + 2
    a2 = _conv_operand(g, dev, dt, N, H, We, c)
    _gemm(checks, name, a2, _w(g, c, 9 * c, dev, dt), _nan((N * H * W, c), dt, dev), launches, M=N * Hp * Wp, Kc=c,
          taps=taps3x3(Wp), bias=_rand(g, c, dev, scale=0.5), residual=_rand(g, (N * H * W, c), dev, dt),
          image_map=(Hp, Wp, 1, 1 + circ, H, W))


def case_resnet_convs(g, dev, dt):
    checks = []
    _resnet_conv1(checks, g, dev, dt, 2, 32, 64, 320, 640, 2, "pano 32x64 conv1 320->640 temb")
    _resnet_conv2(checks, g, dev, dt, 2, 32, 64, 640, 2, "pano 32x64 conv2 640 res16")
    _resnet_conv2(checks, g, dev, dt, 1, 64, 64, 512, 0, "vae 64x64 conv2 512 res16 bn128")
    return checks


def case_resnet_convs_split_k(g, dev, dt):
    """The 8x8 / 8x16-level convolutions at 1280 channels: pf_gemm_splitk_plan splits them, so the reduce kernel applies
    the row bias / residual and makes the 16-bit store (two launches per call)."""
    checks = []
    _resnet_conv1(checks, g, dev, dt, 2, 8, 8, 1280, 1280, 0, "pers 8x8 conv1 1280 temb split-K", launches=2)
    _resnet_conv2(checks, g, dev, dt, 2, 8, 16, 1280, 2, "pano 8x16 conv2 1280 res16 split-K", launches=2)
    return checks


def _strided(checks, g, dev, dt, N, H, W, cin, cout, circ, name, vae=False, act=0):
    """Downsample2D as 9 taps over the four stride-2 phases (engine.py:351 with the panorama crop, engine.py:440 with SiLU,
    vae.py:236 without left / top padding): image map i0 = 0."""
    We = W + 2 * circ
    a = _conv_operand(g, dev, dt, N, H, W, cin, circ=circ, phases=4)
    Ho, Wo = H // 2, We // 2
    Hq, Wq = Ho + 1, Wo + 1
    PS = N * Hq * Wq
    if vae:
        taps = [(((dy + 1) % 2) * 2 + ((dx + 1) % 2)) * PS + ((dy + 1) // 2) * Wq + ((dx + 1) // 2)
                for dy in range(3) for dx in range(3)]
    else:
        taps = [((dy % 2) * 2 + (dx % 2)) * PS + (dy // 2) * Wq + (dx // 2) for dy in range(3) for dx in range(3)]
    crop = 1 if circ else 0
    Wout = Wo - 2 * crop
    _gemm(checks, name, a, _w(g, cout, 9 * cin, dev, dt), _nan((N * Ho * Wout, cout), dt, dev), M=PS, Kc=cin, taps=taps,
          bias=_rand(g, cout, dev, scale=0.5), act=act, image_map=(Hq, Wq, 0, crop, Ho, Wout))


def case_downsamples(g, dev, dt):
    from panfusion_b200 import ops
    checks = []
    _strided(checks, g, dev, dt, 1, 64, 128, 320, 320, 2, "pano 64x128 downsample crop j0=1")
    _strided(checks, g, dev, dt, 1, 64, 64, 256, 256, 0, "vae 64x64 downsample (no left/top pad)", vae=True)
    _strided(checks, g, dev, dt, 1, 128, 128, 128, 256, 0, "controlnet 128x128 downsample silu", act=ops.PF_ACT_SILU)
    return checks


def case_conv_out(g, dev, dt):
    """Branch.conv_out (engine.py:270): 64-wide tile (block_n = 64), fp32 output, panorama crop j0 = 1 + 1."""
    from panfusion_b200.engine import taps3x3
    checks = []
    N, H, W, C, circ = 1, 64, 128, 320, 1
    Hp, Wp = H + 2, W + 2 * circ + 2
    a = _conv_operand(g, dev, dt, N, H, W, C, circ=circ)
    _gemm(checks, "pano 64x128 conv_out fp32 bn64", a, _w(g, 64, 9 * C, dev, dt), _nan((N * H * W, 64), torch.float32, dev),
          M=N * Hp * Wp, Kc=C, taps=taps3x3(Wp), bias=_rand(g, 64, dev, scale=0.5), image_map=(Hp, Wp, 1, 1 + circ, H, W),
          block_n=64)
    return checks


def case_conv_thin_images(g, dev, dt):
    """3x3 convolutions of 1 x W and H x 1 images: every tap of the first and last M-tile reads rows outside the operand."""
    from panfusion_b200.engine import taps3x3
    checks = []
    for N, H, W in ((2, 1, 64), (2, 64, 1)):
        Hp, Wp = H + 2, W + 2
        a = _conv_operand(g, dev, dt, N, H, W, 320)
        _gemm(checks, f"{H}x{W} conv 320 rowbias fp32", a, _w(g, 320, 9 * 320, dev, dt),
              _nan((N * H * W, 320), torch.float32, dev), M=N * Hp * Wp, Kc=320, taps=taps3x3(Wp),
              bias=_rand(g, 320, dev, scale=0.5), rowbias=_rand(g, (N, 320), dev, scale=0.5), image_map=(Hp, Wp, 1, 1, H, W))
    return checks


def case_upsample_phases(g, dev, dt):
    """Branch.upsample (engine.py:367): four 2x2 phase convolutions (engine._Up packing) scattered into one output."""
    from panfusion_b200 import engine, ops
    N, H, W, C, circ = 1, 16, 32, 640, 1
    conv = torch.nn.Conv2d(C, C, 3, padding=1)
    with torch.no_grad():
        conv.weight.copy_(torch.randn(C, C, 3, 3, generator=g) / (9 * C) ** 0.5)
        conv.bias.copy_(torch.randn(C, generator=g) * 0.5)
    u = engine._Up(conv, dev, dt)
    a = _conv_operand(g, dev, dt, N, H, W, C, circ=circ)
    Hp, Wp = H + 2, W + 2 * circ + 2
    out = _nan((N * 2 * H * 2 * W, C), dt, dev)
    parts, k = [], 0
    for pa in (0, 1):
        for pb in (0, 1):
            taps = [(pa + r - 1) * Wp + (pb + cc - 1) for r in (0, 1) for cc in (0, 1)]
            kw = dict(M=N * Hp * Wp, Kc=C, taps=taps, bias=u.b, image_map=(Hp, Wp, 1, 1 + circ, H, W), scatter=(2, 2, pa, pb))
            parts.append(ct.tap_gemm_ref(a, u.phase_w[k], out.shape[0], dt, **kw))
            ops.gemm_taps(a, u.phase_w[k], out, **kw)
            k += 1
    return [("pano 16x32 upsample 640 (4 phases)", out, *ct.merge(parts))]


def case_transformer_tail(g, dev, dt):
    """Transformer2DModel at the 64x64 level (engine.py:331-335): to_out into the column slice fh[:, Fk:] with a 16-bit
    residual and row statistics; the LayerNorm-consumer GEGLU at its production tile width (256) into fh[:, :Fk]; the
    merged ff2 + proj_out GEMM over fh with K = 5C and the block input as residual."""
    from panfusion_b200 import ops
    T, C = 4096, 320
    Fk = 4 * C
    checks = []
    fh = _nan((T, Fk + C), dt, dev)
    h_in = _rand(g, (T, C), dev, dt)
    h, st = _gemm(checks, "to_out -> fh[:, Fk:] res16 row_stats", _rand(g, (T, C), dev, dt), _w(g, C, C, dev, dt),
                  fh[:, Fk:], M=T, Kc=C, bias=_rand(g, C, dev, scale=0.5), residual=h_in, row_stats=True)
    torch.cuda.synchronize()
    assert torch.isnan(fh[:, :Fk]).all(), "to_out wrote outside its column slice"
    # statistics: per-row (sum, sum of squares) of the fp32 values before rounding
    ref, bound = checks[-1][2], checks[-1][3] - ct.ulp_out(checks[-1][2], dt)
    s = st.double().sum(1)
    err_s = (s[:, 0] - ref.sum(1)).abs() / (bound.sum(1) + 2 ** -16 * ref.abs().sum(1))
    err_q = (s[:, 1] - (ref * ref).sum(1)).abs() / ((2 * ref.abs() * bound + bound * bound).sum(1) + 2 ** -16 * (ref * ref).sum(1))
    stats_ratio = max(err_s.max().item(), err_q.max().item())
    bn = ops.pick_block_n(2 * Fk, ops.PF_ACT_GEGLU)
    assert bn == 256
    p = _lin_ln(g, 2 * Fk, C, dev, dt, geglu_bn=bn)
    _gemm(checks, "ff1 LN-consumer GEGLU bn256 -> fh[:, :Fk]", h, p.w, fh[:, :Fk], M=T, Kc=C, bias=p.b,
          act=ops.PF_ACT_GEGLU, block_n=bn, ln=(_ln_stats(h), p.colsum, p.eps))
    x = _rand(g, (T, C), dev, dt)
    _gemm(checks, "tail K=5C res16", fh, _w(g, C, Fk + C, dev, dt), _nan((T, C), dt, dev), M=T, Kc=Fk + C,
          bias=_rand(g, C, dev, scale=0.5), residual=x)
    checks.append(("to_out row statistics (fp32)", None, stats_ratio, None))
    return checks


def case_geglu_ln_1280_and_eppa(g, dev, dt):
    """LayerNorm-consumer GEGLU at C = 1280 (16x16 level, 10240 projection columns) and in the EPPA block tail
    (eppa.py:85: rows of one small pano level, plain [rows, 4C] output)."""
    from panfusion_b200 import ops
    checks = []
    for T, C, name in ((2 * 256, 1280, "unet 16x16 C=1280"), (128, 320, "eppa 8x16 C=320")):
        bn = ops.pick_block_n(8 * C, ops.PF_ACT_GEGLU)
        p = _lin_ln(g, 8 * C, C, dev, dt, geglu_bn=bn)
        x = _rand(g, (T, C), dev, dt, scale=1.5, offset=0.7)
        _gemm(checks, f"{name} LN GEGLU bn{bn}", x, p.w, _nan((T, 4 * C), dt, dev), M=T, Kc=C, bias=p.b,
              act=ops.PF_ACT_GEGLU, block_n=bn, ln=(_ln_stats(x), p.colsum, p.eps))
    return checks


def case_text_tower(g, dev, dt):
    """CLIP text layer (text_encoder.py:103,108) at SD-2's width: 2 x 77 tokens (a ragged second tile), LayerNorm
    consumers without activation (q|k|v) and with GELU (fc1); then the text K/V of every cross-attention layer
    (engine.py:248)."""
    from panfusion_b200 import ops
    checks = []
    T, C = 2 * 77, 1024
    x = _rand(g, (T, C), dev, dt, scale=1.5, offset=0.3)
    st = _ln_stats(x)
    p = _lin_ln(g, 3 * C, C, dev, dt)
    _gemm(checks, "qkv LN-consumer", x, p.w, _nan((T, 3 * C), dt, dev), M=T, Kc=C, bias=p.b, ln=(st, p.colsum, p.eps))
    p = _lin_ln(g, 4 * C, C, dev, dt)
    _gemm(checks, "fc1 LN-consumer GELU", x, p.w, _nan((T, 4 * C), dt, dev), M=T, Kc=C, bias=p.b, act=ops.PF_ACT_GELU,
          ln=(st, p.colsum, p.eps))
    _gemm(checks, "kv_all (24960 columns)", x, _w(g, 24960, C, dev, dt), _nan((T, 24960), dt, dev), M=T, Kc=C)
    return checks


def case_vae_attention(g, dev, dt):
    """_DecoderBranch.attention (vae.py:123-126) at the 64x64 latent: Q K^T with B a column slice of the fused q|k buffer
    (b_ld = 2C > K) and N = L tokens into fp32 logits; V^T = W_v X^T; P V with K = L."""
    checks = []
    L, Cc = 4096, 512
    qk = _rand(g, (L, 2 * Cc), dev, dt, scale=0.25)
    _gemm(checks, "Q K^T (B = column slice) fp32", qk[:, :Cc], qk[:, Cc:], _nan((L, L), torch.float32, dev), M=L, Kc=Cc)
    xn = _rand(g, (L, Cc), dev, dt)
    vt = _gemm(checks, "V^T = W_v X^T", _w(g, Cc, Cc, dev, dt), xn, _nan((Cc, L), dt, dev), M=Cc, Kc=Cc)
    probs = torch.softmax(torch.randn(L, L, generator=g) * 3, -1).to(dt).to(dev)
    _gemm(checks, "P V (K = L)", probs, vt, _nan((L, Cc), dt, dev), M=L, Kc=L)
    return checks


GEMM_CASES = {
    "temb_mlp": ({(1, 1, False, False, False), (1, 0, False, False, True)}, case_temb_mlp),
    "linear_edge_m": ({(1, 2, False, False, True), (1, 1, False, True, False), (1, 0, False, False, False)},
                      case_linear_edge_m),
    "resnet_convs": ({(9, 0, True, False, False), (9, 0, True, True, False)}, case_resnet_convs),
    "resnet_convs_split_k": ({(9, 0, True, False, False), (9, 0, True, True, False)}, case_resnet_convs_split_k),
    "downsamples": ({(9, 0, True, False, False), (9, 1, True, False, False)}, case_downsamples),
    "conv_out": ({(9, 0, True, False, True)}, case_conv_out),
    "conv_thin_images": ({(9, 0, True, False, True)}, case_conv_thin_images),
    "upsample_phases": ({(4, 0, True, False, False)}, case_upsample_phases),
    "transformer_tail": ({(1, 0, False, True, False), (1, 3, False, False, False)}, case_transformer_tail),
    "geglu_ln_1280_and_eppa": ({(1, 3, False, False, False)}, case_geglu_ln_1280_and_eppa),
    "text_tower": ({(1, 0, False, False, False), (1, 2, False, False, False)}, case_text_tower),
    "vae_attention": ({(1, 0, False, False, True), (1, 0, False, False, False)}, case_vae_attention),
}


def _call_class(entry):
    """GEMM_LOG entry (M, N, Kc, num_taps, act, image_map given, residual given, fp32 out) -> call class."""
    return (entry[3], entry[4], entry[5], entry[6], entry[7])


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", list(GEMM_CASES))
def test_gemm_contract(cuda_device, case, dtype):
    from panfusion_b200 import ops
    classes, build = GEMM_CASES[case]
    g = torch.Generator().manual_seed(sum(map(ord, case)))
    ops.GEMM_LOG = []
    try:
        checks = build(g, cuda_device, dtype)
        logged = {_call_class(e) for e in ops.GEMM_LOG}
    finally:
        ops.GEMM_LOG = None
    assert logged == classes, f"the case makes calls of classes {logged}, declared {classes}"
    torch.cuda.synchronize()
    worst = 0.0
    for name, got, ref, bound in checks:
        r = ref if got is None else ct.worst_ratio(got, ref, bound)  # (name, None, ratio, None): checked by the builder
        print(f"[contract] gemm {case} / {name} {dtype}: worst err/bound {r:.3f}")
        worst = max(worst, r)
    assert worst <= 1.0, worst


def test_call_table_covers_the_models(cuda_device):
    """Every tap-GEMM call class of a tiny-config MultiViewBaseModel forward has a case in GEMM_CASES."""
    from oracle import unet as ou
    from panfusion_b200 import ops
    from test_gpu_mvgen import _run_mvgen
    ops.GEMM_LOG = []
    try:
        _run_mvgen(cuda_device, ou.TINY_CONFIG, (16, 32), (16, 16), torch.float16)
        seen = {_call_class(e) for e in ops.GEMM_LOG}
    finally:
        ops.GEMM_LOG = None
    covered = set().union(*(c for c, _ in GEMM_CASES.values()))
    assert seen, "the forward made no tap-GEMM call"
    assert seen <= covered, f"call classes without a contract case: {sorted(seen - covered)}"


# ---- flash-attention call table -----------------------------------------------------------------------------------

def _sparse_bias(g, G, Lq, Lk, dev):
    """An EPPA-like bias: -1 everywhere but a band of random entries per block of query rows."""
    bias = torch.full((G, Lq, Lk), -1.0)
    for gi in range(G):
        for r in range(0, Lq, 16):
            c0 = (r * 37 + gi * 11) % max(1, Lk - 48)
            bias[gi, r:r + 16, c0:c0 + 48] = torch.rand(min(16, Lq - r), min(48, Lk - c0), generator=g) * 2 - 1
    return bias.to(dev)


def fcase_self_attention(g, dev, dt):
    """engine.py:323: q / k / v column slices of the fused [N, L, 3C] buffer, 64x64 level, d = 64."""
    L, C = 4096, 320
    qkv = _rand(g, (1, L, 3 * C), dev, dt)
    return (qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]), dict(heads=5, head_dim=64, scale=64 ** -0.5)


def fcase_cross_attention(g, dev, dt):
    """engine.py:327: K / V column slices (at kv_off) of the hoisted [N, 77, sum(2C)] text K/V of every layer."""
    L, C, kv_off = 1024, 640, 1280
    kv = _rand(g, (2, 77, 24960), dev, dt)
    q = _rand(g, (2, L, C), dev, dt)
    return (q, kv[..., kv_off:kv_off + C], kv[..., kv_off + C:kv_off + 2 * C]), dict(heads=10, head_dim=64, scale=64 ** -0.5)


def fcase_eppa_dir1_packed(g, dev, dt):
    """eppa.py:314: pano queries (16x32) over two 16x16 views' keys, tile-packed bias (ops.bias_pack_tiles), d = 32."""
    from panfusion_b200 import ops
    C, E, mP = 320, 512, 512
    qkv_e, qkv_p = _rand(g, (1, E, 3 * C), dev, dt), _rand(g, (1, mP, 3 * C), dev, dt)
    bias = _sparse_bias(g, 1, E, mP, dev)
    return ((qkv_e[..., :C], qkv_p[..., C:2 * C], qkv_p[..., 2 * C:]),
            dict(heads=10, head_dim=32, scale=32 ** -0.5, bias_tiles=ops.bias_pack_tiles(bias)), bias)


def fcase_eppa_dir2_small(g, dev, dt):
    """eppa.py:318 at the smallest level: one 8x8 view queries (Lq = 64 < 128) over an 8x16 pano, dense bias + flags."""
    from panfusion_b200 import ops
    C, P, E = 320, 64, 128
    qkv_p, qkv_e = _rand(g, (1, P, 3 * C), dev, dt), _rand(g, (1, E, 3 * C), dev, dt)
    bias = _sparse_bias(g, 1, P, E, dev)
    return ((qkv_p[..., :C], qkv_e[..., C:2 * C], qkv_e[..., 2 * C:]),
            dict(heads=10, head_dim=32, scale=32 ** -0.5, bias=bias, bias_flags=ops.bias_tile_flags(bias)))


def fcase_per_batch_bias_flags(g, dev, dt):
    """A per-batch [2, Lq, Lk] bias with its per-batch tile flags (B = 2), ragged in both directions."""
    from panfusion_b200 import ops
    C, Lq, Lk = 320, 300, 200
    q, k, v = (_rand(g, (2, L, C), dev, dt) for L in (Lq, Lk, Lk))
    bias = _sparse_bias(g, 2, Lq, Lk, dev)
    return (q, k, v), dict(heads=10, head_dim=32, scale=32 ** -0.5, bias=bias, bias_flags=ops.bias_tile_flags(bias))


FMHA_CASES = {
    "self_attention": fcase_self_attention,
    "cross_attention": fcase_cross_attention,
    "eppa_dir1_packed": fcase_eppa_dir1_packed,
    "eppa_dir2_small": fcase_eppa_dir2_small,
    "per_batch_bias_flags": fcase_per_batch_bias_flags,
}


def _fmha_check(q, k, v, kw, dense_bias, dt, name):
    from panfusion_b200 import ops
    B, Lq = q.shape[:2]
    out = _nan((B, Lq, kw["heads"] * kw["head_dim"]), dt, q.device)
    ops.fmha(q, k, v, out, **kw)
    ref, pv = ct.fmha_ref(q, k, v, heads=kw["heads"], head_dim=kw["head_dim"], scale=kw["scale"], bias=dense_bias)
    r = ct.worst_ratio(out, ref, ct.fmha_bound(ref, pv, dt))
    print(f"[contract] fmha {name} {dt}: worst err/bound {r:.3f}")
    assert r <= 1.0, r


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", list(FMHA_CASES))
def test_fmha_contract(cuda_device, case, dtype):
    g = torch.Generator().manual_seed(sum(map(ord, case)))
    built = FMHA_CASES[case](g, cuda_device, dtype)
    (q, k, v), kw = built[0], built[1]
    dense = built[2] if len(built) > 2 else kw.get("bias")
    _fmha_check(q, k, v, kw, dense, dtype, case)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("has_bias", [False, True])
@pytest.mark.parametrize("Lk", [1, 63, 65])
@pytest.mark.parametrize("Lq", [1, 127, 129])
def test_fmha_contract_ragged_edges(cuda_device, Lq, Lk, has_bias, dtype):
    """One query / key, one short of a 128-query / 64-key tile and one past it; d = 64 and 32 alternate."""
    d = 64 if (Lq + Lk) % 4 == 2 else 32
    g = torch.Generator().manual_seed(Lq * 100 + Lk)
    H = 2
    q, k, v = (_rand(g, (1, L, H * d), cuda_device, dtype) for L in (Lq, Lk, Lk))
    kw = dict(heads=H, head_dim=d, scale=d ** -0.5)
    if has_bias:  # rows padded to the 4-float alignment the kernel's vector loads need
        kw["bias"] = _rand(g, (Lq, (Lk + 3) // 4 * 4), cuda_device)[:, :Lk]
    _fmha_check(q, k, v, kw, kw.get("bias"), dtype, f"Lq={Lq} Lk={Lk} d={d} bias={has_bias}")
