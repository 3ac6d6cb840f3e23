"""-m gpu: wgmma flash attention (pf_fmha_fwd) against plain PyTorch fp32 softmax(q k^T s + bias) v on the same
16-bit-rounded inputs. The kernel rounds P to the 16-bit type before P V (like every flash kernel), so the
tolerance is one 16-bit ulp of the output scale: fp16 rtol 1e-3 / atol 1e-3; bf16 rtol 8e-3 / atol 8e-3.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


def _ref(q, k, v, heads, d, scale, bias):
    B, Lq, _ = q.shape
    Lk = k.shape[1]
    sp = lambda t, L: t.float().reshape(B, L, heads, d).permute(0, 2, 1, 3)
    s = torch.matmul(sp(q, Lq), sp(k, Lk).transpose(-1, -2)) * scale
    if bias is not None:
        s = s + (bias[:, None] if bias.dim() == 3 else bias[None, None])
    o = torch.matmul(torch.softmax(s, -1), sp(v, Lk))
    return o.permute(0, 2, 1, 3).reshape(B, Lq, heads * d)


CASES = [
    # B, H, Lq, Lk, d, bias
    (2, 5, 256, 256, 64, False),
    (16, 20, 64, 64, 64, False),     # pers 8x8 level: one ragged q tile, one ragged kv tile
    (2, 5, 1024, 77, 64, False),     # text cross attention (77 keys)
    (1, 5, 4096, 4096, 64, False),
    (2, 10, 128, 512, 32, True),     # EPPA dir-1 @ 8x16 pano, 8 views of 8x8
    (2, 10, 512, 128, 32, True),     # EPPA dir-2
    (1, 3, 100, 77, 32, True),       # ragged both ways with bias
    (2, 40, 300, 200, 32, False),
    (1, 10, 2048, 2048, 32, True),
]


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("B,H,Lq,Lk,d,has_bias", CASES)
def test_fmha(cuda_device, dtype, B, H, Lq, Lk, d, has_bias):
    from panfusion_b200 import ops
    g = torch.Generator().manual_seed(B * 1000 + Lq + Lk + d)
    C = H * d
    q = torch.randn(B, Lq, C, generator=g).to(dtype).to(cuda_device)
    k = torch.randn(B, Lk, C, generator=g).to(dtype).to(cuda_device)
    v = torch.randn(B, Lk, C, generator=g).to(dtype).to(cuda_device)
    bias = None
    if has_bias:
        Lk_pad = (Lk + 3) // 4 * 4
        bias_full = (torch.rand(Lq, Lk_pad, generator=g) * 2 - 1).to(cuda_device)
        bias = bias_full[:, :Lk]
    scale = 1.0 / math.sqrt(d)
    ref = _ref(q, k, v, H, d, scale, bias)
    out = torch.empty(B, Lq, C, dtype=dtype, device=cuda_device)
    ops.fmha(q, k, v, out, heads=H, head_dim=d, scale=scale, bias=bias)
    tol = dict(rtol=1e-3, atol=1e-3) if dtype == torch.float16 else dict(rtol=8e-3, atol=8e-3)
    torch.testing.assert_close(out.float(), ref, **tol)


def test_fmha_fused_qkv_views_and_batched_bias(cuda_device):
    """q/k/v as column slices of one [B, L, 3C] buffer; per-batch bias."""
    from panfusion_b200 import ops
    B, H, L, d = 2, 10, 384, 32
    C = H * d
    g = torch.Generator().manual_seed(0)
    qkv = torch.randn(B, L, 3 * C, generator=g).half().to(cuda_device)
    q, k, v = qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
    bias = (torch.rand(B, L, L, generator=g) * 2 - 1).to(cuda_device)
    ref = _ref(q, k, v, H, d, d ** -0.5, bias)
    out = torch.empty(B, L, C, dtype=torch.float16, device=cuda_device)
    ops.fmha(q, k, v, out, heads=H, head_dim=d, scale=d ** -0.5, bias=bias)
    torch.testing.assert_close(out.float(), ref, rtol=1e-3, atol=1e-3)


def test_bias_tile_flags_and_sparse_bias_attention(cuda_device):
    """pf_bias_tile_flags marks 128x64 tiles that are entirely -1; attention with the flag table == without it."""
    from panfusion_b200 import ops
    G, Lq, Lk, H, d = 2, 300, 200, 4, 32
    g = torch.Generator().manual_seed(9)
    bias = torch.full((G, Lq, Lk), -1.0)
    bias[0, 10:40, 70:90] = torch.rand(30, 20, generator=g) * 2 - 1      # touches tiles (0, 1)
    bias[1, 250:300, 0:10] = torch.rand(50, 10, generator=g) * 2 - 1     # touches tiles (1..2, 0)
    bias = bias.to(cuda_device)
    flags = ops.bias_tile_flags(bias)
    assert flags.shape == (G, 3, 4)
    ref = torch.ones(G, 3, 4, dtype=torch.uint8)
    ref[0, 0, 1] = 0
    ref[1, 1, 0] = 0
    ref[1, 2, 0] = 0
    assert torch.equal(flags.cpu(), ref)
    C = H * d
    q = torch.randn(G, Lq, C, generator=g).half().to(cuda_device)
    k = torch.randn(G, Lk, C, generator=g).half().to(cuda_device)
    v = torch.randn(G, Lk, C, generator=g).half().to(cuda_device)
    o1 = torch.empty(G, Lq, C, dtype=torch.float16, device=cuda_device)
    o2 = torch.empty_like(o1)
    ops.fmha(q, k, v, o1, heads=H, head_dim=d, scale=d ** -0.5, bias=bias)
    ops.fmha(q, k, v, o2, heads=H, head_dim=d, scale=d ** -0.5, bias=bias, bias_flags=flags)
    torch.testing.assert_close(o1.float(), o2.float(), rtol=1e-3, atol=1e-3)
    torch.testing.assert_close(o2.float(), _ref(q, k, v, H, d, d ** -0.5, bias), rtol=1e-3, atol=1e-3)


@pytest.mark.parametrize("Lq,Lk,G", [(2048, 8192, 1), (512, 2048, 2), (300, 200, 1), (128, 64, 1)])
def test_tile_packed_bias_equals_dense(cuda_device, Lq, Lk, G):
    """The resident (tile-packed) form of the EPPA bias — only the 128 x 64 tiles that are not entirely -1, plus a tile index
    table — must give exactly the attention output of the dense table (models/modules/transformer.py:57-74 with the mask of
    :68), including ragged edge tiles and per-batch tables."""
    from panfusion_b200 import ops
    B, H, d = max(G, 2) if G > 1 else 2, 3, 32
    B = G if G > 1 else 2
    g = torch.Generator().manual_seed(Lq + Lk)
    bias = torch.full((G, Lq, Lk), -1.0)
    # sparse structure like the correspondence bias: a band of non-constant entries per query row
    for gi in range(G):
        for r in range(0, Lq, 7):
            c0 = (r * 37 + gi * 11) % max(1, Lk - 40)
            bias[gi, r:r + 7, c0:c0 + 40] = torch.rand(min(7, Lq - r), min(40, Lk - c0), generator=g) * 2 - 1
    bias = bias.to(cuda_device)
    store, off = ops.bias_pack_tiles(bias)
    live = int((off >= 0).sum())
    assert store.shape[0] == max(live, 1) and live < off.numel() or Lq <= 300
    # every live tile reproduces the dense tile (zero padding outside), every dropped tile was all -1
    for (gi, qt, kt) in [(0, 0, 0), (G - 1, off.shape[1] - 1, off.shape[2] - 1)]:
        o = int(off[gi, qt, kt])
        dense = bias[gi, qt * 128:(qt + 1) * 128, kt * 64:(kt + 1) * 64]
        if o < 0:
            assert bool((dense == -1).all())
        else:
            assert torch.equal(ops.bias_tile_dense(store[o])[:dense.shape[0], :dense.shape[1]], dense)
    q = torch.randn(B, Lq, H * d, generator=g).bfloat16().to(cuda_device)
    k = torch.randn(B, Lk, H * d, generator=g).bfloat16().to(cuda_device)
    v = torch.randn(B, Lk, H * d, generator=g).bfloat16().to(cuda_device)
    o_dense = torch.empty_like(q)
    o_pack = torch.empty_like(q)
    ops.fmha(q, k, v, o_dense, heads=H, head_dim=d, scale=d ** -0.5, bias=bias, bias_flags=ops.bias_tile_flags(bias))
    ops.fmha(q, k, v, o_pack, heads=H, head_dim=d, scale=d ** -0.5, bias_tiles=(store, off))
    assert torch.equal(o_dense, o_pack)
