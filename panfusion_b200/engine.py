"""Host-side engine: packs the weights of a duck-typed SD-2 `UNet2DConditionModel` once and runs its blocks as
sequences of C-ABI kernel launches on channels-last 16-bit activations.

The reference never calls `unet.forward`; it walks the sub-modules (models/pano/MVGenModel.py:52-295). This file is
the per-sub-module replacement for that walk: `resnet`, `transformer`, `downsample`, `upsample`, `conv_in`,
`conv_out` take and return `Img` activations ([N*H*W, C] tokens) and issue only `panfusion_b200.ops` calls.
Semantics follow diffusers 0.24.0 ResnetBlock2D / Transformer2DModel / Downsample2D / Upsample2D [3P] with the
panorama branch's circular padding (utils/pano.py:74-105) folded into the kernels.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import torch
from torch import Tensor

from . import ops
from .packing import pack_conv3x3, pack_geglu, pack_upsample_phases


@dataclass
class Img:
    """Channels-last activation: t is [N*H*W, C] (row stride may exceed C)."""
    t: Tensor
    N: int
    H: int
    W: int

    @property
    def C(self) -> int:
        return self.t.shape[1]

    def nchw(self) -> Tensor:
        return self.t.reshape(self.N, self.H, self.W, self.C).permute(0, 3, 1, 2)


def img_from_nchw(x: Tensor, dtype: torch.dtype) -> Img:
    n, c, h, w = x.shape
    return Img(x.permute(0, 2, 3, 1).reshape(n * h * w, c).to(dtype).contiguous(), n, h, w)


def taps3x3(row_pitch: int) -> list[int]:
    return [(dy - 1) * row_pitch + (dx - 1) for dy in range(3) for dx in range(3)]


class _Lin:
    """Packed nn.Linear / 1x1 conv: W [N, K] 16-bit, bias fp32."""

    def __init__(self, w: Tensor, b: Optional[Tensor], dev, dt):
        self.w = w.detach().reshape(w.shape[0], -1).to(dev, dt).contiguous()
        self.b = b.detach().to(dev, torch.float32).contiguous() if b is not None else None
        self.n, self.k = self.w.shape


class _LinLN:
    """nn.Linear applied to LayerNorm(x): W' = gamma * W (16-bit), colsum[n] = sum_k W'[n,k] of the ROUNDED weights (so the
    mean term cancels exactly), bias' = W beta + b. `geglu_bn` packs W' for the GEGLU epilogue (value|gate per tile)."""

    def __init__(self, w: Tensor, b: Optional[Tensor], norm, dev, dt, geglu_bn: int = 0):
        w64 = w.detach().double().reshape(w.shape[0], -1)
        g, be = norm.weight.detach().double().to(w64.device), norm.bias.detach().double().to(w64.device)
        wp = (w64 * g[None, :]).float()
        bp = (w64 @ be + (b.detach().double() if b is not None else 0.0)).float()
        if geglu_bn:
            wp, bp = pack_geglu(wp, bp, geglu_bn)
        self.w = wp.to(dev, dt).contiguous()
        self.b = bp.to(dev, torch.float32).contiguous()
        self.colsum = self.w.float().sum(1).contiguous()
        self.eps = float(norm.eps)
        self.n, self.k = self.w.shape


class _Norm:
    def __init__(self, mod, dev):
        self.g = mod.weight.detach().to(dev, torch.float32).contiguous()
        self.b = mod.bias.detach().to(dev, torch.float32).contiguous()
        self.eps = float(mod.eps)
        self.groups = int(getattr(mod, "num_groups", 0))


class _Conv3:
    def __init__(self, conv, dev, dt):
        self.w = pack_conv3x3(conv.weight.detach()).to(dev, dt).contiguous()
        self.b = conv.bias.detach().to(dev, torch.float32).contiguous() if conv.bias is not None else None
        self.cout, self.cin = conv.weight.shape[0], conv.weight.shape[1]


class _Up:
    """Upsample2D (nearest x2 + 3x3 conv) as four 2x2 phase convolutions of the original-resolution image (2.25x fewer
    MACs, no up-sampled copy)."""

    def __init__(self, conv, dev, dt):
        self.phase_w = [w.to(dev, dt).contiguous() for w in pack_upsample_phases(conv.weight)]
        self.b = conv.bias.detach().to(dev, torch.float32).contiguous() if conv.bias is not None else None
        self.cout, self.cin = conv.weight.shape[0], conv.weight.shape[1]


class _Resnet:
    def __init__(self, r, dev, dt):
        self.norm1, self.norm2 = _Norm(r.norm1, dev), _Norm(r.norm2, dev)
        self.conv1, self.conv2 = _Conv3(r.conv1, dev, dt), _Conv3(r.conv2, dev, dt)
        self.short = _Lin(r.conv_shortcut.weight, r.conv_shortcut.bias, dev, dt) if getattr(r, "conv_shortcut", None) is not None else None
        self.temb_off = -1  # column offset into the per-forward temb projection table


class _Transformer:
    def __init__(self, t, dev, dt):
        blk = t.transformer_blocks[0]
        assert len(t.transformer_blocks) == 1
        self.norm = _Norm(t.norm, dev)
        self.proj_in = _Lin(t.proj_in.weight, t.proj_in.bias, dev, dt)
        self.heads = int(blk.attn1.heads)
        a1, a2 = blk.attn1, blk.attn2
        self.out1 = _Lin(a1.to_out[0].weight, a1.to_out[0].bias, dev, dt)
        self.kv2_w = torch.cat([a2.to_k.weight, a2.to_v.weight], 0).detach()  # merged across layers by UNetPack
        self.out2 = _Lin(a2.to_out[0].weight, a2.to_out[0].bias, dev, dt)
        self.kv_off = -1
        ff1, ff2 = blk.ff.net[0].proj, blk.ff.net[2]
        self.ff1_bn = ops.pick_block_n(ff1.weight.shape[0], ops.PF_ACT_GEGLU)
        self.ff_dim = ff2.weight.shape[1]  # 4C
        # ff2 and proj_out back to back are ONE linear map of [f | h]: proj_out(ff2(f) + h) = f (Wp W2)^T + h Wp^T + (Wp b2 + bp).
        # The GEGLU output f and the residual stream h are written side by side ([T, 4C | C]), so the tail of the block is a
        # single GEMM with K = 5C (same MACs, one launch and one [T, C] round trip through HBM less).
        wp, w2 = t.proj_out.weight.detach().double().flatten(1), ff2.weight.detach().double()
        self.tail = _Lin(torch.cat([wp @ w2, wp], 1).float(),
                         (wp @ ff2.bias.detach().double() + t.proj_out.bias.detach().double()).float(), dev, dt)
        self.C = self.proj_in.n
        # the three LayerNorms folded into their consumer GEMMs
        self.qkv_ln = _LinLN(torch.cat([a1.to_q.weight, a1.to_k.weight, a1.to_v.weight], 0), None, blk.norm1, dev, dt)
        self.q2_ln = _LinLN(a2.to_q.weight, None, blk.norm2, dev, dt)
        self.ff1_ln = _LinLN(ff1.weight, ff1.bias, blk.norm3, dev, dt, geglu_bn=self.ff1_bn)


class UNetPack:
    """All weights of one UNet, packed for the kernels; built once per (device, dtype)."""

    def __init__(self, unet, dev, dt, encoder_only: bool = False):
        """encoder_only: a ControlNet (conv_in, time embedding, down_blocks, mid_block; no decoder / conv_out)."""
        self.dev, self.dt = dev, dt
        self.groups = int(unet.down_blocks[0].resnets[0].norm1.num_groups)
        f32 = lambda t: t.detach().to(dev, torch.float32).contiguous()
        self.conv_in_w, self.conv_in_b = f32(unet.conv_in.weight), f32(unet.conv_in.bias)
        if not encoder_only:
            # conv_out (C -> 4) on the tensor cores: output channels zero-padded to one 64-wide tap-GEMM tile
            co = unet.conv_out.weight.shape[0]
            wpad = torch.zeros((64, *unet.conv_out.weight.shape[1:]), dtype=unet.conv_out.weight.dtype,
                               device=unet.conv_out.weight.device)
            wpad[:co] = unet.conv_out.weight.detach()
            self.conv_out_packed = pack_conv3x3(wpad).to(dev, dt).contiguous()
            bpad = torch.zeros(64, dtype=torch.float32, device=dev)
            bpad[:co] = f32(unet.conv_out.bias)
            self.conv_out_bpad, self.conv_out_c = bpad, co
            self.norm_out = _Norm(unet.conv_norm_out, dev)
        te = unet.time_embedding
        self.t_dim = te.linear_1.weight.shape[1]
        self.te1, self.te2 = _Lin(te.linear_1.weight, te.linear_1.bias, dev, dt), _Lin(te.linear_2.weight, te.linear_2.bias, dev, dt)
        self.resnets: list[_Resnet] = []
        self.transformers: list[_Transformer] = []

        def res(r):
            p = _Resnet(r, dev, dt)
            p._src = r
            self.resnets.append(p)
            return p

        def tr(t):
            p = _Transformer(t, dev, dt)
            self.transformers.append(p)
            return p

        self.down = []
        for blk in unet.down_blocks:
            has_attn = bool(getattr(blk, "has_cross_attention", False))
            self.down.append(dict(
                resnets=[res(r) for r in blk.resnets],
                attns=[tr(t) for t in blk.attentions] if has_attn else None,
                down=[_Conv3(d.conv, dev, dt) for d in blk.downsamplers] if blk.downsamplers is not None else None))
        self.mid = dict(resnets=[res(r) for r in unet.mid_block.resnets], attns=[tr(t) for t in unet.mid_block.attentions])
        self.up = []
        for blk in ([] if encoder_only else unet.up_blocks):
            has_attn = bool(getattr(blk, "has_cross_attention", False))
            self.up.append(dict(
                resnets=[res(r) for r in blk.resnets],
                attns=[tr(t) for t in blk.attentions] if has_attn else None,
                up=[_Up(u.conv, dev, dt) for u in blk.upsamplers] if blk.upsamplers is not None else None))
        # one GEMM for every ResnetBlock2D.time_emb_proj (applied to silu(temb))
        off, ws, bs = 0, [], []
        for p in self.resnets:
            p.temb_off = off
            ws.append(p._src.time_emb_proj.weight.detach())
            bs.append(p._src.time_emb_proj.bias.detach())
            off += p.conv1.cout
            del p._src
        self.temb_all = _Lin(torch.cat(ws, 0), torch.cat(bs, 0), dev, dt)
        # one GEMM for every text cross-attention K/V projection
        off, ws = 0, []
        for t in self.transformers:
            t.kv_off = off
            ws.append(t.kv2_w)
            off += t.kv2_w.shape[0]
            del t.kv2_w
        self.kv_all = _Lin(torch.cat(ws, 0), None, dev, dt) if ws else None


class Branch:
    """One UNet branch (perspective or panorama) bound to its per-forward context (temb table, text K/V)."""

    def __init__(self, pack: UNetPack, circular: bool):
        self.p = pack
        self.circ = circular  # panorama branch with pano_pad=True
        self.dt = pack.dt
        self.temb: Optional[Tensor] = None   # [N, sum(Cout)] fp32
        self.text_kv: Optional[Tensor] = None  # [N, 77, sum(2C)]
        self._text_key = None

    # ---- per-forward context ---------------------------------------------------------------------
    def set_timesteps(self, t: Tensor) -> None:
        """time_proj -> time_embedding -> every time_emb_proj(silu(.)) (MVGenModel.py:52-60 + ResnetBlock2D)."""
        p = self.p
        t = t.reshape(-1).to(torch.float32)
        n = t.numel()
        e0 = ops.timestep_embed(t, p.t_dim, self.dt)
        e1 = torch.empty((n, p.te1.n), dtype=self.dt, device=p.dev)
        ops.gemm_taps(e0, p.te1.w, e1, M=n, Kc=p.te1.k, bias=p.te1.b, act=ops.PF_ACT_SILU)
        e2 = torch.empty((n, p.te2.n), dtype=self.dt, device=p.dev)
        ops.gemm_taps(e1, p.te2.w, e2, M=n, Kc=p.te2.k, bias=p.te2.b, act=ops.PF_ACT_SILU)  # = silu(temb)
        self.temb = torch.empty((n, p.temb_all.n), dtype=torch.float32, device=p.dev)
        ops.gemm_taps(e2, p.temb_all.w, self.temb, M=n, Kc=p.temb_all.k, bias=p.temb_all.b)

    def set_text(self, prompt: Tensor, key=None) -> None:
        """prompt [N, L, ctx] -> K/V of every cross-attention layer. The text does not change across denoising steps
        (PanFusion.py:134-138 embeds it once), so the result is cached on the identity + version of the caller's
        tensor (`key`, taken before any slicing/reshaping). In-place edits — also through views, which share the base's
        version counter — invalidate the entry; only writes through `.data` bypass version tracking (PyTorch-wide caveat):
        call `MultiViewBaseModel.update_text` / `invalidate()` after such a write."""
        key = key if key is not None else (prompt.data_ptr(), prompt._version, tuple(prompt.shape))
        if key == self._text_key:
            return
        p = self.p
        n, L, ctx = prompt.shape
        x = prompt.reshape(n * L, ctx).to(self.dt).contiguous()
        # a new text of the same shape is projected INTO the existing buffer: captured CUDA graphs read it by address
        if self.text_kv is not None and tuple(self.text_kv.shape) == (n, L, p.kv_all.n):
            kv = self.text_kv.reshape(n * L, p.kv_all.n)
        else:
            kv = torch.empty((n * L, p.kv_all.n), dtype=self.dt, device=p.dev)
        ops.gemm_taps(x, p.kv_all.w, kv, M=n * L, Kc=ctx)
        self.text_kv = kv.reshape(n, L, p.kv_all.n)
        self._text_key = key
        # the key is the tensor's IDENTITY (address, version): hold the storage so that the address cannot be handed
        # to a different tensor while this entry is alive
        self._text_owner = prompt

    # ---- blocks ------------------------------------------------------------------------------------
    def conv_in(self, latent: Tensor) -> Img:
        n, _, h, w = latent.shape
        t = ops.conv_in(latent.to(torch.float32).contiguous(), self.p.conv_in_w, self.p.conv_in_b, self.dt, self.circ)
        return Img(t, n, h, w)

    def conv_out(self, x: Img) -> Tensor:
        p = self.p
        c = 1 if self.circ else 0
        xp = self._norm_prep(x.t, x.N, x.H, x.W, p.norm_out, act=ops.PF_ACT_SILU, circ_stats=0, circ=c,
                             halo=1)  # statistics of the un-padded tensor (MVGenModel.py:288)
        # 3x3 conv as 9 taps (the 64-column tile holds the 4 real output channels + zero padding), fp32 out
        We = x.W + 2 * c
        Hp, Wp = x.H + 2, We + 2
        o = torch.empty((x.N * x.H * x.W, 64), dtype=torch.float32, device=x.t.device)
        ops.gemm_taps(xp, p.conv_out_packed, o, M=x.N * Hp * Wp, Kc=x.C, taps=taps3x3(Wp), bias=p.conv_out_bpad,
                      image_map=(Hp, Wp, 1, 1 + c, x.H, x.W), block_n=64)
        return o[:, :p.conv_out_c].reshape(x.N, x.H, x.W, p.conv_out_c).permute(0, 3, 1, 2).contiguous()

    def _norm_prep(self, xt: Tensor, N: int, H: int, W: int, norm: _Norm, *, act: int, circ_stats: int, circ: int,
                   halo: int) -> Tensor:
        """GroupNorm (+SiLU) of a token tensor into the tap-GEMM A layout."""
        return ops.gn_prep(xt, N, H, W, gamma=norm.g, beta=norm.b, groups=self.p.groups, eps=norm.eps, act=act,
                           circ_stats=circ_stats, circ=circ, halo=halo)

    def resnet(self, x: Img, r: _Resnet, skip: Optional[Img] = None) -> Img:
        """ResnetBlock2D; panorama: pad_pano(2) -> block -> unpad_pano(2) (MVGenModel.py:110-115). `skip`: the decoder's
        torch.cat([hidden, skip], dim=1) input (MVGenModel.py:223,231,246,254)."""
        c = 2 if self.circ else 0
        N, H, W = x.N, x.H, x.W
        We = W + 2 * c
        xt = x.t
        if skip is not None:  # torch.cat([hidden, skip], 1) (MVGenModel.py:223,231): folded into the norm1 launches
            a1, xt = ops.gn_prep(x.t, N, H, W, gamma=r.norm1.g, beta=r.norm1.b, groups=self.p.groups, eps=r.norm1.eps,
                                 act=ops.PF_ACT_SILU, circ_stats=c, circ=c, halo=1, x2=skip.t, want_cat=True)
        else:
            a1 = self._norm_prep(xt, N, H, W, r.norm1, act=ops.PF_ACT_SILU, circ_stats=c, circ=c, halo=1)
        Hp, Wp = H + 2, We + 2
        h1 = torch.empty((N * H * We, r.conv1.cout), dtype=self.dt, device=x.t.device)
        ops.gemm_taps(a1, r.conv1.w, h1, M=N * Hp * Wp, Kc=r.conv1.cin, taps=taps3x3(Wp), bias=r.conv1.b,
                      rowbias=self.temb[:, r.temb_off:r.temb_off + r.conv1.cout], image_map=(Hp, Wp, 1, 1, H, We))
        # norm2 sees the padded-width tensor, borders included
        a2 = self._norm_prep(h1, N, H, We, r.norm2, act=ops.PF_ACT_SILU, circ_stats=0, circ=0, halo=1)
        if r.short is not None:
            res = torch.empty((N * H * W, r.short.n), dtype=self.dt, device=x.t.device)
            ops.gemm_taps(xt, r.short.w, res, M=N * H * W, Kc=r.short.k, bias=r.short.b)
        else:
            res = xt
        out = torch.empty((N * H * W, r.conv2.cout), dtype=self.dt, device=x.t.device)
        ops.gemm_taps(a2, r.conv2.w, out, M=N * Hp * Wp, Kc=r.conv2.cin, taps=taps3x3(Wp), bias=r.conv2.b,
                      residual=res, image_map=(Hp, Wp, 1, 1 + c, H, W))
        return Img(out, N, H, W)

    def transformer(self, x: Img, t: _Transformer) -> Img:
        """Transformer2DModel (GroupNorm -> proj_in -> self-attn -> text cross-attn -> GEGLU FF -> proj_out + x)."""
        N, H, W, C = x.N, x.H, x.W, t.C
        L, T = H * W, N * H * W
        dev, dt = x.t.device, self.dt
        new = lambda n: torch.empty((T, n), dtype=dt, device=dev)
        xn = self._norm_prep(x.t, N, H, W, t.norm, act=ops.PF_ACT_NONE, circ_stats=0, circ=0, halo=0)
        d = C // t.heads
        kv = self.text_kv
        o = torch.empty((N, L, C), dtype=dt, device=dev)
        # every LayerNorm is folded into its consumer: the producer GEMM emits per-row (sum, sum^2) partials, the
        # consumer (gamma-scaled weights) normalises in its epilogue — the normalised tensor is never stored
        h, st = ops.gemm_taps(xn, t.proj_in.w, new(C), M=T, Kc=t.proj_in.k, bias=t.proj_in.b, row_stats=True)
        qkv = ops.gemm_taps(h, t.qkv_ln.w, new(3 * C), M=T, Kc=C, bias=t.qkv_ln.b,
                            ln=(st, t.qkv_ln.colsum, t.qkv_ln.eps)).reshape(N, L, 3 * C)
        ops.fmha(qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:], o, heads=t.heads, head_dim=d, scale=d ** -0.5)
        h, st = ops.gemm_taps(o.reshape(T, C), t.out1.w, new(C), M=T, Kc=C, bias=t.out1.b, residual=h, row_stats=True)
        q = ops.gemm_taps(h, t.q2_ln.w, new(C), M=T, Kc=C, bias=t.q2_ln.b,
                          ln=(st, t.q2_ln.colsum, t.q2_ln.eps)).reshape(N, L, C)
        ops.fmha(q, kv[..., t.kv_off:t.kv_off + C], kv[..., t.kv_off + C:t.kv_off + 2 * C], o, heads=t.heads,
                 head_dim=d, scale=d ** -0.5)
        Fk = t.ff_dim
        fh = new(Fk + C)  # [T, f | h]: A operand of the merged ff2 + proj_out GEMM
        h, st = ops.gemm_taps(o.reshape(T, C), t.out2.w, fh[:, Fk:], M=T, Kc=C, bias=t.out2.b, residual=h,
                              row_stats=True)
        ops.gemm_taps(h, t.ff1_ln.w, fh[:, :Fk], M=T, Kc=C, bias=t.ff1_ln.b, act=ops.PF_ACT_GEGLU, block_n=t.ff1_bn,
                      ln=(st, t.ff1_ln.colsum, t.ff1_ln.eps))
        out = ops.gemm_taps(fh, t.tail.w, new(x.C), M=T, Kc=Fk + C, bias=t.tail.b, residual=x.t)
        return Img(out, N, H, W)

    def downsample(self, x: Img, d: _Conv3) -> Img:
        """Downsample2D (3x3, stride 2, pad 1); panorama: pad_pano(2) -> conv -> unpad_pano(1) (MVGenModel.py:139-144)."""
        c = 2 if self.circ else 0
        N, H, W = x.N, x.H, x.W
        We = W + 2 * c
        a = ops.conv_prep(x.t, N, H, W, circ=c, phases=4, halo=1)
        Ho, Wo = H // 2, We // 2
        Hq, Wq = Ho + 1, Wo + 1
        PS = N * Hq * Wq
        taps = [((dy % 2) * 2 + (dx % 2)) * PS + (dy // 2) * Wq + (dx // 2) for dy in range(3) for dx in range(3)]
        crop = 1 if self.circ else 0
        Wout = Wo - 2 * crop
        out = torch.empty((N * Ho * Wout, d.cout), dtype=self.dt, device=x.t.device)
        ops.gemm_taps(a, d.w, out, M=PS, Kc=d.cin, taps=taps, bias=d.b, image_map=(Hq, Wq, 0, crop, Ho, Wout))
        return Img(out, N, Ho, Wout)

    def upsample(self, x: Img, u: "_Up") -> Img:
        """Upsample2D (nearest x2 -> 3x3 conv); panorama: pad_pano(1) -> up -> unpad_pano(2) (MVGenModel.py:272-277).
        Output pixel (2i+a, 2j+b) depends on a 2x2 neighbourhood of the ORIGINAL image only, so the layer runs as four
        4-tap GEMMs over the zero-haloed original image, each scattering its phase into the 2x larger output."""
        c = 1 if self.circ else 0
        N, H, W = x.N, x.H, x.W
        a = ops.conv_prep(x.t, N, H, W, circ=c, up=1, halo=1)
        Hp, Wp = H + 2, W + 2 * c + 2
        out = torch.empty((N * 2 * H * 2 * W, u.cout), dtype=self.dt, device=x.t.device)
        k = 0
        for pa in (0, 1):
            for pb in (0, 1):
                taps = [(pa + r - 1) * Wp + (pb + cc - 1) for r in (0, 1) for cc in (0, 1)]
                ops.gemm_taps(a, u.phase_w[k], out, M=N * Hp * Wp, Kc=u.cin, taps=taps, bias=u.b,
                              image_map=(Hp, Wp, 1, 1 + c, H, W), scatter=(2, 2, pa, pb))
                k += 1
        return Img(out, N, 2 * H, 2 * W)


# ---- ControlNet (BASELINE config 5) ------------------------------------------------------------------------------

def _pad64(c: int) -> int:
    return (c + 63) // 64 * 64


class _Conv3Padded:
    """3x3 conv whose channel counts are zero-padded to multiples of 64 (the tap-GEMM's K-slab / narrowest tile)."""

    def __init__(self, conv, dev, dt):
        w = conv.weight.detach()
        self.cout_real, self.cin_real = w.shape[0], w.shape[1]
        self.cout, self.cin = _pad64(w.shape[0]), _pad64(w.shape[1])
        wp = torch.zeros((self.cout, self.cin, 3, 3), dtype=w.dtype, device=w.device)
        wp[:w.shape[0], :w.shape[1]] = w
        self.w = pack_conv3x3(wp).to(dev, dt).contiguous()
        self.b = torch.zeros(self.cout, dtype=torch.float32, device=dev)
        self.b[:w.shape[0]] = conv.bias.detach().to(dev, torch.float32)
        self.stride = int(conv.stride[0])


class ControlNetPack(UNetPack):
    """Weights of a duck-typed diffusers `ControlNetModel` [3P] (built by the reference with
    `ControlNetModel.from_unet`, models/pano/PanoGenerator.py:153-157): the UNet-encoder copy + conditioning embedding
    (3x3 convs 3->16->16->32->32->96->96->256->320, SiLU between, strides 1,1,2,1,2,1,2,1) + one 1x1 conv per skip tensor
    and one for the mid output."""

    def __init__(self, cn, dev, dt):
        super().__init__(cn, dev, dt, encoder_only=True)
        ce = cn.controlnet_cond_embedding
        w0 = ce.conv_in.weight.detach()
        c0 = _pad64(w0.shape[0])
        self.ce_in_w = torch.zeros((c0, *w0.shape[1:]), dtype=torch.float32, device=dev)
        self.ce_in_w[:w0.shape[0]] = w0.to(dev, torch.float32)
        self.ce_in_b = torch.zeros(c0, dtype=torch.float32, device=dev)
        self.ce_in_b[:w0.shape[0]] = ce.conv_in.bias.detach().to(dev, torch.float32)
        self.ce_blocks = [_Conv3Padded(b, dev, dt) for b in ce.blocks]
        self.ce_out = _Conv3Padded(ce.conv_out, dev, dt)
        assert self.ce_out.cout == self.ce_out.cout_real, "conditioning embedding width must be a multiple of 64"
        self.zero_down = [_Lin(c.weight, c.bias, dev, dt) for c in cn.controlnet_down_blocks]
        self.zero_mid = _Lin(cn.controlnet_mid_block.weight, cn.controlnet_mid_block.bias, dev, dt)


class ControlBranch(Branch):
    """The ControlNet encoder. The reference hands it the UN-padded latent and calls it as a black box
    (MVGenModel.py:66-83), so every convolution here is zero-padded even on the panorama (`circular=False`)."""

    def __init__(self, pack: ControlNetPack):
        super().__init__(pack, circular=False)
        self._cond_cache: dict = {}

    def _conv3(self, x: Img, c: _Conv3Padded, act: int, residual: Optional[Tensor] = None, prepared=None) -> Img:
        N, H, W = x.N, x.H, x.W
        dev = x.t.device
        if c.stride == 1:
            a = prepared if prepared is not None else ops.conv_prep(x.t, N, H, W, halo=1)
            Hp, Wp = H + 2, W + 2
            out = torch.empty((N * H * W, c.cout), dtype=self.dt, device=dev)
            ops.gemm_taps(a, c.w, out, M=N * Hp * Wp, Kc=c.cin, taps=taps3x3(Wp), bias=c.b, act=act, residual=residual,
                          image_map=(Hp, Wp, 1, 1, H, W))
            return Img(out, N, H, W)
        a = ops.conv_prep(x.t, N, H, W, phases=4, halo=1)
        Ho, Wo = H // 2, W // 2
        Hq, Wq = Ho + 1, Wo + 1
        PS = N * Hq * Wq
        taps = [((dy % 2) * 2 + (dx % 2)) * PS + (dy // 2) * Wq + (dx // 2) for dy in range(3) for dx in range(3)]
        out = torch.empty((N * Ho * Wo, c.cout), dtype=self.dt, device=dev)
        ops.gemm_taps(a, c.w, out, M=PS, Kc=c.cin, taps=taps, bias=c.b, act=act, image_map=(Hq, Wq, 0, 0, Ho, Wo))
        return Img(out, N, Ho, Wo)

    def cond_features(self, cond: Tensor, key=None):
        """controlnet_cond_embedding up to (not including) its last convolution, returned as that convolution's
        prepared A operand. Depends only on the layout image, which the sampler merely rolls by a quarter turn per
        step (PanFusion.py:152-153): cached on the identity + version of the caller's tensor, like the text K/V."""
        key = key if key is not None else (cond.data_ptr(), cond._version, tuple(cond.shape))
        hit = self._cond_cache.get(key)
        if hit is not None:
            return hit[:4]
        p = self.p
        n, _, hc, wc = cond.shape
        x = Img(ops.conv_in(cond.to(torch.float32).contiguous(), p.ce_in_w, p.ce_in_b, self.dt, False,
                            act=ops.PF_ACT_SILU), n, hc, wc)
        for blk in p.ce_blocks:
            x = self._conv3(x, blk, ops.PF_ACT_SILU)
        # entry keeps `cond` alive: the key is its identity, so its address must not be reused while cached
        hit = (ops.conv_prep(x.t, x.N, x.H, x.W, halo=1), x.N, x.H, x.W, cond)
        if len(self._cond_cache) >= 8:
            self._cond_cache.clear()
        self._cond_cache[key] = hit
        return hit[:4]

    def encode(self, latent: Tensor, cond: Tensor, cond_key=None):
        """-> (12 skip-shaped tensors, mid tensor) BEFORE the zero convs (applied by `add_down` / `add_mid` where the
        reference adds the residuals). set_timesteps / set_text must have been called."""
        p = self.p
        a, n, h, w = self.cond_features(cond, cond_key)
        x = self.conv_in(latent)
        assert (n, h, w) == (x.N, x.H, x.W), "layout condition must be 8x the latent resolution"
        x = self._conv3(x, p.ce_out, ops.PF_ACT_NONE, residual=x.t, prepared=a)  # conv_in(sample) + embedding(cond)
        res = [x]
        for blk in p.down:
            for j, r in enumerate(blk["resnets"]):
                x = self.resnet(x, r)
                if blk["attns"] is not None:
                    x = self.transformer(x, blk["attns"][j])
                res.append(x)
            if blk["down"] is not None:
                for d in blk["down"]:
                    x = self.downsample(x, d)
                res.append(x)
        x = self.resnet(x, p.mid["resnets"][0])
        for i, t in enumerate(p.mid["attns"]):
            x = self.transformer(x, t)
            x = self.resnet(x, p.mid["resnets"][i + 1])
        return res, x

    def _zero(self, lin: _Lin, r: Img, target: Img) -> Img:
        T = r.t.shape[0]
        out = torch.empty((T, lin.n), dtype=self.dt, device=r.t.device)
        ops.gemm_taps(r.t, lin.w, out, M=T, Kc=lin.k, bias=lin.b, residual=target.t)
        return Img(out, target.N, target.H, target.W)

    def add_down(self, res: list, skips: list) -> list:
        """skip_i + controlnet_down_blocks[i](res_i)  (MVGenModel.py:154-170), one GEMM with residual epilogue each."""
        assert len(res) == len(skips) == len(self.p.zero_down)
        return [self._zero(z, r, s) for z, r, s in zip(self.p.zero_down, res, skips)]

    def add_mid(self, mid: Img, hidden: Img) -> Img:
        """hidden + controlnet_mid_block(mid)  (MVGenModel.py:200-203)."""
        return self._zero(self.p.zero_mid, mid, hidden)
