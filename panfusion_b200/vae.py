"""Image-space tail of the sampling loop: VAE decode with circular latent padding + `tensor_to_image`
(SURVEY.md §8f rank 1) behind the reference's function names — and, for the training step's forward half (§8f rank 4), the
VAE encoder behind `encode_image` (PanoGenerator.py:214-225) with the circular IMAGE padding of PanFusion.py:69-71.

Reference: `decode_latent` models/pano/PanoGenerator.py:272-278, the padded panorama decode PanFusion.py:166-172
(`pad_pano(latent=True)` with `latent_pad = 8`, PanoGenerator.py:227-238), `tensor_to_image`
models/modules/utils.py:9-15. The decoder is diffusers `AutoencoderKL` [3P]; like the UNets it is consumed by
attribute walk to read its parameters once (`VAEDecoder.prepare`) and then runs on the kernels of the denoiser:
conv_in on `pf_conv_in`, every 3x3 conv / shortcut / linear on the tap-GEMM (Upsample2D as four phase convolutions),
GroupNorm + SiLU + zero halo in `pf_groupnorm_stats` (the statistics launch of `pf_gn_prep`) / `pf_conv_prep`. The
mid-block attention has one head of width 512 — outside the flash kernel's head sizes and 0.1 % of the decoder's
FLOPs — and runs as tap-GEMM (Q K^T, fp32) -> `pf_softmax_rows` -> tap-GEMM (P V^T-operand). No PyTorch compute
fallback.
"""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch
from torch import Tensor

from . import _lib, ops
from .engine import Branch, Img, _Conv3, _Lin, _Norm, _Up, taps3x3
from .packing import pack_conv3x3
from .pano import pad_pano, unpad_pano


class _VResnet:
    def __init__(self, r, dev, dt):
        self.norm1, self.norm2 = _Norm(r.norm1, dev), _Norm(r.norm2, dev)
        self.conv1, self.conv2 = _Conv3(r.conv1, dev, dt), _Conv3(r.conv2, dev, dt)
        sc = getattr(r, "conv_shortcut", None)
        self.short = _Lin(sc.weight, sc.bias, dev, dt) if sc is not None else None
        self.temb_off = -1  # no time embedding in the VAE


class VAEDecoderPack:
    def __init__(self, vae, dev, dt):
        self.dev, self.dt = dev, dt
        d = vae.decoder
        self.groups = int(d.conv_norm_out.num_groups)
        self.scaling_factor = float(vae.config.scaling_factor)
        # post_quant_conv (1x1, 4 -> 4) folded EXACTLY into conv_in: composed weights for the latent channels plus one
        # extra input channel of ones that carries post_quant_conv's bias (zero outside the image, like the padding)
        wq = vae.post_quant_conv.weight.detach().double().flatten(1)      # [4, 4]
        bq = vae.post_quant_conv.bias.detach().double()                   # [4]
        wi = d.conv_in.weight.detach().double()                           # [C, 4, 3, 3]
        w_lat = torch.einsum("octs,ci->oits", wi, wq)
        w_one = torch.einsum("octs,c->ots", wi, bq)[:, None]
        self.conv_in_w = torch.cat([w_lat, w_one], 1).to(dev, torch.float32).contiguous()  # [C, 5, 3, 3]
        # same with decode_latent's `1 / scaling_factor * latents` (PanoGenerator.py:274) folded into the latent channels
        self.conv_in_w_unscale = torch.cat([w_lat / self.scaling_factor, w_one], 1).to(dev, torch.float32).contiguous()
        self.conv_in_b = d.conv_in.bias.detach().to(dev, torch.float32).contiguous()
        self.mid_res = [_VResnet(r, dev, dt) for r in d.mid_block.resnets]
        a = d.mid_block.attentions[0]
        self.att_norm = _Norm(a.group_norm, dev)
        self.att_qk = _Lin(torch.cat([a.to_q.weight, a.to_k.weight], 0), torch.cat([a.to_q.bias, a.to_k.bias], 0), dev, dt)
        self.att_v = a.to_v.weight.detach().to(dev, dt).contiguous()     # used as the A operand: V^T = W_v X^T
        # rows of P sum to one, so to_v's bias passes through the attention unchanged: fold it into to_out's bias
        wo, bo = a.to_out[0].weight.detach().double(), a.to_out[0].bias.detach().double()
        self.att_out = _Lin(a.to_out[0].weight, (bo + wo @ a.to_v.bias.detach().double()).float(), dev, dt)
        self.C_mid = self.att_out.n
        self.up = []
        for blk in d.up_blocks:
            self.up.append(dict(resnets=[_VResnet(r, dev, dt) for r in blk.resnets],
                                up=[_Up(u.conv, dev, dt) for u in blk.upsamplers] if blk.upsamplers is not None else None))
        self.norm_out = _Norm(d.conv_norm_out, dev)
        co = d.conv_out.weight.shape[0]
        wpad = torch.zeros((64, *d.conv_out.weight.shape[1:]), dtype=d.conv_out.weight.dtype, device=d.conv_out.weight.device)
        wpad[:co] = d.conv_out.weight.detach()
        self.conv_out_packed = pack_conv3x3(wpad).to(dev, dt).contiguous()
        self.conv_out_bpad = torch.zeros(64, dtype=torch.float32, device=dev)
        self.conv_out_bpad[:co] = d.conv_out.bias.detach().to(dev, torch.float32)
        self.conv_out_c = co


class _DecoderBranch(Branch):
    """Reuses Branch.resnet / Branch.upsample (zero padding, no time embedding)."""

    def __init__(self, pack):
        super().__init__(pack, circular=False)

    def resnet(self, x: Img, r) -> Img:
        N, H, W = x.N, x.H, x.W
        g = self.p.groups
        s1 = ops.groupnorm_stats(x.t, N, H, W, g, r.norm1.eps, 0)
        a1 = ops.conv_prep(x.t, N, H, W, stats=s1, gamma=r.norm1.g, beta=r.norm1.b, groups=g, act=ops.PF_ACT_SILU, halo=1)
        Hp, Wp = H + 2, W + 2
        h1 = torch.empty((N * H * W, r.conv1.cout), dtype=self.dt, device=x.t.device)
        ops.gemm_taps(a1, r.conv1.w, h1, M=N * Hp * Wp, Kc=r.conv1.cin, taps=taps3x3(Wp), bias=r.conv1.b,
                      image_map=(Hp, Wp, 1, 1, H, W))
        s2 = ops.groupnorm_stats(h1, N, H, W, g, r.norm2.eps, 0)
        a2 = ops.conv_prep(h1, N, H, W, stats=s2, gamma=r.norm2.g, beta=r.norm2.b, groups=g, act=ops.PF_ACT_SILU, halo=1)
        if r.short is not None:
            res = torch.empty((N * H * W, r.short.n), dtype=self.dt, device=x.t.device)
            ops.gemm_taps(x.t, r.short.w, res, M=N * H * W, Kc=r.short.k, bias=r.short.b)
        else:
            res = x.t
        out = torch.empty((N * H * W, r.conv2.cout), dtype=self.dt, device=x.t.device)
        ops.gemm_taps(a2, r.conv2.w, out, M=N * Hp * Wp, Kc=r.conv2.cin, taps=taps3x3(Wp), bias=r.conv2.b, residual=res,
                      image_map=(Hp, Wp, 1, 1, H, W))
        return Img(out, N, H, W)

    def attention(self, x: Img) -> Img:
        """GroupNorm -> q, k, v (with bias) -> softmax(q k^T / sqrt(C)) v -> to_out -> + x; one head of width C."""
        p = self.p
        N, H, W, Cc = x.N, x.H, x.W, p.C_mid
        L = H * W
        if L % 64:
            raise NotImplementedError(f"VAE attention needs H*W divisible by 64 (got {H}x{W})")
        dev, dt = x.t.device, self.dt
        s = ops.groupnorm_stats(x.t, N, H, W, p.groups, p.att_norm.eps, 0)
        xn = ops.conv_prep(x.t, N, H, W, stats=s, gamma=p.att_norm.g, beta=p.att_norm.b, groups=p.groups, halo=0)
        qk = ops.gemm_taps(xn, p.att_qk.w, torch.empty((N * L, 2 * Cc), dtype=dt, device=dev), M=N * L, Kc=Cc,
                           bias=p.att_qk.b)
        o = torch.empty((N * L, Cc), dtype=dt, device=dev)
        logits = torch.empty((L, L), dtype=torch.float32, device=dev)
        probs = torch.empty((L, L), dtype=dt, device=dev)
        vt = torch.empty((Cc, L), dtype=dt, device=dev)
        for n in range(N):  # one image at a time: the [L, L] logits are the only large temporary (340 MB at 64x144)
            rows = slice(n * L, (n + 1) * L)
            ops.gemm_taps(qk[rows, :Cc], qk[rows, Cc:], logits, M=L, Kc=Cc)           # Q K^T, fp32
            ops.softmax_rows(logits, probs, Cc ** -0.5)
            ops.gemm_taps(p.att_v, xn[rows], vt, M=Cc, Kc=Cc)                           # V^T = W_v X^T (bias folded)
            ops.gemm_taps(probs, vt, o[rows], M=L, Kc=L)                                # P V
        out = torch.empty((N * L, Cc), dtype=dt, device=dev)
        ops.gemm_taps(o, p.att_out.w, out, M=N * L, Kc=Cc, bias=p.att_out.b, residual=x.t)
        return Img(out, N, H, W)


class VAEDecoder:
    """`VAEDecoder(vae).decode(z)` == `vae.decode(z).sample` for z [N, 4, h, w] -> fp32 [N, 3, 8h, 8w]."""

    def __init__(self, vae, compute_dtype=torch.bfloat16):
        self.vae, self.compute_dtype = vae, compute_dtype
        self.config = vae.config
        self._b: Optional[_DecoderBranch] = None

    def prepare(self, device=None, dtype=None) -> "VAEDecoder":
        device = torch.device(device or "cuda")
        if device.type == "cuda" and device.index is None:  # "cuda" != "cuda:0": would re-pack on every decode
            device = torch.device("cuda", torch.cuda.current_device())
        _lib.check(_lib.lib().pf_check_device())
        self._b = _DecoderBranch(VAEDecoderPack(self.vae, device, dtype or self.compute_dtype))
        return self

    @torch.no_grad()
    def decode(self, z: Tensor, unscale: bool = False) -> Tensor:
        """unscale=True decodes z / scaling_factor (the division folded into conv_in's weights)."""
        _lib.require_cuda(z)
        if self._b is None or self._b.p.dev != z.device:
            self.prepare(z.device)
        b = self._b
        p = b.p
        N, _, h, w = z.shape
        zf = z.to(torch.float32)
        z_aug = torch.cat([zf, torch.ones((N, 1, h, w), dtype=torch.float32, device=z.device)], 1).contiguous()
        x = Img(ops.conv_in(z_aug, p.conv_in_w_unscale if unscale else p.conv_in_w, p.conv_in_b, b.dt, False), N, h, w)
        x = b.resnet(x, p.mid_res[0])
        x = b.attention(x)
        x = b.resnet(x, p.mid_res[1])
        for blk in p.up:
            for r in blk["resnets"]:
                x = b.resnet(x, r)
            if blk["up"] is not None:
                for u in blk["up"]:
                    x = b.upsample(x, u)
        # conv_norm_out -> SiLU -> conv_out (3 channels in one 64-wide tap-GEMM tile, fp32 out)
        st = ops.groupnorm_stats(x.t, x.N, x.H, x.W, p.groups, p.norm_out.eps, 0)
        xp = ops.conv_prep(x.t, x.N, x.H, x.W, stats=st, gamma=p.norm_out.g, beta=p.norm_out.b, groups=p.groups,
                           act=ops.PF_ACT_SILU, halo=1)
        Hp, Wp = x.H + 2, x.W + 2
        o = torch.empty((x.N * x.H * x.W, 64), dtype=torch.float32, device=z.device)
        ops.gemm_taps(xp, p.conv_out_packed, o, M=x.N * Hp * Wp, Kc=x.C, taps=taps3x3(Wp), bias=p.conv_out_bpad,
                      image_map=(Hp, Wp, 1, 1, x.H, x.W), block_n=64)
        return o[:, :p.conv_out_c].reshape(x.N, x.H, x.W, p.conv_out_c).permute(0, 3, 1, 2).contiguous()


# ---- encoder (training step only: PanoGenerator.encode_image, PanFusion.py:66-71) ---------------------------------------------

class VAEEncoderPack:
    def __init__(self, vae, dev, dt):
        self.dev, self.dt = dev, dt
        e = vae.encoder
        self.groups = int(e.conv_norm_out.num_groups)
        self.scaling_factor = float(vae.config.scaling_factor)
        self.latent_channels = int(vae.quant_conv.weight.shape[0]) // 2
        self.conv_in_w = e.conv_in.weight.detach().to(dev, torch.float32).contiguous()   # [C0, 3, 3, 3]
        self.conv_in_b = e.conv_in.bias.detach().to(dev, torch.float32).contiguous()
        self.down = []
        for blk in e.down_blocks:
            self.down.append(dict(resnets=[_VResnet(r, dev, dt) for r in blk.resnets],
                                  down=[_Conv3(d.conv, dev, dt) for d in blk.downsamplers] if blk.downsamplers is not None else None))
        self.mid_res = [_VResnet(r, dev, dt) for r in e.mid_block.resnets]
        a = e.mid_block.attentions[0]
        self.att_norm = _Norm(a.group_norm, dev)
        self.att_qk = _Lin(torch.cat([a.to_q.weight, a.to_k.weight], 0), torch.cat([a.to_q.bias, a.to_k.bias], 0), dev, dt)
        self.att_v = a.to_v.weight.detach().to(dev, dt).contiguous()
        wo, bo = a.to_out[0].weight.detach().double(), a.to_out[0].bias.detach().double()
        self.att_out = _Lin(a.to_out[0].weight, (bo + wo @ a.to_v.bias.detach().double()).float(), dev, dt)
        self.C_mid = self.att_out.n
        self.norm_out = _Norm(e.conv_norm_out, dev)
        # quant_conv (1x1, 2L -> 2L) folded EXACTLY into conv_out: W' = Wq W_out, b' = Wq b_out + bq; padded to one 64-wide tile
        wq = vae.quant_conv.weight.detach().double().flatten(1)            # [2L, 2L]
        bq = vae.quant_conv.bias.detach().double()
        wc = e.conv_out.weight.detach().double()                           # [2L, C, 3, 3]
        w2 = torch.einsum("oc,cits->oits", wq, wc)
        b2 = wq @ e.conv_out.bias.detach().double() + bq
        co = w2.shape[0]
        wpad = torch.zeros((64, *w2.shape[1:]), dtype=torch.float32)
        wpad[:co] = w2.float()
        self.conv_out_packed = pack_conv3x3(wpad).to(dev, dt).contiguous()
        self.conv_out_bpad = torch.zeros(64, dtype=torch.float32, device=dev)
        self.conv_out_bpad[:co] = b2.float().to(dev)


class _EncoderBranch(_DecoderBranch):
    """The decoder's resnet / attention blocks plus the encoder's Downsample2D: zero-pad right and bottom by one, 3x3
    stride-2 convolution (diffusers Downsample2D(padding=0) [3P]). Like Branch.downsample it runs on the four stride-2 phases
    of the zero-haloed image; the taps start one pixel later because there is no padding on the left / top:
    out(i, j) = sum w[dy, dx] x[2i + dy, 2j + dx]."""

    def downsample(self, x: Img, d: _Conv3) -> Img:
        N, H, W = x.N, x.H, x.W
        if H % 2 or W % 2:
            raise NotImplementedError(f"VAE encoder needs even image sizes at every level (got {H}x{W})")
        a = ops.conv_prep(x.t, N, H, W, phases=4, halo=1)
        Ho, Wo = H // 2, W // 2
        Hq, Wq = Ho + 1, Wo + 1
        PS = N * Hq * Wq
        # phase (a, b) holds x[2i + a - 1, 2j + b - 1]: x[2i + dy] = phase (dy + 1) % 2 at row i + (dy + 1) // 2
        taps = [(((dy + 1) % 2) * 2 + ((dx + 1) % 2)) * PS + ((dy + 1) // 2) * Wq + ((dx + 1) // 2)
                for dy in range(3) for dx in range(3)]
        out = torch.empty((N * Ho * Wo, d.cout), dtype=self.dt, device=x.t.device)
        ops.gemm_taps(a, d.w, out, M=PS, Kc=d.cin, taps=taps, bias=d.b, image_map=(Hq, Wq, 0, 0, Ho, Wo))
        return Img(out, N, Ho, Wo)


class VAEEncoder:
    """`VAEEncoder(vae).encode(x, noise)` == `vae.encode(x).latent_dist.sample()` for x [N, 3, H, W] in [-1, 1] -> fp32
    [N, 4, H/8, W/8] (optionally times scaling_factor), on the kernels of the decoder + `pf_gaussian_sample`."""

    def __init__(self, vae, compute_dtype=torch.bfloat16):
        self.vae, self.compute_dtype = vae, compute_dtype
        self.config = vae.config
        self._b: Optional[_EncoderBranch] = None

    def prepare(self, device=None, dtype=None) -> "VAEEncoder":
        device = torch.device(device or "cuda")
        if device.type == "cuda" and device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        _lib.check(_lib.lib().pf_check_device())
        self._b = _EncoderBranch(VAEEncoderPack(self.vae, device, dtype or self.compute_dtype))
        return self

    @torch.no_grad()
    def moments(self, x: Tensor):
        """-> (fp32 rows [N*h*w, 64] whose first 2L columns are mean | logvar after quant_conv, N, h, w)."""
        _lib.require_cuda(x)
        if self._b is None or self._b.p.dev != x.device:
            self.prepare(x.device)
        b = self._b
        p = b.p
        N, _, H, W = x.shape
        h = Img(ops.conv_in(x.to(torch.float32).contiguous(), p.conv_in_w, p.conv_in_b, b.dt, False), N, H, W)
        for blk in p.down:
            for r in blk["resnets"]:
                h = b.resnet(h, r)
            if blk["down"] is not None:
                for d in blk["down"]:
                    h = b.downsample(h, d)
        h = b.resnet(h, p.mid_res[0])
        h = b.attention(h)
        h = b.resnet(h, p.mid_res[1])
        st = ops.groupnorm_stats(h.t, h.N, h.H, h.W, p.groups, p.norm_out.eps, 0)
        xp = ops.conv_prep(h.t, h.N, h.H, h.W, stats=st, gamma=p.norm_out.g, beta=p.norm_out.b, groups=p.groups,
                           act=ops.PF_ACT_SILU, halo=1)
        Hp, Wp = h.H + 2, h.W + 2
        o = torch.empty((h.N * h.H * h.W, 64), dtype=torch.float32, device=x.device)
        ops.gemm_taps(xp, p.conv_out_packed, o, M=h.N * Hp * Wp, Kc=h.C, taps=taps3x3(Wp), bias=p.conv_out_bpad,
                      image_map=(Hp, Wp, 1, 1, h.H, h.W), block_n=64)
        return o, h.N, h.H, h.W

    @torch.no_grad()
    def encode(self, x: Tensor, noise: Optional[Tensor] = None, generator=None, scale: bool = False) -> Tensor:
        """noise: the standard-normal draw of `latent_dist.sample()` ([N, 4, h, w]); drawn on the device when None.
        scale=True multiplies by vae.config.scaling_factor (encode_image's last line)."""
        o, N, h, w = self.moments(x)
        L = self._b.p.latent_channels
        if noise is None:
            noise = torch.randn((N, L, h, w), device=x.device, dtype=torch.float32, generator=generator)
        return ops.gaussian_sample(o, noise.to(torch.float32).contiguous(), L, self._b.p.scaling_factor if scale else 1.0)


def encode_image(x_input: Tensor, vae: VAEEncoder, noise: Optional[Tensor] = None, generator=None) -> Tensor:
    """PanoGenerator.py:214-225: [b, l, 3, H, W] -> sampled latents [b, l, 4, H/8, W/8] * scaling_factor (fp32)."""
    b = x_input.shape[0]
    z = vae.encode(x_input.flatten(0, 1), noise=noise.flatten(0, 1) if noise is not None else None, generator=generator,
                   scale=True)
    return z.reshape(b, -1, *z.shape[1:])


def encode_pano(pano: Tensor, vae: VAEEncoder, latent_pad: int = 8, noise: Optional[Tensor] = None, generator=None) -> Tensor:
    """PanFusion.py:69-71: pad the IMAGE circularly by 8 * latent_pad pixels, encode, crop latent_pad latent columns.
    `noise` (if given) has the PADDED latent width, like the draw inside the reference's encode."""
    return unpad_pano(encode_image(pad_pano(pano, 8 * latent_pad), vae, noise, generator), latent_pad)


# ---- the reference's functions ---------------------------------------------------------------------------------

def decode_latent(latents: Tensor, vae: VAEDecoder) -> Tensor:
    """PanoGenerator.py:272-278: [b, m, 4, h, w] -> [b, m, 3, 8h, 8w] (fp32)."""
    b = latents.shape[0]
    image = vae.decode(latents.flatten(0, 1), unscale=True)
    return image.reshape(b, -1, *image.shape[1:])


def decode_pano(pano_latent: Tensor, vae: VAEDecoder, latent_pad: int = 8) -> Tensor:
    """PanFusion.py:169-171: pad the LATENT circularly by latent_pad columns, decode, crop 8 * latent_pad pixels."""
    return unpad_pano(decode_latent(pad_pano(pano_latent, latent_pad), vae), 8 * latent_pad)


def tensor_to_image(image: Tensor) -> np.ndarray:
    """models/modules/utils.py:9-15: float [-1, 1] [..., c, h, w] -> uint8 numpy [..., h, w, c]."""
    if image.dtype == torch.uint8:
        return image.cpu().numpy().transpose(*range(image.ndim - 3), -2, -1, -3)
    _lib.require_cuda(image)
    return ops.tensor_to_image(image.to(torch.float32)).cpu().numpy()
