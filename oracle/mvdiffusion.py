"""Oracle: MVDiffusion's denoiser (external/MVDiffusion/pano/MVGenModel.py, pano/modules.py, pano/utils.py) restated in
plain PyTorch fp32, plus the golden generator that executes the reference's own files by path. Test infrastructure.

    python -m oracle.mvdiffusion               # mints tests/golden/mvdiff_{tables,cpattn,tiny,mp2e}.npz
    python -m oracle.mvdiffusion --only c2     # the SD-2-width 8-view CFG step (minutes on 8 cores): mvdiff_c2.npz

The restatement computes the CPAttn geometry as per-(view, query pixel, key slot) tables — the layout of
pf_cpattn_tables: slot s = n * 9 + (di + 1) * 3 + (dj + 1), n = 0 for view i-1 and 1 for view i+1, di moving x and dj
moving y — with the reference's fp32 operations, so that the positional-encoding arguments match bit for bit (the
frequencies reach 2^79 at C = 320, where one ulp of the argument changes the encoding completely).
"""
from __future__ import annotations

import importlib
import sys
import types
from pathlib import Path

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from .eppa import BasicTransformerBlock

OUT = Path(__file__).resolve().parent.parent / "tests" / "golden"


def get_K_R(fov: float, theta: float, phi: float, size: int):
    """dataset/PanoDataset.py:16-31 (square views): pinhole K and the yaw-then-pitch rotation, as float32 arrays."""
    import cv2
    f = 0.5 * size / np.tan(0.5 * fov / 180.0 * np.pi)
    c = (size - 1) / 2.0
    K = np.array([[f, 0, c], [0, f, c], [0, 0, 1]], np.float32)
    R1, _ = cv2.Rodrigues(np.array([0.0, 1.0, 0.0], np.float32) * np.radians(theta))
    R2, _ = cv2.Rodrigues(np.dot(R1, np.array([1.0, 0.0, 0.0], np.float32)) * np.radians(phi))
    return K, (R2 @ R1).astype(np.float32)


def horizon_cameras(m: int, batch: int = 1, fov: float = 90.0, size: int = 512):
    """cam_sampler='horizon' (utils/pano.py:28-31, PanoDataset.py:106-115): m yaws evenly spaced, pitch 0 -> K, R [batch, m, 3, 3]."""
    theta = np.rad2deg(np.linspace(0, 2 * np.pi, m, endpoint=False))
    KR = [get_K_R(fov, t, 0.0, size) for t in theta]
    K = torch.from_numpy(np.stack([k for k, _ in KR]))[None].repeat(batch, 1, 1, 1)
    R = torch.from_numpy(np.stack([r for _, r in KR]))[None].repeat(batch, 1, 1, 1)
    return K, R


# ---- CPAttn geometry ----------------------------------------------------------------------------------------------
def _neighbours(i: int, m: int):
    return [(i - 1 + m) % m, (i + 1) % m]


def _apply(H: torch.Tensor, pts: torch.Tensor) -> torch.Tensor:
    """H [..., 3, 3] @ [x; y; 1] columns pts [..., 3, n] -> [..., 2, n] (dehomogenised), fp32 like the reference."""
    r = H @ pts
    return r[..., :2, :] / r[..., 2:, :]


def tables(K: torch.Tensor, R: torch.Tensor, h: int, img: int):
    """K, R [B, m, 3, 3] -> (pos [B, m, h*h, 18, 2] window positions in key-map pixels (before grid_sample's
    normalisation), mask bool [B, m, h*h, 18], xy_rel [B, m, h*h, 18, 2]) for the h x h level of img x img views."""
    B, m = K.shape[:2]
    s = img // h
    c = (s // 2 + s * torch.arange(h)).float()
    yy, xx = torch.meshgrid(c, c, indexing="ij")
    q = torch.stack([xx.reshape(-1), yy.reshape(-1), torch.ones(h * h)])          # [3, P] image positions
    inv = torch.inverse
    pos, mask, rel = [], [], []
    for i in range(m):
        pv, mv, rv = [], [], []
        for j in _neighbours(i, m):
            Hl = K[:, j] @ inv(R[:, j]) @ R[:, i] @ inv(K[:, i])                  # view i -> view j (utils.py:26-27)
            Hr = K[:, i] @ inv(R[:, i]) @ R[:, j] @ inv(K[:, j])                  # view j -> view i (modules.py:57-58)
            p = _apply(Hl, q[None].expand(B, 3, -1)) / s - 0.5                   # [B, 2, P]
            for di in (-1, 0, 1):
                for dj in (-1, 0, 1):
                    n = torch.stack([p[:, 0] + di, p[:, 1] + dj], 1)              # [B, 2, P]
                    sc = (n + 0.5) * s
                    mv.append((sc[:, 0] > 0) & (sc[:, 0] < img) & (sc[:, 1] > 0) & (sc[:, 1] < img))
                    back = _apply(Hr, torch.cat([sc, torch.ones(B, 1, h * h)], 1))
                    rv.append(((back - q[None, :2]) / s).transpose(1, 2))
                    pv.append(n.transpose(1, 2))
        pos.append(torch.stack(pv, 2))
        mask.append(torch.stack(mv, 2))
        rel.append(torch.stack(rv, 2))
    return torch.stack(pos, 1), torch.stack(mask, 1), torch.stack(rel, 1)


def pos_embedding(xy: torch.Tensor, freq_bands: torch.Tensor) -> torch.Tensor:
    """[..., 2] -> [..., 4N] = [sin(x f), sin(y f), cos(x f), cos(y f)] (modules/transformer.py:191-209)."""
    e = xy[..., :, None] * freq_bands.reshape(-1)
    return torch.cat([e.sin(), e.cos()], -2).flatten(-2)


def gather_keys(x: torch.Tensor, pos: torch.Tensor, mask: torch.Tensor, rel: torch.Tensor, freq_bands: torch.Tensor):
    """x [B, m, C, h, w] -> key tokens [B, m, h*w, 18, C] = (bilinear sample + PE(xy_rel)) * mask."""
    B, m, C, h, w = x.shape
    out = []
    for i in range(m):
        ks = []
        for n, j in enumerate(_neighbours(i, m)):
            p = pos[:, i, :, 9 * n:9 * n + 9]                                      # [B, P, 9, 2]
            g = torch.stack([p[..., 0] / (w - 1) * 2 - 1, p[..., 1] / (h - 1) * 2 - 1], -1)
            ks.append(F.grid_sample(x[:, j], g, align_corners=True).permute(0, 2, 3, 1))  # [B, P, 9, C]
        out.append(torch.cat(ks, 2))
    v = torch.stack(out, 1)
    return (v + pos_embedding(rel, freq_bands)) * mask[..., None]


class PosEmbedding(nn.Module):
    def __init__(self, n_freqs):
        super().__init__()
        base = 2 if n_freqs <= 80 else 5000 ** (1 / (n_freqs / 2.5))
        self.register_buffer("freq_bands", base ** torch.linspace(0, n_freqs - 1, n_freqs)[None, None])


class CPAttn(nn.Module):
    def __init__(self, dim, flag360=False):
        super().__init__()
        self.flag360 = flag360
        self.transformer = BasicTransformerBlock(dim, dim // 32, 32, dim)
        self.pe = PosEmbedding(dim // 4)

    def forward(self, x, correspondences, img_h, img_w, R, K, m):
        bm, C, h, w = x.shape
        x5 = x.reshape(bm // m, m, C, h, w)
        pos, mask, rel = tables(K, R, h, img_h)
        keys = gather_keys(x5, pos, mask, rel, self.pe.freq_bands).reshape(-1, 18, C)
        q = x5.permute(0, 1, 3, 4, 2).reshape(-1, 1, C)
        # the reference's softmax runs over all 18 keys, masked ones included: no attention bias
        out = self.transformer(q, keys, torch.zeros(q.shape[0], 1, 18),
                               query_pe=pos_embedding(torch.zeros(1, 2), self.pe.freq_bands))
        return out.reshape(bm // m, m, h, w, C).permute(0, 1, 4, 2, 3).reshape(bm, C, h, w)


class MultiViewBaseModel(nn.Module):
    """MVGenModel.py:8-155 over the oracle's SD-2 UNet restatement (oracle/unet.py)."""

    def __init__(self, unet, pers_cn=None):
        super().__init__()
        self.unet, self.pers_cn = unet, pers_cn
        self.cp_blocks_encoder = nn.ModuleList([CPAttn(b.resnets[-1].out_channels, True) for b in unet.down_blocks])
        self.cp_blocks_mid = CPAttn(unet.mid_block.resnets[-1].out_channels, True)
        self.cp_blocks_decoder = nn.ModuleList([CPAttn(b.resnets[-1].out_channels, True) for b in unet.up_blocks])

    def forward(self, latents, timestep, prompt_embd, meta, pers_layout_cond=None):
        K, R = meta["K"], meta["R"]
        b, m, _, h, w = latents.shape
        img = h * 8
        ctx = prompt_embd.flatten(0, 1)
        u = self.unet
        emb = u.time_embedding(u.time_proj(timestep.reshape(-1)))
        cp = (lambda blk, x: blk(x, None, img, img, R, K, m)) if m > 1 else (lambda blk, x: x)
        x = u.conv_in(latents.flatten(0, 1))
        skips = [x]
        for i, blk in enumerate(u.down_blocks):
            for j, r in enumerate(blk.resnets):
                x = r(x, emb)
                if getattr(blk, "has_cross_attention", False):
                    x = blk.attentions[j](x, encoder_hidden_states=ctx).sample
                skips.append(x)
            x = cp(self.cp_blocks_encoder[i], x)
            if blk.downsamplers is not None:
                for d in blk.downsamplers:
                    x = d(x)
                skips.append(x)
        x = u.mid_block.resnets[0](x, emb)
        x = cp(self.cp_blocks_mid, x)
        for at, r in zip(u.mid_block.attentions, u.mid_block.resnets[1:]):
            x = r(at(x, encoder_hidden_states=ctx).sample, emb)
        for i, blk in enumerate(u.up_blocks):
            for j, r in enumerate(blk.resnets):
                x = r(torch.cat([x, skips.pop()], 1), emb)
                if getattr(blk, "has_cross_attention", False):
                    x = blk.attentions[j](x, encoder_hidden_states=ctx).sample
            x = cp(self.cp_blocks_decoder[i], x)
            if blk.upsamplers is not None:
                for up in blk.upsamplers:
                    x = up(x)
        s = u.conv_out(u.conv_act(u.conv_norm_out(x)))
        return s.reshape(b, m, *s.shape[1:])


# ---- seeded cases shared by the golden generator and the tests ----------------------------------------------------
def build_model(model_cls, config, seed: int = 0):
    """A seeded oracle UNet + the nine CP blocks with their zero-initialised projections redrawn."""
    from . import synth, unet as ounet
    st = torch.random.get_rng_state()
    torch.manual_seed(seed + 100)
    model = model_cls(ounet.build_unet(config, seed=seed + 1)).eval()
    torch.random.set_rng_state(st)
    synth.randomize_zero_init(model, seed + 3)
    return model


def step_inputs_cfg(m: int, hw: int, ctx_dim: int, seed: int = 0, t: int = 981):
    """One CFG-batched denoiser call as MvDiffusion.forward_cls_free makes it (MvDiffusion.py:58-80,95-121): latents
    and cameras duplicated, prompts [null; text] per view."""
    g = torch.Generator().manual_seed(seed)
    lat = torch.randn(1, m, 4, hw, hw, generator=g)
    text = torch.randn(1, 1, 77, ctx_dim, generator=g).repeat(1, m, 1, 1)
    null = torch.randn(1, 1, 77, ctx_dim, generator=g).repeat(1, m, 1, 1)
    K, R = horizon_cameras(m, batch=2, size=hw * 8)
    return dict(latents=torch.cat([lat] * 2), timestep=torch.full((2, m), t, dtype=torch.long),
                prompt_embd=torch.cat([null, text]), meta=dict(K=K, R=R))


def cpattn_case(block_cls, dim: int = 320, m: int = 8, h: int = 8, img: int = 512, seed: int = 7):
    """One CPAttn(dim) with redrawn zero-init weights on m horizon views of an h x h level of img x img images."""
    from . import synth
    torch.manual_seed(seed)
    blk = block_cls(dim, flag360=True).eval()
    holder = nn.Module()
    holder.cp_blocks = blk
    synth.randomize_zero_init(holder, seed + 4)
    x = torch.randn(m, dim, h, h, generator=torch.Generator().manual_seed(seed + 1))
    K, R = horizon_cameras(m, size=img)
    return blk, x, K, R


def sample_loop(model, latents, prompt_embd, K, R, guidance: float = 9.0, steps: int = 50, num_steps=None):
    """MvDiffusion.inference's loop (MvDiffusion.py:95-121) from given initial latents [1, m, 4, h, w]: CFG pair with
    prompts [null; text], DDIM on the SD-2 schedule; `num_steps` stops after the first few iterations."""
    from .sampler import DDIM
    sch = DDIM()
    sch.set_timesteps(steps)
    m = latents.shape[1]
    meta = dict(K=torch.cat([K] * 2), R=torch.cat([R] * 2))
    for t in sch.timesteps[:num_steps]:
        ts = torch.full((1, m), int(t), dtype=torch.long)
        eps = model(torch.cat([latents] * 2), torch.cat([ts] * 2), prompt_embd, meta)
        un, tx = eps.chunk(2)
        latents = sch.step(un + guidance * (tx - un), t, latents)
    return latents


# mp2e case: 8 horizon views of 64^2 uint8 images stitched into a 64 x 128 panorama (MvDiffusion.py:136-140)
MP2E_CASE = dict(m=8, hw=64, out_hw=(64, 128), fov=90.0)


def mp2e_inputs():
    c = MP2E_CASE
    rng = np.random.default_rng(11)
    imgs = rng.integers(0, 256, (c["m"], c["hw"], c["hw"], 3)).astype(np.uint8)
    theta = np.rad2deg(np.linspace(0, 2 * np.pi, c["m"], endpoint=False))
    return imgs, np.full(c["m"], c["fov"]), theta, np.zeros(c["m"])


TABLE_LEVELS = ((8, 512), (64, 512))  # (level side, image side); the 64^2 level is stored for every 8th query row / col


def _table_rows(h: int):
    return slice(None) if h <= 16 else slice(None, None, 8)


# ---- golden generator (reference checkout only) ---------------------------------------------------------------------
def load_reference():
    from . import ref_loader
    if not ref_loader.available():
        raise RuntimeError("the reference checkout is not available")
    for p in (str(ref_loader.SHIMS), str(ref_loader.REF)):  # p2e.py imports kornia: the oracle's shim
        if p not in sys.path:
            sys.path.insert(0, p)
    ns = types.SimpleNamespace()
    ns.MVGenModel = importlib.import_module("external.MVDiffusion.pano.MVGenModel")
    ns.modules = importlib.import_module("external.MVDiffusion.pano.modules")
    ns.utils = importlib.import_module("external.MVDiffusion.pano.utils")
    return ns


def _trunc10(a):
    return (np.ascontiguousarray(a, dtype=np.float32).view(np.uint32) & np.uint32(0xFFFFFC00)).view(np.float32)


def _ref_tables(ref, K, R, h, img):
    """Window positions / masks / xy_rel from the reference's own get_correspondences + get_key_value."""
    m = K.shape[1]
    corr = ref.utils.get_correspondences(R, K, img, img)
    s = img // h
    pos, mask, rel = [], [], []
    for i in range(m):
        idx = _neighbours(i, m)
        Rl, Kl = R[:, i:i + 1].repeat(1, 2, 1, 1).reshape(-1, 3, 3), K[:, i:i + 1].repeat(1, 2, 1, 1).reshape(-1, 3, 3)
        homo_r = (Kl @ torch.inverse(Rl) @ R[:, idx].reshape(-1, 3, 3) @ torch.inverse(K[:, idx].reshape(-1, 3, 3)))
        homo_r = homo_r.reshape(K.shape[0], 2, 3, 3)
        feat = torch.zeros(K.shape[0], 2, 1, h, h)
        _, _, xy, mk = ref.utils.get_query_value(feat[:, 0], feat, corr[:, i, idx], homo_r, img, img)
        xl = corr[:, i, idx][:, :, s // 2::s, s // 2::s] / s - 0.5                  # [B, 2, h, h, 2]
        off = torch.tensor([[di, dj] for di in (-1, 0, 1) for dj in (-1, 0, 1)], dtype=torch.float32)
        p = xl[:, :, None] + off[None, None, :, None, None]                         # [B, 2, 9, h, h, 2]
        pos.append(p.permute(0, 3, 4, 1, 2, 5).reshape(K.shape[0], h * h, 18, 2))
        mask.append(mk.permute(0, 2, 3, 1).reshape(K.shape[0], h * h, 18))
        rel.append(xy.permute(0, 2, 3, 1, 4).reshape(K.shape[0], h * h, 18, 2))
    return torch.stack(pos, 1), torch.stack(mask, 1), torch.stack(rel, 1)


def golden_c2(ref) -> float:
    """The SD-2-width denoiser at the default configuration (8 horizon views of 64^2 latents, CFG pair): ONE reference
    MultiViewBaseModel.forward on the host, stored with its 10 low significand bits cleared (like mvgen_c2.npz) so that
    the fixture stays under 1 MB."""
    from . import unet as ounet
    cfg = ounet.SD2_CONFIG
    model_r = build_model(ref.MVGenModel.MultiViewBaseModel, cfg)
    for mod in model_r.modules():
        if hasattr(mod, "use_checkpoint"):
            mod.use_checkpoint = False
    inp = step_inputs_cfg(8, 64, cfg["cross_attention_dim"])
    rs = model_r(**inp)
    np.savez_compressed(OUT / "mvdiff_c2.npz", sample=_trunc10(rs.numpy()))
    model_o = build_model(MultiViewBaseModel, cfg)
    model_o.load_state_dict(model_r.state_dict())
    del model_r
    err = (model_o(**inp) - rs).abs().max().item()
    print(f"  MultiViewBaseModel c2: max |oracle - reference| = {err:.3e} (max|ref| {rs.abs().max():.3e})")
    return err


def main() -> int:
    import argparse
    from . import unet as ounet
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", choices=["c2"])
    args = ap.parse_args()
    ref = load_reference()
    torch.set_grad_enabled(False)
    if args.only == "c2":
        return 0 if golden_c2(ref) < 1e-4 else 1
    worst = 0.0

    def report(name, a, b):
        nonlocal worst
        err = max((x.float() - y.float()).abs().max().item() for x, y in zip(a, b))
        print(f"  {name}: max |oracle - reference| = {err:.3e}")
        worst = max(worst, err)

    # 1. CPAttn geometry on the 8-view horizon ring
    K, R = horizon_cameras(8)
    out = dict(K=K[0].numpy(), R=R[0].numpy())
    for h, img in TABLE_LEVELS:
        rp, rm, rr = _ref_tables(ref, K, R, h, img)
        op, om_, orl = tables(K, R, h, img)
        report(f"tables {h}^2 positions / masks", [rp, rm], [op, om_])
        bits = (orl != rr).float().mean().item()
        print(f"  tables {h}^2: xy_rel bit-identical fraction {1 - bits:.4f}")
        worst = max(worst, bits)
        sel = _table_rows(h)
        keep = lambda t: t[0].reshape(8, h, h, *t.shape[3:])[:, sel, sel].numpy()
        out.update({f"pos_{h}": keep(rp), f"mask_{h}": keep(rm).astype(np.uint8), f"rel_{h}": keep(rr)})
    np.savez_compressed(OUT / "mvdiff_tables.npz", **out)

    # 2. one CPAttn(320) at the 8^2 level of 512^2 views (masked keys present, frequencies up to 2^79)
    blk_r, x, K, R = cpattn_case(ref.modules.CPAttn)
    blk_r.transformer.use_checkpoint = False
    y = blk_r(x, ref.utils.get_correspondences(R, K, 512, 512), 512, 512, R, K, 8)
    blk_o, _, _, _ = cpattn_case(CPAttn)
    blk_o.load_state_dict(blk_r.state_dict())
    report("CPAttn(320)", [y], [blk_o(x, None, 512, 512, R, K, 8)])
    np.savez_compressed(OUT / "mvdiff_cpattn.npz", out=_trunc10(y.numpy()))

    # 3. the whole denoiser with narrow UNets: 8 horizon views of 16 x 16 latents, CFG pair
    cfg = ounet.TINY_CONFIG
    model_r = build_model(ref.MVGenModel.MultiViewBaseModel, cfg)
    for mod in model_r.modules():
        if hasattr(mod, "use_checkpoint"):
            mod.use_checkpoint = False
    model_o = build_model(MultiViewBaseModel, cfg)
    model_o.load_state_dict(model_r.state_dict())
    inp = step_inputs_cfg(8, 16, cfg["cross_attention_dim"])
    rs = model_r(**inp)
    report("MultiViewBaseModel tiny", [rs], [model_o(**inp)])
    np.savez_compressed(OUT / "mvdiff_tiny.npz", sample=rs.numpy())

    # 4. panorama stitching (external/Perspective_and_Equirectangular/mp2e.py) as inference_and_save calls it: no
    # mode argument, which its numpy path hands to cv2.remap as interpolation None = INTER_NEAREST
    pe = importlib.import_module("external.Perspective_and_Equirectangular")
    imgs, fov, theta, phi = mp2e_inputs()
    np.savez_compressed(OUT / "mvdiff_mp2e.npz", pano=pe.mp2e(imgs, fov, theta, phi, MP2E_CASE["out_hw"]))
    print(f"worst oracle-vs-reference deviation: {worst:.3e}")
    return 0 if worst < 1e-4 else 1


if __name__ == "__main__":
    sys.exit(main())
