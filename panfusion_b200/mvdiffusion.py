"""MVDiffusion's denoiser behind the reference's interface (external/MVDiffusion/pano/MVGenModel.py, pano/modules.py).

`MultiViewBaseModel(unet, pers_cn=None)` and `CPAttn(dim, flag360=False)` keep the reference's attribute and parameter
names (`cp_blocks_encoder`, `cp_blocks_mid`, `cp_blocks_decoder`, `transformer.attn1.{to_q,to_k,to_v,to_out}`,
`transformer.ff.net.{0.proj,2}`, `transformer.norm1/2`, buffer `pe.freq_bands`), so a reference checkpoint loads with
`load_state_dict` or `checkpoint.load_reference_state_dict(prefix='mv_base_model.')`. The UNet is read once into
engine.UNetPack and runs as the same kernels as PanFusion's perspective branch; each CPAttn runs as

    LayerNorm(x + PE(0)) -> to_q                     pf_layernorm, tap-GEMM
    18 keys per pixel: bilinear window + PE, masked  pf_cpattn_gather (+ per-row LayerNorm statistics)
    norm1 folded into one K|V GEMM over 18 T rows    tap-GEMM with ln_stats
    softmax over the 18 keys                         pf_cpattn_attn
    to_out + x, x + FF(norm2(x))                     eppa.block_tail

The sample positions, masks and key positional arguments are per (camera set, level) tables built by pf_cpattn_tables
and cached (`CPTables`). There is no PyTorch fallback: without a CUDA device and the built library the forward raises.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn as nn
from torch import Tensor

from . import _lib, ops
from .engine import Branch, Img, UNetPack, _Lin, _LinLN, _Norm, img_from_nchw
from .eppa import _Block, block_tail, pack_block
from .sampler import PanFusionSampler


class _PosEmbedding(nn.Module):  # external/MVDiffusion/modules/transformer.py:169-189 (logscale): frequency table only
    def __init__(self, n_freqs):
        super().__init__()
        base = 2 if n_freqs <= 80 else 5000 ** (1 / (n_freqs / 2.5))
        self.register_buffer("freq_bands", base ** torch.linspace(0, n_freqs - 1, n_freqs)[None, None])


def homographies(K: Tensor, R: Tensor) -> tuple[Tensor, Tensor]:
    """K, R [G, m, 3, 3] -> (homo_l, homo_r) fp32 [G, m, 2, 3, 3] for the neighbours (i-1) mod m and (i+1) mod m,
    computed on the host with the reference's fp32 operations and operand order (pano/utils.py:14-27,
    pano/modules.py:44-58), so that the tables reproduce its correspondences bit for bit."""
    K, R = K.detach().to("cpu", torch.float32), R.detach().to("cpu", torch.float32)
    G, m = K.shape[:2]
    hl = torch.empty((G, m, 2, 3, 3))
    hr = torch.empty((G, m, 2, 3, 3))
    for i in range(m):
        idx = [(i - 1 + m) % m, (i + 1) % m]
        for n, j in enumerate(idx):  # get_correspondences: one (i, j) pair at a time, batch G
            Rr, Kr, Rl, Kl = R[:, j], K[:, j], R[:, i], K[:, i]
            hl[:, i, n] = Kr @ torch.inverse(Rr) @ Rl @ torch.inverse(Kl)
        # CPAttn.forward: both neighbours in one batch of 2 G
        Rr, Kr = R[:, idx].reshape(-1, 3, 3), K[:, idx].reshape(-1, 3, 3)
        Rl, Kl = R[:, i:i + 1].repeat(1, 2, 1, 1).reshape(-1, 3, 3), K[:, i:i + 1].repeat(1, 2, 1, 1).reshape(-1, 3, 3)
        hr[:, i] = (Kl @ torch.inverse(Rl) @ Rr @ torch.inverse(Kr)).reshape(G, 2, 3, 3)
    return hl, hr


class CPTables:
    """Per (camera set, level) cache of pf_cpattn_tables' sample positions / masks. Cameras do not change across the
    denoising steps, and the two CFG halves carry the same cameras (MvDiffusion.py:62-66), so one entry per level serves
    the whole sampling loop. LRU-bounded over camera sets, like eppa.CameraTables."""

    def __init__(self, max_camera_sets: int = 16):
        self.max_camera_sets = max_camera_sets
        self._tables: dict = {}
        self._lru: list = []
        self._keys: dict = {}

    def camera_key(self, K: Tensor, R: Tensor) -> tuple:
        """-> key of the camera set; identical cameras in every batch element are kept once. Reading K and R costs a
        device-to-host copy when they live on the GPU; the result is remembered per tensor identity (address and
        version, the tensors held alive), so a sampling loop that passes the same camera tensors pays it once."""
        ident = (K.data_ptr(), K._version, R.data_ptr(), R._version, tuple(K.shape), tuple(R.shape), str(K.device))
        hit = self._keys.get(ident)
        if hit is not None:
            return hit[0]
        Kc, Rc = K.detach().to("cpu", torch.float32), R.detach().to("cpu", torch.float32)
        if all(torch.equal(Kc[b], Kc[0]) and torch.equal(Rc[b], Rc[0]) for b in range(Kc.shape[0])):
            Kc, Rc = Kc[:1], Rc[:1]
        out = (tuple(Kc.reshape(-1).tolist()), tuple(Rc.reshape(-1).tolist()), tuple(Kc.shape))
        if len(self._keys) >= 8:
            self._keys.clear()
        self._keys[ident] = (out, K, R)
        return out

    def get(self, key: tuple, h: int, w: int, img_size: int, dev) -> tuple[Tensor, Tensor]:
        """Tables of camera set `key` (from camera_key) at the h x w level of img_size^2 views."""
        if key in self._lru:
            self._lru.remove(key)
        self._lru.append(key)
        while len(self._lru) > self.max_camera_sets:
            old = self._lru.pop(0)
            for k in [k for k in self._tables if k[0] == old]:
                del self._tables[k]
        k = (key, h, w, img_size, dev)
        if k not in self._tables:
            shape = key[2]
            hl, hr = homographies(torch.tensor(key[0]).reshape(shape), torch.tensor(key[1]).reshape(shape))
            self._tables[k] = ops.cpattn_tables(hl.to(dev).contiguous(), hr.to(dev).contiguous(), h, w, img_size)
        return self._tables[k]

    def tensors_of(self, key: tuple) -> list:
        """Every cached table of camera set `key`: whoever captured their addresses (a CUDA graph) holds these, so
        that an LRU eviction cannot free memory a replay still reads."""
        return [t for k, v in self._tables.items() if k[0] == key for t in v]

    def clear(self) -> None:
        self._tables.clear()
        self._lru.clear()
        self._keys.clear()


class CPAttn(nn.Module):
    """external/MVDiffusion/pano/modules.py:22-86. `flag360` is stored and unused, as in the reference."""

    def __init__(self, dim, flag360=False):
        super().__init__()
        self.flag360 = flag360
        self.dim = dim
        self.transformer = _Block(dim, dim // 32)
        self.pe = _PosEmbedding(dim // 4)
        self._packed = None
        self.tables = CPTables()  # MultiViewBaseModel replaces this with one shared cache

    def _pack(self, dev, dt):
        if self._packed is not None and self._packed["key"] == (dev, dt):
            return self._packed
        t = self.transformer
        a = t.attn1
        w = pack_block(t, dev, dt)
        n = self.dim // 4
        w.update(
            q=_Lin(a.to_q.weight, None, dev, dt),
            kv_ln=_LinLN(torch.cat([a.to_k.weight, a.to_v.weight], 0), None, t.norm1, dev, dt),
            ln1=_Norm(t.norm1, dev),
            # PosEmbedding(0) = [sin 0 (2N), cos 0 (2N)]: the query's constant PE row (modules.py:74-75)
            query_pe=torch.cat([torch.zeros(2 * n), torch.ones(2 * n)])[None].to(dev).contiguous(),
            freq=self.pe.freq_bands.detach().reshape(-1).to(dev, torch.float32).contiguous())
        self._packed = w
        return w

    def invalidate(self):
        self._packed = None

    def forward_tokens(self, x: Img, m: int, cam_key: tuple, img_size: int) -> Img:
        """x: (b*m) views of h x w tokens; cam_key = tables.camera_key(K, R) of the [b, m, 3, 3] cameras; img_size =
        image side in pixels (8 x the latent side)."""
        dev, dt = x.t.device, x.t.dtype
        w = self._pack(dev, dt)
        C, T = self.dim, x.t.shape[0]
        B = x.N // m
        pos, mask = self.tables.get(cam_key, x.H, x.W, img_size, dev)
        new = lambda r, n: torch.empty((r, n), dtype=dt, device=dev)
        qn = ops.layernorm(x.t, w["ln1"].g, w["ln1"].b, w["ln1"].eps, w["query_pe"])
        q = ops.gemm_taps(qn, w["q"].w, new(T, C), M=T, Kc=C)
        keys, st = ops.cpattn_gather(x.t, B, m, x.H, x.W, pos, mask, w["freq"])
        rows = keys.shape[0]
        kv = ops.gemm_taps(keys, w["kv_ln"].w, new(rows, 2 * C), M=rows, Kc=C, bias=w["kv_ln"].b,
                           ln=(st, w["kv_ln"].colsum, w["kv_ln"].eps))
        o = ops.cpattn_attn(q, kv, new(T, C), 32 ** -0.5)
        return Img(block_tail(w, o, x.t, T), x.N, x.H, x.W)

    def forward(self, x: Tensor, correspondences, img_h: int, img_w: int, R: Tensor, K: Tensor, m: int,
                compute_dtype: torch.dtype | None = None) -> Tensor:
        """The reference's signature (modules.py:30). `correspondences` is not read: the tables kernel derives the same
        positions from K and R."""
        _lib.require_cuda(x)
        if img_h != img_w:
            raise ValueError("CPAttn: square images only (the reference samples both axes with img_h)")
        dt = compute_dtype or (x.dtype if x.dtype in (torch.float16, torch.bfloat16) else torch.bfloat16)
        out = self.forward_tokens(img_from_nchw(x, dt), m, self.tables.camera_key(K, R), img_h)
        return out.nchw().to(x.dtype).contiguous()


class MultiViewBaseModel(nn.Module):
    """external/MVDiffusion/pano/MVGenModel.py:8-155 on the sm_90a kernels."""

    def __init__(self, unet, pers_cn=None, compute_dtype=torch.bfloat16):
        super().__init__()
        if pers_cn is not None:
            raise NotImplementedError("MVDiffusion's layout ControlNet (pers_cn) is not supported")
        self.unet = unet
        self.pers_cn = pers_cn
        self.compute_dtype = compute_dtype
        self.cp_blocks_encoder = nn.ModuleList(
            [CPAttn(blk.resnets[-1].out_channels, flag360=True) for blk in unet.down_blocks])
        self.cp_blocks_mid = CPAttn(unet.mid_block.resnets[-1].out_channels, flag360=True)
        self.cp_blocks_decoder = nn.ModuleList(
            [CPAttn(blk.resnets[-1].out_channels, flag360=True) for blk in unet.up_blocks])
        self.trainable_parameters = [(list(self.cp_blocks_mid.parameters())
                                      + list(self.cp_blocks_decoder.parameters())
                                      + list(self.cp_blocks_encoder.parameters()), 1.0)]
        tables = CPTables()
        for blk in self._cp_blocks():
            blk.tables = tables
        self._branch = None
        self.last_camera_key = None

    def _cp_blocks(self):
        return [*self.cp_blocks_encoder, self.cp_blocks_mid, *self.cp_blocks_decoder]

    def prepare(self, device=None, dtype=None) -> "MultiViewBaseModel":
        """Pack all weights for the kernels (call again after loading new weights)."""
        device = torch.device(device or "cuda")
        if device.type == "cuda" and device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        dtype = dtype or self.compute_dtype
        _lib.check(_lib.lib().pf_check_device())
        self._branch = (Branch(UNetPack(self.unet, device, dtype), circular=False), device)
        for blk in self._cp_blocks():
            blk.invalidate()
        return self

    def invalidate(self):
        self._branch = None

    @torch.no_grad()
    def update_text(self, prompt_embd: Tensor) -> None:
        """Re-project the text K/V for new prompt embeddings of the same shape into the buffer the previous call used: a
        captured CUDA graph of `forward` reads it by address and does not contain the (cached) text projection."""
        if self._branch is not None:
            self._branch[0].set_text(prompt_embd.flatten(0, 1),
                                     (prompt_embd.data_ptr(), prompt_embd._version, tuple(prompt_embd.shape)))

    @torch.no_grad()
    def forward(self, latents: Tensor, timestep: Tensor, prompt_embd: Tensor, meta: dict, pers_layout_cond=None):
        _lib.require_cuda(latents)
        if self._branch is None or self._branch[1] != latents.device:
            self.prepare(latents.device)
        br = self._branch[0]
        b, m, _, h, w = latents.shape
        img_h, img_w = h * 8, w * 8
        if img_h != img_w:
            raise ValueError("MultiViewBaseModel: square views only (CPAttn samples both axes with img_h)")
        tables = self.cp_blocks_mid.tables
        cam_key = tables.camera_key(meta["K"], meta["R"])  # once per forward, shared by the nine CP blocks
        self.last_camera_key = cam_key
        br.set_timesteps(timestep.reshape(-1))  # MVGenModel.py:46-48
        br.set_text(prompt_embd.flatten(0, 1), (prompt_embd.data_ptr(), prompt_embd._version, tuple(prompt_embd.shape)))

        def cp(block, x):
            return block.forward_tokens(x, m, cam_key, img_h) if m > 1 else x

        x = br.conv_in(latents.flatten(0, 1))  # MVGenModel.py:62-63
        skips = [x]
        for i, blk in enumerate(br.p.down):  # MVGenModel.py:67-89: skips are taken BEFORE the CP block
            for j, r in enumerate(blk["resnets"]):
                x = br.resnet(x, r)
                if blk["attns"] is not None:
                    x = br.transformer(x, blk["attns"][j])
                skips.append(x)
            x = cp(self.cp_blocks_encoder[i], x)
            if blk["down"] is not None:
                for d in blk["down"]:
                    x = br.downsample(x, d)
                skips.append(x)
        x = br.resnet(x, br.p.mid["resnets"][0])  # MVGenModel.py:102-113
        x = cp(self.cp_blocks_mid, x)
        for i, at in enumerate(br.p.mid["attns"]):
            x = br.transformer(x, at)
            x = br.resnet(x, br.p.mid["resnets"][i + 1])
        for i, blk in enumerate(br.p.up):  # MVGenModel.py:120-148: CP block BEFORE the upsampler
            for j, r in enumerate(blk["resnets"]):
                x = br.resnet(x, r, skip=skips.pop())
                if blk["attns"] is not None:
                    x = br.transformer(x, blk["attns"][j])
            x = cp(self.cp_blocks_decoder[i], x)
            if blk["up"] is not None:
                for u in blk["up"]:
                    x = br.upsample(x, u)
        s = br.conv_out(x)  # MVGenModel.py:151-155
        return s.reshape(b, m, *s.shape[1:]).to(latents.dtype)


class MvDiffusionSampler(PanFusionSampler):
    """MvDiffusion.inference (models/pano/MvDiffusion.py:95-121) and the panorama of inference_and_save (:123-146):
    CFG pair [null; text], DDIM on the SD-2 schedule through pf_cfg_ddim_step_dev, VAE decode + tensor_to_image of the
    views, pf_mp2e stitching. There is no rotation, so one captured CUDA graph serves every step; the graph, static
    buffer and table-ownership machinery is PanFusionSampler's."""

    _state_keys = ("latents",)

    def __init__(self, mv_base_model: MultiViewBaseModel, guidance_scale: float = 9.0, diff_timestep: int = 50,
                 use_cuda_graph: bool = True):
        super().__init__(mv_base_model, guidance_scale, diff_timestep, rot_diff=0.0, use_cuda_graph=use_cuda_graph)

    @torch.no_grad()
    def start(self, latents: Tensor, prompt_embd: Tensor, K: Tensor, R: Tensor) -> None:
        """latents [1, m, 4, h, w]; prompt_embd [2, m, 77, C] = [null; text] per view (MvDiffusion.py:105-106);
        K, R [1, m, 3, 3]."""
        if latents.shape[0] != 1:
            raise NotImplementedError(f"MvDiffusionSampler runs one panorama per call; got batch {latents.shape[0]}")
        dev = latents.device
        m = latents.shape[1]
        self.scheduler.set_timesteps(self.diff_timestep)
        sig = (str(dev), tuple(latents.shape), tuple(prompt_embd.shape), self.diff_timestep,
               id(self.mv_base_model._branch))
        if self._st is not None and getattr(self, "_sig", None) == sig:
            st = self._st  # same shapes: the captured graph reads these buffers by address
            st["latents"].copy_(latents)
            st["prompt"].copy_(prompt_embd)
            if self._graphs:
                self.mv_base_model.update_text(st["prompt"])
        else:
            coefs = torch.tensor([self.scheduler.coefficients(int(t)) for t in self.scheduler.timesteps],
                                 dtype=torch.float32)
            st = dict(latents=latents.to(torch.float32).contiguous().clone(),
                      timestep=torch.zeros((1, m), dtype=torch.float32, device=dev),
                      prompt=prompt_embd.contiguous().clone(), coef=torch.zeros(2, dtype=torch.float32, device=dev),
                      coef_table=coefs.to(dev), ts_table=self.scheduler.timesteps.to(dev, torch.float32))
            st["latents_next"] = torch.empty_like(st["latents"])
            self._st, self._sig = st, sig
            self._graphs = {}
        # the CFG pair's cameras (MvDiffusion.py:62-66), read on the host once (CPTables.camera_key)
        self._cameras = {k: torch.cat([v.detach().to("cpu", torch.float32)] * 2) for k, v in (("K", K), ("R", R))}
        self._curr_rot = 0.0

    def _step_body(self, st, cameras):
        dup = lambda t: torch.cat([t] * 2)
        eps = self.mv_base_model(dup(st["latents"]), dup(st["timestep"]), st["prompt"], cameras)
        ops.cfg_ddim_step_dev(st["latents"], eps.contiguous(), st["latents_next"], self.guidance_scale, st["coef"])
        st["latents"].copy_(st["latents_next"])

    def _graph_key(self, st, cameras) -> tuple:
        return (self.mv_base_model.cp_blocks_mid.tables.camera_key(cameras["K"], cameras["R"]),
                tuple(st["latents"].shape), st["latents"].data_ptr(), st["prompt"].data_ptr())

    def _graph_tables(self, cameras) -> list:
        tables = self.mv_base_model.cp_blocks_mid.tables
        return tables.tensors_of(tables.camera_key(cameras["K"], cameras["R"]))

    @torch.no_grad()
    def finish(self) -> Tensor:
        return self._st["latents"].clone()

    @torch.no_grad()
    def denoise(self, latents: Tensor, prompt_embd: Tensor, K: Tensor, R: Tensor, num_steps=None) -> Tensor:
        self.start(latents, prompt_embd, K, R)
        for i in range(num_steps or self.diff_timestep):
            self.step(i)
        return self.finish().to(latents.dtype)

    @torch.no_grad()
    def inference(self, K: Tensor, R: Tensor, prompt_embd: Tensor, vae, fov_deg, theta_deg, phi_deg, pano_hw,
                  image_hw: int = 512, device="cuda", generator=None, latents: Optional[Tensor] = None,
                  num_steps: Optional[int] = None):
        """randn latents -> the denoising loop -> decode_latent + tensor_to_image -> mp2e. Returns (views uint8
        [1, m, h, w, 3], panorama uint8 [H, W, 3]) on the device. `vae` is a panfusion_b200.vae.VAEDecoder; the
        camera angles (degrees, per view) are those of batch['cameras'] that inference_and_save stitches with."""
        from . import vae as pv
        m = K.shape[1]
        if latents is None:
            latents = torch.randn(1, m, 4, image_hw // 8, image_hw // 8, generator=generator, device=device)
        lat = self.denoise(latents.to(device), prompt_embd.to(device), K, R, num_steps=num_steps)
        images = ops.tensor_to_image(pv.decode_latent(lat, vae))
        return images, ops.mp2e(images[0].contiguous(), fov_deg, theta_deg, phi_deg, pano_hw)
