"""The sampling loop around the denoiser behind the reference's method names.

Reference: models/pano/PanFusion.py:30-43 (init_noise), :100-112 (forward_cls_free), :114-123 (rotate_latent),
:146-164 (the 50-step loop), models/pano/PanoGenerator.py:240-269 (CFG pair / combine, latent roll) and diffusers
DDIMScheduler [3P] (SD-2 config). Per step the reference runs: torch.roll + theta += 90, torch.cat x2 of every
input, the denoiser, the CFG combine, two scheduler.step calls. Here the combine, both DDIM updates and the NEXT
step's roll are one tiny kernel per latent (pf_cfg_ddim_step_dev), the view noise is the e2p-nearest kernel, and
— because every shape is static and all camera-dependent tables are cached — the whole step is captured once per
rotation phase into a CUDA graph and replayed.
"""
from __future__ import annotations

import math
from typing import Optional

import numpy as np
import torch
from torch import Tensor

from . import geometry, ops


class DDIMSchedule:
    """Coefficients of diffusers DDIMScheduler for the SD-2 config (scaled_linear betas, steps_offset 1, epsilon
    prediction, eta 0, set_alpha_to_one False, 'leading' spacing) [3P]."""

    def __init__(self, num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, steps_offset=1):
        betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float32) ** 2
        self.alphas_cumprod = torch.cumprod(1.0 - betas, dim=0)
        self.final_alpha_cumprod = self.alphas_cumprod[0]
        self.num_train_timesteps, self.steps_offset = num_train_timesteps, steps_offset
        self.timesteps: Optional[Tensor] = None
        self.num_inference_steps = 0

    def set_timesteps(self, n: int) -> None:
        self.num_inference_steps = n
        ratio = self.num_train_timesteps // n
        self.timesteps = torch.from_numpy((np.arange(0, n) * ratio).round()[::-1].copy().astype(np.int64)
                                          + self.steps_offset)

    def alphas(self, t: int) -> tuple[float, float]:
        prev_t = t - self.num_train_timesteps // self.num_inference_steps
        a_t = float(self.alphas_cumprod[t])
        a_prev = float(self.alphas_cumprod[prev_t]) if prev_t >= 0 else float(self.final_alpha_cumprod)
        return a_t, a_prev

    def coefficients(self, t: int) -> tuple[float, float]:
        """x_prev = c_x * x + c_eps * eps."""
        a_t, a_prev = self.alphas(t)
        sa = math.sqrt(a_prev / a_t)
        return sa, math.sqrt(1.0 - a_prev) - sa * math.sqrt(1.0 - a_t)


def init_noise(bs, equi_h, equi_w, pers_h, pers_w, cameras, device, generator=None):
    """PanFusion.init_noise (PanFusion.py:30-43): one panorama noise field per sample; every view's noise is its
    nearest-neighbour e2p resampling. Shared by the sampler and the training-step forward (training.py)."""
    cams = {k: v.flatten(0, 1) for k, v in cameras.items()}
    m = len(cams["FoV"]) // bs
    pano_noise = torch.randn(bs, 1, 4, equi_h, equi_w, device=device, generator=generator)
    noise = geometry.e2p(pano_noise[:, 0], cams["FoV"], cams["theta"], cams["phi"], (pers_h, pers_w), mode="nearest",
                         views_per_image=m)  # = e2p of the panorama expanded to its m views (PanFusion.py:33-37)
    return pano_noise, noise.reshape(bs, m, *noise.shape[1:])


class PanFusionSampler:
    _state_keys = ("latents", "pano")  # the static buffers a step updates in place (restored after a warm-up step)

    def __init__(self, mv_base_model, guidance_scale: float = 9.0, diff_timestep: int = 50, rot_diff: float = 90.0,
                 use_cuda_graph: bool = True):
        self.mv_base_model = mv_base_model
        self.guidance_scale, self.diff_timestep, self.rot_diff = guidance_scale, diff_timestep, rot_diff
        self.scheduler = DDIMSchedule()
        self.use_cuda_graph = use_cuda_graph
        self._graphs = {}
        self.max_graphs = 16   # captured steps kept (one per rotation phase and rig); oldest dropped first
        self._pool = None
        self.launches_per_step = None
        self._st = None
        self._cond_phases = None

    # ---- PanFusion.py:30-43 -------------------------------------------------------------------------
    def init_noise(self, bs, equi_h, equi_w, pers_h, pers_w, cameras, device, generator=None):
        return init_noise(bs, equi_h, equi_w, pers_h, pers_w, cameras, device, generator)

    # ---- PanFusion.py:114-123 / PanoGenerator.py:264-269 ------------------------------------------
    def rotate_latent(self, pano_latent, cameras, degree=None):
        degree = self.rot_diff if degree is None else degree
        if degree % 360 == 0:
            return pano_latent, cameras
        pano_latent = torch.roll(pano_latent, int(degree / 360 * pano_latent.shape[-1]), dims=-1)
        cameras = dict(cameras)
        cameras["theta"] = (cameras["theta"] + degree) % 360
        return pano_latent, cameras

    # ---- PanFusion.py:100-112 -----------------------------------------------------------------------
    @torch.no_grad()
    def forward_cls_free(self, latents, pano_latent, timestep, prompt_embd, pano_prompt_embd, cameras,
                         pers_layout_cond=None, pano_layout_cond=None):
        dup = lambda t: torch.cat([t] * 2) if t is not None else None
        cams2 = {k: dup(v) for k, v in cameras.items()}
        eps, pano_eps = self.mv_base_model(dup(latents), dup(pano_latent), dup(timestep), prompt_embd,
                                           pano_prompt_embd, cams2, dup(pers_layout_cond), dup(pano_layout_cond))
        comb = lambda e: e[:e.shape[0] // 2] + self.guidance_scale * (e[e.shape[0] // 2:] - e[:e.shape[0] // 2])
        return comb(eps), comb(pano_eps)

    # ---- one iteration of PanFusion.py:146-162 on static buffers ------------------------------------
    def _step_body(self, st, cameras):
        """st: dict of static device tensors. The pano latent in st is ALREADY rotated for this step; the DDIM
        kernel writes the next step's latent pre-rotated by rot_diff."""
        dup = lambda t: torch.cat([t] * 2)
        cams2 = {k: dup(v) for k, v in cameras.items()}
        eps, pano_eps = self.mv_base_model(dup(st["latents"]), dup(st["pano"]), dup(st["timestep"]), st["prompt"],
                                           st["pano_prompt"], cams2, st.get("pers_cond"), st.get("pano_cond"))
        ops.cfg_ddim_step_dev(st["latents"], eps.contiguous(), st["latents_next"], self.guidance_scale, st["coef"])
        W = st["pano"].shape[-1]
        ops.cfg_ddim_step_dev(st["pano"], pano_eps.contiguous(), st["pano_next"], self.guidance_scale, st["coef"],
                              roll=int(self.rot_diff / 360 * W) % W)
        st["latents"].copy_(st["latents_next"])
        st["pano"].copy_(st["pano_next"])

    # ---- the hot loop (PanFusion.py:146-164) as start / step / finish ---------------------------------
    @torch.no_grad()
    def start(self, latents: Tensor, pano_latent: Tensor, prompt_embd: Tensor, pano_prompt_embd: Tensor,
              cameras: dict, pers_layout_cond: Optional[Tensor] = None,
              pano_layout_cond: Optional[Tensor] = None) -> None:
        """Bind static buffers. prompt_embd [2, m, 77, C] / pano_prompt_embd [2, 1, 77, C] are the CFG concatenations
        [null; text] (PanFusion.py:135-138); cameras: dict of tensors [1, m] (CPU or CUDA). Layout conditions
        (ControlNet): pano_layout_cond [1, 1, 3, 8H, 8W] is rolled by rot_diff EVERY step like the latent
        (PanFusion.py:152-153); pers_layout_cond [1, m, 3, 8h, 8w] is passed through unchanged (:103-104)."""
        dev = latents.device
        self.scheduler.set_timesteps(self.diff_timestep)
        if latents.shape[0] != 1:
            raise NotImplementedError("PanFusionSampler runs one panorama per call (batch 1, like `main.py predict`); "
                                      f"got batch {latents.shape[0]}")
        m = latents.shape[1]
        W = pano_latent.shape[-1]
        self._roll = int(self.rot_diff / 360 * W) if self.rot_diff % 360 else 0
        dup = lambda t: torch.cat([t] * 2).contiguous()
        # Static buffers and captured graphs are kept ACROSS calls: a new image of the same shapes copies its inputs into
        # the existing buffers (the graphs read them by address) and re-projects the text K/V in place. Layout
        # conditions carry cached ControlNet features bound to tensor identities, so conditioned runs start afresh.
        sig = (str(dev), tuple(latents.shape), tuple(pano_latent.shape), tuple(prompt_embd.shape),
               tuple(pano_prompt_embd.shape), self.diff_timestep, self.rot_diff,
               id(getattr(self.mv_base_model, "_branches", None)))
        reuse = (getattr(self, "_st", None) is not None and getattr(self, "_sig", None) == sig
                 and pers_layout_cond is None and pano_layout_cond is None and "pers_cond" not in self._st
                 and self._cond_phases is None)
        if reuse:
            st = self._st
            st["latents"].copy_(latents)
            st["pano"].copy_(torch.roll(pano_latent.to(torch.float32), self._roll, dims=-1))
            st["prompt"].copy_(prompt_embd)
            st["pano_prompt"].copy_(pano_prompt_embd)
            if self._graphs:
                self.mv_base_model.update_text(st["prompt"], st["pano_prompt"])
        else:
            coefs = torch.tensor([self.scheduler.coefficients(int(t)) for t in self.scheduler.timesteps],
                                 dtype=torch.float32)
            st = dict(latents=latents.to(torch.float32).contiguous().clone(),
                      # the rotation of the first step (PanFusion.py:149); later ones are fused into the DDIM kernel
                      pano=torch.roll(pano_latent.to(torch.float32), self._roll, dims=-1).contiguous(),
                      timestep=torch.zeros((1, m), dtype=torch.float32, device=dev),
                      prompt=prompt_embd.contiguous().clone(), pano_prompt=pano_prompt_embd.contiguous().clone(),
                      coef=torch.zeros(2, dtype=torch.float32, device=dev),
                      coef_table=coefs.to(dev), ts_table=self.scheduler.timesteps.to(dev, torch.float32))
            st["latents_next"], st["pano_next"] = torch.empty_like(st["latents"]), torch.empty_like(st["pano"])
            if pers_layout_cond is not None:
                st["pers_cond"] = dup(pers_layout_cond.to(dev))
            self._cond_phases = None
            if pano_layout_cond is not None:
                # the rolled conditions repeat with a short period (4 for 90 degrees): keep every phase as its own
                # tensor, so the ControlNet's conditioning embedding is computed once per phase and cached on the
                # tensor identity
                Wc = pano_layout_cond.shape[-1]
                r = int(self.rot_diff / 360 * Wc) % Wc if self.rot_diff % 360 else 0
                period = Wc // math.gcd(Wc, r) if r else 1
                if period > 8:
                    raise NotImplementedError(f"layout condition with rot_diff={self.rot_diff}: {period} distinct rolls")
                self._cond_phases = [dup(torch.roll(pano_layout_cond.to(dev), (k + 1) * r, dims=-1)) for k in range(period)]
            self._st, self._sig = st, sig
            self._graphs = {}
        self._cameras = {k: v.detach().to("cpu", torch.float32) for k, v in cameras.items()}
        self._curr_rot = 0.0
        self._n_rot = 0

    @torch.no_grad()
    def step(self, i: int) -> None:
        """Iteration i of the loop: rotate (cameras here, latent already rotated), CFG forward, DDIM updates."""
        st = self._st
        self._curr_rot += self.rot_diff
        if self.rot_diff % 360:
            self._cameras = dict(self._cameras)
            self._cameras["theta"] = (self._cameras["theta"] + self.rot_diff) % 360
        st["timestep"].copy_(st["ts_table"][i].expand_as(st["timestep"]))
        st["coef"].copy_(st["coef_table"][i])
        if self._cond_phases is not None:
            self._n_rot = getattr(self, "_n_rot", 0)
            st["pano_cond"] = self._cond_phases[self._n_rot % len(self._cond_phases)]
            self._n_rot += 1
        self._run_step(st, self._cameras)

    @torch.no_grad()
    def finish(self, rotate_back: bool = True):
        """-> (latents, pano_latent). rotate_back applies PanFusion.py:164 (roll by -sum of rotations); without it the
        panorama is returned in the last step's rotated frame (what the loop variable holds in the reference)."""
        st = self._st
        W = st["pano"].shape[-1]
        shift = -self._roll  # the DDIM kernel pre-rotated for a step that never ran
        if rotate_back and self.rot_diff % 360:
            shift += int(-self._curr_rot / 360 * W)
        return st["latents"].clone(), torch.roll(st["pano"], shift % W, dims=-1)

    @torch.no_grad()
    def denoise(self, latents, pano_latent, prompt_embd, pano_prompt_embd, cameras, num_steps=None, start_step=0,
                rotate_back=True, pers_layout_cond=None, pano_layout_cond=None):
        self.start(latents, pano_latent, prompt_embd, pano_prompt_embd, cameras, pers_layout_cond, pano_layout_cond)
        for i in range(start_step, start_step + (num_steps or self.diff_timestep)):
            self.step(i)
        lat, pano = self.finish(rotate_back)
        return lat.to(latents.dtype), pano.to(pano_latent.dtype)

    # ---- PanFusion.inference (PanFusion.py:125-172) after the text encoder ---------------------------------
    @torch.no_grad()
    def inference(self, cameras, prompt_embd, pano_prompt_embd, vae, pano_hw, pers_hw, device="cuda", generator=None,
                  pano_noise: Optional[Tensor] = None, pano_layout_cond: Optional[Tensor] = None, latent_pad: int = 8,
                  num_steps: Optional[int] = None, pers_layout_cond: Optional[Tensor] = None):
        """init_noise -> the denoising loop -> rotate back -> VAE decode (views: plain; panorama: circularly padded
        latent, PanFusion.py:166-172) -> tensor_to_image. Returns (images uint8 [1, m, h, w, 3], pano uint8
        [1, 1, H, W, 3]) like the reference. `pers_layout_cond` / `pano_layout_cond` are
        batch['images_layout_cond'] / batch['pano_layout_cond'] (PanFusion.py:155-157). `vae` is a panfusion_b200.vae.VAEDecoder; prompt embeddings are the CFG
        concatenations [null; text] (the CLIP text encoder is outside this path). `pano_noise` [1, 1, 4, H/8, W/8]
        overrides the random draw (the view noise is always its e2p-nearest resampling)."""
        from . import vae as pv
        if pano_noise is None:
            pano_noise, noise = self.init_noise(1, *pano_hw, *pers_hw, cameras, device, generator)
        else:
            cams = {k: v.flatten(0, 1) for k, v in cameras.items()}
            m = len(cams["FoV"])
            pano_noise = pano_noise.to(device)
            noise = geometry.e2p(pano_noise[:, 0], cams["FoV"], cams["theta"], cams["phi"], tuple(pers_hw), mode="nearest",
                                 views_per_image=m)[None]
        lat, pano = self.denoise(noise, pano_noise, prompt_embd.to(device), pano_prompt_embd.to(device), cameras,
                                 num_steps=num_steps, pers_layout_cond=pers_layout_cond,
                                 pano_layout_cond=pano_layout_cond)
        images = pv.tensor_to_image(pv.decode_latent(lat, vae))
        pano_img = pv.tensor_to_image(pv.decode_pano(pano, vae, latent_pad))
        return images, pano_img

    def _graph_key(self, st, cameras) -> tuple:
        """What a captured step depends on besides the contents of its static buffers."""
        return (tuple(cameras["theta"].reshape(-1).tolist()), tuple(cameras["phi"].reshape(-1).tolist()),
                tuple(cameras["FoV"].reshape(-1).tolist()), tuple(st["latents"].shape), tuple(st["pano"].shape),
                st["latents"].data_ptr(), st["pano"].data_ptr(), st["prompt"].data_ptr(),
                st["pano_cond"].data_ptr() if "pano_cond" in st else 0)

    def _graph_tables(self, cameras) -> list:
        """The cached camera tables a captured step reads by address."""
        tables = getattr(getattr(self.mv_base_model, "cp_blocks_mid", None), "tables", None)
        if tables is None:
            return []
        cam2 = {k: torch.cat([v] * 2).flatten(0, 1) for k, v in cameras.items()}
        return tables.tensors_of(tables.camera_key(cam2))

    def _run_step(self, st, cameras):
        par = getattr(self.mv_base_model, "_par", None)
        self._steps_run = getattr(self, "_steps_run", 0) + 1
        if not self.use_cuda_graph:
            self.mv_base_model.par_slot = self._steps_run % 2  # consecutive steps: different receive buffers
            l0 = ops.LAUNCHES
            self._step_body(st, cameras)
            self.launches_per_step = ops.LAUNCHES - l0
            return
        key = self._graph_key(st, cameras)
        if par is not None and not (self.rot_diff % 360):
            key += (self._steps_run % 2,)  # a single rotation phase: still alternate between two graphs / buffer sets
        entry = self._graphs.get(key)
        if entry is None:
            # eager warm-up builds the camera tables / packs weights / sets kernel attributes, then capture
            snap = {k: st[k].clone() for k in self._state_keys}
            self._slot_seq = getattr(self, "_slot_seq", 1) + 1
            self.mv_base_model.par_slot = self._slot_seq  # this graph's own all-gather receive buffers
            self._step_body(st, cameras)
            torch.cuda.synchronize()
            if par is not None and getattr(par, "device_gather", False) and hasattr(par, "group"):
                # every rank has CONSUMED what the warm-up step gathered before the same receive buffers are used again
                import torch.distributed as dist
                dist.barrier(group=par.group)
            for k in self._state_keys:
                st[k].copy_(snap[k])
            if self._pool is None:
                self._pool = torch.cuda.graph_pool_handle()
            l0 = ops.LAUNCHES
            if par is not None and not par.device_gather:
                # sharded step over NCCL: the collectives stay OUTSIDE the graphs (parallel.GraphSegments); the default
                # device-side all-gather (pf_allgather_views) is an ordinary kernel and is captured like everything else
                from .parallel import GraphSegments
                g = GraphSegments(self._pool)
                par.segments = g
                try:
                    g.capture(lambda: self._step_body(st, cameras))
                finally:
                    par.segments = None
            else:
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, pool=self._pool):
                    self._step_body(st, cameras)
            self.launches_per_step = ops.LAUNCHES - l0  # kernels of ours inside one replayed step
            # the graph reads the camera tables by address: it co-owns them (the table cache is LRU-bounded)
            g._pf_tables = self._graph_tables(cameras)
            while len(self._graphs) >= self.max_graphs:
                self._graphs.pop(next(iter(self._graphs)))
            self._graphs[key] = g
            for k in self._state_keys:
                st[k].copy_(snap[k])
            entry = g
        entry.replay()
