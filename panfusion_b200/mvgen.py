"""`MultiViewBaseModel` behind the reference's interface (models/pano/MVGenModel.py:8-297).

Same constructor `(unet, pano_unet, pers_cn=None, pano_cn=None, pano_pad=True)`, same attributes (`unet`,
`pano_unet`, `cp_blocks_encoder`, `cp_blocks_mid`, `cp_blocks_decoder`, `trainable_parameters`), same forward
signature and return value. The UNets are consumed by attribute walk exactly like the reference does, but only to
READ their parameters once (engine.UNetPack); every block then runs as hand-written sm_90a kernels on
channels-last 16-bit activations. There is no PyTorch fallback: without a CUDA device / the built library the
forward raises.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn as nn
from torch import Tensor

from . import _lib
from .engine import Branch, ControlBranch, ControlNetPack, Img, UNetPack
from .eppa import CameraTables, WarpAttn


class MultiViewBaseModel(nn.Module):
    def __init__(self, unet, pano_unet, pers_cn=None, pano_cn=None, pano_pad=True, compute_dtype=torch.bfloat16,
                 overlap_branches=True):
        super().__init__()
        self.unet = unet
        self.pano_unet = pano_unet
        self.pers_cn = pers_cn
        self.pano_cn = pano_cn
        self.pano_pad = pano_pad
        self.compute_dtype = compute_dtype
        self.overlap_branches = overlap_branches  # run the panorama branch on a second CUDA stream
        self._side = None
        if self.unet is not None:  # MVGenModel.py:17-36
            self.cp_blocks_encoder = nn.ModuleList(
                [WarpAttn(blk.downsamplers[-1].out_channels) for blk in unet.down_blocks if blk.downsamplers is not None])
            self.cp_blocks_mid = WarpAttn(unet.mid_block.resnets[-1].out_channels)
            self.cp_blocks_decoder = nn.ModuleList(
                [WarpAttn(blk.upsamplers[0].channels) for blk in unet.up_blocks if blk.upsamplers is not None])
            self.trainable_parameters = [(list(self.cp_blocks_mid.parameters())
                                          + list(self.cp_blocks_decoder.parameters())
                                          + list(self.cp_blocks_encoder.parameters()), 1.0)]
            tables = CameraTables()
            for w in [*self.cp_blocks_encoder, self.cp_blocks_mid, *self.cp_blocks_decoder]:
                w.tables = tables
        self._branches = None
        self._par = None
        # which set of all-gather receive buffers this forward uses (parallel.DeviceAllGather): consecutive steps must
        # use different slots; the sampler sets it (one slot per captured graph, or the step parity when eager)
        self.par_slot = 0

    def set_view_parallel(self, group=None, batch_shards=None, view_shards=None) -> None:
        """Shard the step over the ranks of `group` (parallel.ViewParallel): CFG halves first, then views."""
        from .parallel import ViewParallel
        self._par = ViewParallel(group, batch_shards, view_shards)

    # ---- packing -----------------------------------------------------------------------------------
    def prepare(self, device=None, dtype=None) -> "MultiViewBaseModel":
        """Pack all weights for the kernels (call again after loading new weights)."""
        device = torch.device(device or "cuda")
        if device.type == "cuda" and device.index is None:  # "cuda" != "cuda:0": would re-pack on every forward
            device = torch.device("cuda", torch.cuda.current_device())
        dtype = dtype or self.compute_dtype
        _lib.check(_lib.lib().pf_check_device())
        pers = Branch(UNetPack(self.unet, device, dtype), circular=False) if self.unet is not None else None
        pano = Branch(UNetPack(self.pano_unet, device, dtype), circular=bool(self.pano_pad))
        self._branches = (pers, pano, device, dtype)
        # ControlNets (MVGenModel.py:13-14): optional encoder copies whose outputs are added to the skips / mid output
        self._cn = (ControlBranch(ControlNetPack(self.pers_cn, device, dtype)) if self.pers_cn is not None and pers else None,
                    ControlBranch(ControlNetPack(self.pano_cn, device, dtype)) if self.pano_cn is not None else None)
        if self.unet is not None:
            for w in [*self.cp_blocks_encoder, self.cp_blocks_mid, *self.cp_blocks_decoder]:
                w.invalidate()
        return self

    def invalidate(self):
        self._branches = None

    @torch.no_grad()
    def update_text(self, prompt_embd: Optional[Tensor], pano_prompt_embd: Tensor) -> None:
        """Re-project the text K/V of both branches for new prompt embeddings of the SAME shapes, into the buffers the
        previous call used. A captured CUDA graph of `forward` does not contain the (cached) text projection; the
        sampler calls this when it reuses its graphs for a new prompt (PanFusion.py:134-138 embeds once per image)."""
        if self._branches is None:
            return
        pers, pano, dev, dt = self._branches
        tkey = lambda t, tag: (t.data_ptr(), t._version, tuple(t.shape), tag)
        par = self._par if pers is not None else None
        text_key = tkey(prompt_embd, "pers") if prompt_embd is not None else None
        pano_text_key = tkey(pano_prompt_embd, "pano")
        if par is not None:
            b_full, m_full = prompt_embd.shape[:2]
            par.configure(b_full, m_full)
            bsl, vsl = par.slices(b_full, m_full)
            prompt_embd, pano_prompt_embd = prompt_embd[bsl, vsl], pano_prompt_embd[bsl]
        if pers is not None and prompt_embd is not None:
            pers.set_text(prompt_embd.flatten(0, 1), text_key)
        pano.set_text(pano_prompt_embd.flatten(0, 1), pano_text_key)

    # ---- forward -----------------------------------------------------------------------------------
    @torch.no_grad()
    def forward(self, latents: Optional[Tensor], pano_latent: Tensor, timestep: Tensor, prompt_embd: Optional[Tensor],
                pano_prompt_embd: Tensor, cameras: Optional[dict], pers_layout_cond=None, pano_layout_cond=None):
        if self.pers_cn is None or self.unet is None:  # MVGenModel.py:62-65
            pers_layout_cond = None
        if self.pano_cn is None:
            pano_layout_cond = None
        _lib.require_cuda(pano_latent)
        if self._branches is None or self._branches[2] != pano_latent.device:
            self.prepare(pano_latent.device)
        pers, pano, dev, dt = self._branches
        has_pers = pers is not None

        tkey = lambda t, tag: (t.data_ptr(), t._version, tuple(t.shape), tag)
        text_key = tkey(prompt_embd, "pers") if prompt_embd is not None else None
        pano_text_key = tkey(pano_prompt_embd, "pano")
        par = self._par if has_pers else None
        if par is not None:
            # keep this rank's CFG/batch elements and views; cameras of ALL views stay (EPPA bias needs them)
            b_full, m_full = latents.shape[:2]
            par.configure(b_full, m_full)
            par.begin_step(self.par_slot)
            bsl, vsl = par.slices(b_full, m_full)
            latents, timestep, prompt_embd = latents[bsl, vsl], timestep[bsl, vsl], prompt_embd[bsl, vsl]
            pano_latent, pano_prompt_embd = pano_latent[bsl], pano_prompt_embd[bsl]
            cameras = {k: v[bsl] for k, v in cameras.items()}
            pers_layout_cond = pers_layout_cond[bsl, vsl] if pers_layout_cond is not None else None
            pano_layout_cond = pano_layout_cond[bsl] if pano_layout_cond is not None else None
        if has_pers:
            b, m = latents.shape[:2]
            cam_key = CameraTables.camera_key({k: v.flatten(0, 1) for k, v in cameras.items()})
            pers.set_timesteps(timestep.reshape(-1))          # MVGenModel.py:53-56
            pano.set_timesteps(timestep[:, 0])                # MVGenModel.py:53,59-60
            pers.set_text(prompt_embd.flatten(0, 1), text_key)
        else:
            pano.set_timesteps(timestep)
        pano.set_text(pano_prompt_embd.flatten(0, 1), pano_text_key)

        # The two branches only meet inside EPPA. The panorama branch (batch b, many under-filled launches) runs on a
        # side stream and the perspective branch on the caller's stream; they join before / fork after every fusion.
        main = torch.cuda.current_stream()
        two = bool(self.overlap_branches and has_pers)
        if two and self._side is None:
            # the panorama branch (many small launches that every fusion waits for) runs at higher stream priority: 25.9 -> 25.7 ms
            # single GPU, 9.60 -> 9.55 ms for a rank of the 8-GPU layout
            self._side = torch.cuda.Stream(device=dev, priority=-1)
        side = self._side if two else main
        keep = []  # tensors produced on `main` but consumed on `side`: kept alive until the next join

        def fork():
            if two:
                side.wait_event(main.record_event())

        def join():
            if two:
                main.wait_event(side.record_event())
                keep.clear()

        def fuse(block, h, p):
            join()
            # direction 1 of the fusion continues on the side stream and feeds the panorama branch there; direction 2
            # stays on the main stream: after the block the two streams are already forked again
            return block.forward_tokens(h, p, cam_key, par, side=side if two else None, keep=keep)

        fork()
        # ControlNets (MVGenModel.py:66-83): black-box encoder passes on the UN-padded latents; their outputs are only
        # needed after the encoder, so the panorama one simply runs first on the side stream
        pers_cn, pano_cn = self._cn
        pers_cn_out = pano_cn_out = None
        if pers_layout_cond is not None:
            pers_cn.set_timesteps(timestep.reshape(-1))
            pers_cn.set_text(prompt_embd.flatten(0, 1), text_key + ("cn",))
            pers_cn_out = pers_cn.encode(latents.flatten(0, 1), pers_layout_cond.flatten(0, 1),
                                         tkey(pers_layout_cond, "pers_cond") if par is None else None)
        if pano_layout_cond is not None:
            with torch.cuda.stream(side):
                pano_cn.set_timesteps(timestep[:, 0] if has_pers else timestep)
                pano_cn.set_text(pano_prompt_embd.flatten(0, 1), pano_text_key + ("cn",))
                pano_cn_out = pano_cn.encode(pano_latent.flatten(0, 1), pano_layout_cond.flatten(0, 1),
                                             tkey(pano_layout_cond, "pano_cond") if par is None else None)
        # conv_in (MVGenModel.py:85-91)
        h = pers.conv_in(latents.flatten(0, 1)) if has_pers else None
        with torch.cuda.stream(side):
            p = pano.conv_in(pano_latent.flatten(0, 1))
        skips, pano_skips = ([h] if has_pers else []), [p]

        # encoder (MVGenModel.py:98-152)
        for i, pblk in enumerate(pano.p.down):
            for j, pres in enumerate(pblk["resnets"]):
                if has_pers:
                    blk = pers.p.down[i]
                    h = pers.resnet(h, blk["resnets"][j])
                    if blk["attns"] is not None:
                        h = pers.transformer(h, blk["attns"][j])
                    skips.append(h)
                with torch.cuda.stream(side):
                    p = pano.resnet(p, pres)
                    if pblk["attns"] is not None:
                        p = pano.transformer(p, pblk["attns"][j])
                pano_skips.append(p)
            if pblk["down"] is not None:
                for j, pd in enumerate(pblk["down"]):
                    if has_pers:
                        h = pers.downsample(h, pers.p.down[i]["down"][j])
                    with torch.cuda.stream(side):
                        p = pano.downsample(p, pd)
                if has_pers:
                    skips.append(h)
                pano_skips.append(p)  # skips are taken BEFORE the fusion (MVGenModel.py:146-152)
                if has_pers:
                    h, p = fuse(self.cp_blocks_encoder[i], h, p)

        # ControlNet residuals join the SKIP tensors only after the whole encoder has run (MVGenModel.py:154-170)
        if pers_cn_out is not None:
            skips = pers_cn.add_down(pers_cn_out[0], skips)
        if pano_cn_out is not None:
            with torch.cuda.stream(side):
                pano_skips = pano_cn.add_down(pano_cn_out[0], pano_skips)

        # mid (MVGenModel.py:172-207)
        if has_pers:
            h = pers.resnet(h, pers.p.mid["resnets"][0])
        with torch.cuda.stream(side):
            p = pano.resnet(p, pano.p.mid["resnets"][0])
        for i, pat in enumerate(pano.p.mid["attns"]):
            if has_pers:
                h = pers.transformer(h, pers.p.mid["attns"][i])
                h = pers.resnet(h, pers.p.mid["resnets"][i + 1])
            with torch.cuda.stream(side):
                p = pano.transformer(p, pat)
                p = pano.resnet(p, pano.p.mid["resnets"][i + 1])
        if pers_cn_out is not None:  # MVGenModel.py:200-203
            h = pers_cn.add_mid(pers_cn_out[1], h)
        if pano_cn_out is not None:
            with torch.cuda.stream(side):
                p = pano_cn.add_mid(pano_cn_out[1], p)
        if has_pers:
            h, p = fuse(self.cp_blocks_mid, h, p)

        # decoder (MVGenModel.py:210-277)
        for i, pblk in enumerate(pano.p.up):
            for j, pres in enumerate(pblk["resnets"]):
                if has_pers:
                    blk = pers.p.up[i]
                    h = pers.resnet(h, blk["resnets"][j], skip=skips.pop())
                    if blk["attns"] is not None:
                        h = pers.transformer(h, blk["attns"][j])
                with torch.cuda.stream(side):
                    p = pano.resnet(p, pres, skip=pano_skips.pop())
                    if pblk["attns"] is not None:
                        p = pano.transformer(p, pblk["attns"][j])
            if pblk["up"] is not None:
                if has_pers:
                    h, p = fuse(self.cp_blocks_decoder[i], h, p)  # fusion BEFORE the upsampler (MVGenModel.py:264-267)
                for j, pu in enumerate(pblk["up"]):
                    if has_pers:
                        h = pers.upsample(h, pers.p.up[i]["up"][j])
                    with torch.cuda.stream(side):
                        p = pano.upsample(p, pu)

        # heads (MVGenModel.py:279-297)
        sample = None
        if has_pers:
            s = pers.conv_out(h)
            sample = s.reshape(b, m, *s.shape[1:]).to(latents.dtype)
        with torch.cuda.stream(side):
            ps = pano.conv_out(p)[:, None]
        join()
        if par is not None:
            sample, ps = par.gather_outputs(sample, ps, b_full, m_full)
        return sample, ps.to(pano_latent.dtype)
