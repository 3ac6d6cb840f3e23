"""The CLIP text encoder of the sampling loop + the prompt-embedding cache (SURVEY.md 8f rank 3).

Reference: `PanoGenerator.encode_text` (models/pano/PanoGenerator.py:197-211: tokenizer -> `CLIPTextModel(input_ids)[0]`, the
final-layer-normed hidden states, loaded at :117-121 from the SD-2 `text_encoder` sub-folder), `PanFusion.embed_prompt`
(models/pano/PanFusion.py:45-62) and the CFG concatenation [null; text] of `inference` (:134-138). The encoder is
transformers `CLIPTextModel` [3P] (OpenCLIP ViT-H text tower for SD-2: 1024 wide, 16 heads of 64, 23 pre-LN layers, erf-GELU
MLP, causal mask, learned positions). Like the UNets it is consumed by attribute walk to read its parameters once; the
forward runs on the denoiser's kernels:

  pf_embed_tokens                      token + position embedding, row statistics for the first LayerNorm
  per layer  pf_gemm_taps (LN1 folded) fused q|k|v projection          -> pf_fmha_fwd (head dim 64, causal additive bias)
             pf_gemm_taps              out_proj + residual, row statistics
             pf_gemm_taps (LN2 folded) fc1 + erf-GELU                   -> pf_gemm_taps fc2 + residual, row statistics
  pf_layernorm                         final_layer_norm

The tokenizer is host-side string processing and needs the vocabulary files of the checkpoint: this module starts at
`input_ids`. There is no PyTorch compute fallback.
"""
from __future__ import annotations

from collections import OrderedDict
from typing import Optional

import torch
from torch import Tensor

from . import _lib, ops
from .engine import _Lin, _LinLN, _Norm


class _Layer:
    def __init__(self, layer, dev, dt):
        a = layer.self_attn
        w = torch.cat([a.q_proj.weight, a.k_proj.weight, a.v_proj.weight], 0)
        b = torch.cat([a.q_proj.bias, a.k_proj.bias, a.v_proj.bias], 0)
        self.qkv = _LinLN(w, b, layer.layer_norm1, dev, dt)
        self.out = _Lin(a.out_proj.weight, a.out_proj.bias, dev, dt)
        self.fc1 = _LinLN(layer.mlp.fc1.weight, layer.mlp.fc1.bias, layer.layer_norm2, dev, dt)
        self.fc2 = _Lin(layer.mlp.fc2.weight, layer.mlp.fc2.bias, dev, dt)


# transformers' ACT2FN names of the CLIP MLP -> the tap-GEMM epilogue that applies them
ACTIVATIONS = {"gelu": ops.PF_ACT_GELU, "quick_gelu": ops.PF_ACT_QUICK_GELU}


def encoder_layers(x: Tensor, st: Tensor, layers, B: int, L: int, heads: int, act: int,
                   bias: Optional[Tensor] = None) -> Tensor:
    """The pre-LN CLIP encoder layers (CLIPEncoderLayer [3P]) of both towers over x [B*L, C] (16-bit residual stream) with
    st = its row statistics [B*L, 2, 2]; bias = the attention's additive fp32 bias [L, >=L] (the text tower's causal
    mask) or None (the vision tower). Returns the residual stream after the last layer."""
    T, C = x.shape
    dt, dev = x.dtype, x.device
    new = lambda n: torch.empty((T, n), dtype=dt, device=dev)
    for l in layers:
        qkv = ops.gemm_taps(x, l.qkv.w, new(3 * C), M=T, Kc=C, bias=l.qkv.b,
                            ln=(st, l.qkv.colsum, l.qkv.eps)).reshape(B, L, 3 * C)
        o = torch.empty((B, L, C), dtype=dt, device=dev)
        ops.fmha(qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:], o, heads=heads, head_dim=64, scale=64 ** -0.5,
                 bias=bias)
        x, st = ops.gemm_taps(o.reshape(T, C), l.out.w, new(C), M=T, Kc=C, bias=l.out.b, residual=x, row_stats=True)
        h = ops.gemm_taps(x, l.fc1.w, new(l.fc1.n), M=T, Kc=C, bias=l.fc1.b, act=act,
                          ln=(st, l.fc1.colsum, l.fc1.eps))
        x, st = ops.gemm_taps(h, l.fc2.w, new(C), M=T, Kc=l.fc2.k, bias=l.fc2.b, residual=x, row_stats=True)
    return x


class CLIPTextEncoder:
    """`text_encoder(input_ids)[0]` of a duck-typed transformers `CLIPTextModel` (anything exposing
    `.text_model.{embeddings.{token_embedding,position_embedding}, encoder.layers[i].{layer_norm1, self_attn.{q,k,v,out}_proj,
    layer_norm2, mlp.{fc1,fc2}}, final_layer_norm}` and `.config`)."""

    def __init__(self, text_encoder, compute_dtype=torch.bfloat16):
        self.src = text_encoder
        self.compute_dtype = compute_dtype
        self._packed = None

    def prepare(self, device=None, dtype=None) -> "CLIPTextEncoder":
        dev = torch.device(device or "cuda")
        if dev.type == "cuda" and dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        dt = dtype or self.compute_dtype
        _lib.check(_lib.lib().pf_check_device())
        tm = self.src.text_model
        cfg = self.src.config
        act = getattr(cfg, "hidden_act", "gelu")
        if act not in ACTIVATIONS:
            raise NotImplementedError(f"CLIP text encoder with hidden_act={act!r}: 'gelu' (SD-2's tower, PF_ACT_GELU) "
                                      "and 'quick_gelu' (OpenAI CLIP, PF_ACT_QUICK_GELU) are served")
        heads = int(cfg.num_attention_heads)
        C = int(cfg.hidden_size)
        if C // heads != 64:
            raise NotImplementedError(f"CLIP text encoder with head dim {C // heads}: pf_fmha_fwd serves 32 and 64")
        f32 = lambda t: t.detach().to(dev, torch.float32).contiguous()
        L = tm.embeddings.position_embedding.weight.shape[0]
        # causal mask as the additive fp32 bias of the attention kernel, shared by batch and heads ([Lq, Lk], rows padded
        # to the 4-float alignment the kernel's vector loads need)
        ld = (L + 3) // 4 * 4
        bias = torch.zeros((L, ld), dtype=torch.float32)
        bias[:, :L] = torch.full((L, L), torch.finfo(torch.float32).min).triu(1)
        self._packed = dict(
            dev=dev, dt=dt, C=C, heads=heads, L=L, act=ACTIVATIONS[act], vocab=tm.embeddings.token_embedding.weight.shape[0],
            tok=f32(tm.embeddings.token_embedding.weight), pos=f32(tm.embeddings.position_embedding.weight),
            layers=[_Layer(l, dev, dt) for l in tm.encoder.layers], final=_Norm(tm.final_layer_norm, dev),
            causal=bias.to(dev))
        return self

    @torch.no_grad()
    def __call__(self, input_ids: Tensor) -> Tensor:
        """input_ids int64 [B, L] -> last_hidden_state [B, L, C] in the compute dtype (PanoGenerator.py:207-211)."""
        if self._packed is None or (input_ids.is_cuda and self._packed["dev"] != input_ids.device):
            self.prepare(input_ids.device if input_ids.is_cuda else None)
        w = self._packed
        dev, dt, C, H, L = w["dev"], w["dt"], w["C"], w["heads"], w["L"]
        ids = input_ids.to(dev, torch.int64).contiguous()
        B, Lx = ids.shape
        if Lx > L:
            raise ValueError(f"sequence length {Lx} exceeds max_position_embeddings {L}")
        T = B * Lx
        x = torch.empty((T, C), dtype=dt, device=dev)
        st = torch.empty((T, 2, 2), dtype=torch.float32, device=dev)
        Cv = _lib.C.c_void_p
        ops._count(1)
        _lib.check(_lib.lib().pf_embed_tokens(Cv(ids.data_ptr()), Cv(w["tok"].data_ptr()), Cv(w["pos"].data_ptr()),
                                              Cv(x.data_ptr()), _lib.dtype_code(dt), Cv(st.data_ptr()), T, Lx, C, w["vocab"],
                                              Cv(_lib.stream_ptr())))
        x = encoder_layers(x, st, w["layers"], B, Lx, H, w["act"], bias=w["causal"][:Lx])
        out = ops.layernorm(x, w["final"].g, w["final"].b, w["final"].eps)
        return out.reshape(B, Lx, C)


class PromptEmbedder:
    """`encode_text` + `embed_prompt` + the CFG concatenation of `inference` (PanoGenerator.py:197-211, PanFusion.py:45-62,
    134-138) on token ids, with an LRU cache of per-prompt embeddings: the null prompt is needed for every image, the
    panorama prompt is repeated for every view (`copy_pano_prompt`), and `predict` re-embeds the same prompts for every
    batch — each distinct token row is encoded once."""

    def __init__(self, encoder: CLIPTextEncoder, max_entries: int = 256):
        self.encoder = encoder
        self.max_entries = max_entries
        self._cache: "OrderedDict[tuple, Tensor]" = OrderedDict()
        self.hits = self.misses = 0

    def invalidate(self) -> None:
        self._cache.clear()

    @torch.no_grad()
    def encode_text(self, input_ids: Tensor) -> Tensor:
        """input_ids [B, L] (CPU or CUDA) -> [B, L, C]; rows already seen come from the cache."""
        rows = [tuple(r) for r in input_ids.to("cpu", torch.int64).tolist()]
        todo = list(OrderedDict.fromkeys(r for r in rows if r not in self._cache))
        self.misses += len(todo)
        self.hits += len(rows) - len(todo)
        if todo:
            emb = self.encoder(torch.tensor(todo, dtype=torch.int64))
            for r, e in zip(todo, emb):
                self._cache[r] = e
        out = torch.stack([self._cache[r] for r in rows])
        for r in rows:
            self._cache.move_to_end(r)
        while len(self._cache) > self.max_entries:
            self._cache.popitem(last=False)
        return out

    @torch.no_grad()
    def embed_prompt(self, pano_ids: Tensor, null_ids: Tensor, num_cameras: int, pers_ids: Optional[Tensor] = None):
        """-> (pers_prompt_embd [2b, m, L, C], pano_prompt_embd [2b, 1, L, C]) = [null; text] along the batch, the layout
        `forward_cls_free` expects. pano_ids [b, L]; null_ids [1, L] (the tokenised empty string); pers_ids [b*m, L] for
        `use_pers_prompt`, else every view carries the panorama prompt (`copy_pano_prompt`, PanFusion.py:17)."""
        b = pano_ids.shape[0]
        pano = self.encode_text(pano_ids)[:, None]                                  # [b, 1, L, C]
        if pers_ids is not None:
            pers = self.encode_text(pers_ids).reshape(b, num_cameras, *pano.shape[2:])
        else:
            pers = pano.repeat(1, num_cameras, 1, 1)
        null = self.encode_text(null_ids)[:, None].repeat(b, 1, 1, 1)               # PanFusion.py:135
        pano_prompt_embd = torch.cat([null, pano])
        pers_prompt_embd = torch.cat([null.repeat(1, num_cameras, 1, 1), pers])
        return pers_prompt_embd, pano_prompt_embd
