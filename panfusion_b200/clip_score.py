"""CLIP score (torchmetrics' CLIPScore('openai/clip-vit-base-patch16'), as models/pano/EvalPanoGen.py:33-46 builds it)
on the sm_90a kernels.

`CLIPEncoder` packs a CLIP model once (fp16 weights, LayerNorms folded into the following GEMMs) and runs both towers:

  image  pf_clip_prep        CLIPImageProcessor: Pillow-exact bicubic resize, centre crop, normalise -> patch rows
         pf_gemm_taps        patch embedding (one GEMM over the patch rows)
         pf_clip_embed       class token + positions + pre_layrnorm, row statistics for layer 0's folded LN1
         12 x encoder layer  text_encoder.encoder_layers (pf_gemm_taps with PF_ACT_QUICK_GELU, pf_fmha_fwd, no mask)
         pf_layernorm        post_layernorm of the CLS rows (a strided view) -> pf_gemm_taps visual_projection
  text   text_encoder.CLIPTextEncoder (causal, quick_gelu) -> the row at input_ids.argmax(-1) (host index)
         -> pf_gemm_taps text_projection
  score  pf_clip_score       100 * cosine per sample, the batch sum added to the fp64 state in sample order

`CLIPScore` keeps torchmetrics' states and behaviour. Tokenisation is host string processing. Nothing is downloaded, and
there is no PyTorch compute fallback.
"""
from __future__ import annotations

import ctypes as C
import json
import warnings
from pathlib import Path
from types import SimpleNamespace
from typing import Callable, Optional

import torch
from torch import nn

from . import _lib, ops
from .engine import _Lin, _Norm
from .text_encoder import ACTIVATIONS, CLIPTextEncoder, _Layer, encoder_layers

PATCH = 16
GRID = 14
TOKENS = GRID * GRID + 1  # 196 patches and the class token


def _get(cfg, key, default=None):
    if cfg is None:
        return default
    if isinstance(cfg, dict):
        return cfg.get(key, default)
    return getattr(cfg, key, default)


def _config(config) -> dict:
    """CLIPConfig object or config.json dict -> the geometry the towers need, checked."""
    out = {}
    for tower, width in (("text_config", 512), ("vision_config", 768)):
        c = _get(config, tower)
        if c is None:
            raise ValueError(f"CLIP config: missing {tower!r}")
        d = dict(hidden=int(_get(c, "hidden_size", width)), heads=int(_get(c, "num_attention_heads", 8)),
                 layers=int(_get(c, "num_hidden_layers", 12)), inter=int(_get(c, "intermediate_size", 4 * width)),
                 act=str(_get(c, "hidden_act", "quick_gelu")), eps=float(_get(c, "layer_norm_eps", 1e-5)))
        if d["hidden"] % d["heads"] or d["hidden"] // d["heads"] != 64:
            raise ValueError(f"CLIP {tower}: head dim {d['hidden'] / d['heads']:g} (hidden_size {d['hidden']}, "
                             f"{d['heads']} heads); only head dim 64 is served")
        if d["act"] not in ACTIVATIONS:
            raise ValueError(f"CLIP {tower}: hidden_act {d['act']!r} not served ({sorted(ACTIVATIONS)})")
        if tower == "text_config":
            d["vocab"] = int(_get(c, "vocab_size", 49408))
            d["max_pos"] = int(_get(c, "max_position_embeddings", 77))
        else:
            if int(_get(c, "patch_size", PATCH)) != PATCH or int(_get(c, "image_size", 224)) != GRID * PATCH or \
                    int(_get(c, "num_channels", 3)) != 3:
                raise ValueError("CLIP vision_config: only 224x224 RGB images in 16x16 patches are served")
        out[tower[:-7]] = d
    out["proj"] = int(_get(config, "projection_dim", 512))
    return out


def expected_shapes(cfg: dict) -> dict[str, tuple]:
    """Every key CLIPModel's two towers read, with its shape."""
    t, v, p = cfg["text"], cfg["vision"], cfg["proj"]
    want = {"text_model.embeddings.token_embedding.weight": (t["vocab"], t["hidden"]),
            "text_model.embeddings.position_embedding.weight": (t["max_pos"], t["hidden"]),
            "text_model.final_layer_norm.weight": (t["hidden"],), "text_model.final_layer_norm.bias": (t["hidden"],),
            "vision_model.embeddings.class_embedding": (v["hidden"],),
            "vision_model.embeddings.patch_embedding.weight": (v["hidden"], 3, PATCH, PATCH),
            "vision_model.embeddings.position_embedding.weight": (TOKENS, v["hidden"]),
            "vision_model.pre_layrnorm.weight": (v["hidden"],), "vision_model.pre_layrnorm.bias": (v["hidden"],),
            "vision_model.post_layernorm.weight": (v["hidden"],), "vision_model.post_layernorm.bias": (v["hidden"],),
            "visual_projection.weight": (p, v["hidden"]), "text_projection.weight": (p, t["hidden"])}
    for tower, d in (("text_model", t), ("vision_model", v)):
        C, I = d["hidden"], d["inter"]
        for i in range(d["layers"]):
            pre = f"{tower}.encoder.layers.{i}"
            for n in ("q_proj", "k_proj", "v_proj", "out_proj"):
                want[f"{pre}.self_attn.{n}.weight"] = (C, C)
                want[f"{pre}.self_attn.{n}.bias"] = (C,)
            for n in ("layer_norm1", "layer_norm2"):
                want[f"{pre}.{n}.weight"] = (C,)
                want[f"{pre}.{n}.bias"] = (C,)
            want[f"{pre}.mlp.fc1.weight"], want[f"{pre}.mlp.fc1.bias"] = (I, C), (I,)
            want[f"{pre}.mlp.fc2.weight"], want[f"{pre}.mlp.fc2.bias"] = (C, I), (C,)
    return want


def load_state(source, config=None) -> tuple[dict, dict, Optional[Path]]:
    """-> (checked fp32 state dict, geometry, local directory or None) from a local directory (config.json and
    model.safetensors or pytorch_model.bin), a state dict with CLIPModel key names plus `config`, or a CLIPModel-like
    object (state_dict() and .config). Raises ValueError naming a missing or mis-shaped key; nothing is downloaded."""
    path = None
    if isinstance(source, (str, Path)):
        path = Path(source)
        if not path.is_dir():
            raise ValueError(f"CLIP model {str(source)!r} is not a local directory; nothing is downloaded — pass the "
                             "directory of a snapshot holding config.json and model.safetensors or pytorch_model.bin")
        if not (path / "config.json").is_file():
            raise ValueError(f"CLIP model directory {path}: missing config.json")
        config = json.loads((path / "config.json").read_text())
        if (path / "model.safetensors").is_file():
            from safetensors.torch import load_file
            state = load_file(str(path / "model.safetensors"))
        elif (path / "pytorch_model.bin").is_file():
            state = torch.load(path / "pytorch_model.bin", map_location="cpu", weights_only=True)
        else:
            raise ValueError(f"CLIP model directory {path}: missing model.safetensors or pytorch_model.bin")
    elif hasattr(source, "state_dict") and hasattr(source, "config"):
        state, config = source.state_dict(), source.config
    else:
        state = source
        if config is None:
            raise ValueError("a CLIP state dict needs its config (a CLIPConfig or the config.json dict)")
    cfg = _config(config)
    sd = {k: v.detach() for k, v in dict(state).items()}
    for k, shape in expected_shapes(cfg).items():
        if k not in sd:
            raise ValueError(f"CLIP state dict: missing key {k!r}")
        if tuple(sd[k].shape) != shape:
            raise ValueError(f"CLIP state dict: {k!r} has shape {tuple(sd[k].shape)}, expected {shape}")
    return {k: sd[k].float().cpu() for k in expected_shapes(cfg)}, cfg, path


def _ns_norm(sd, p, eps):
    return SimpleNamespace(weight=sd[f"{p}.weight"], bias=sd[f"{p}.bias"], eps=eps)


def _ns_lin(sd, p):
    return SimpleNamespace(weight=sd[f"{p}.weight"], bias=sd.get(f"{p}.bias"))


def _ns_layers(sd, tower, d):
    out = []
    for i in range(d["layers"]):
        p = f"{tower}.encoder.layers.{i}"
        out.append(SimpleNamespace(
            layer_norm1=_ns_norm(sd, f"{p}.layer_norm1", d["eps"]), layer_norm2=_ns_norm(sd, f"{p}.layer_norm2", d["eps"]),
            self_attn=SimpleNamespace(**{n: _ns_lin(sd, f"{p}.self_attn.{n}") for n in ("q_proj", "k_proj", "v_proj",
                                                                                          "out_proj")}),
            mlp=SimpleNamespace(fc1=_ns_lin(sd, f"{p}.mlp.fc1"), fc2=_ns_lin(sd, f"{p}.mlp.fc2"))))
    return out


def eos_rows(input_ids: torch.Tensor) -> torch.Tensor:
    """The pooled row of each prompt: input_ids.argmax(-1) (transformers 4.26.1; EOS is the largest id, so this is the
    first EOS, and the largest id of a prompt truncated before its EOS)."""
    return input_ids.to("cpu", torch.int64).argmax(-1)


class CLIPEncoder(nn.Module):
    """CLIPModel's get_image_features / get_text_features on the GPU. `source`: a local snapshot directory, a state dict
    with CLIPModel key names (with `config`), or a CLIPModel-like object. The checked fp32 weights stay on the host; each
    device gets its packed fp16 copy once, on first use."""

    def __init__(self, source, config=None, compute_dtype: torch.dtype = torch.float16):
        super().__init__()
        self._sd, self.cfg, self.path = load_state(source, config)
        self.compute_dtype = compute_dtype
        t = self.cfg["text"]
        text = SimpleNamespace(
            text_model=SimpleNamespace(
                embeddings=SimpleNamespace(
                    token_embedding=SimpleNamespace(weight=self._sd["text_model.embeddings.token_embedding.weight"]),
                    position_embedding=SimpleNamespace(
                        weight=self._sd["text_model.embeddings.position_embedding.weight"])),
                encoder=SimpleNamespace(layers=_ns_layers(self._sd, "text_model", t)),
                final_layer_norm=_ns_norm(self._sd, "text_model.final_layer_norm", t["eps"])),
            config=SimpleNamespace(hidden_act=t["act"], num_attention_heads=t["heads"], hidden_size=t["hidden"]))
        self._text = CLIPTextEncoder(text, compute_dtype=compute_dtype)
        self._packed: dict = {}
        self._taps: dict = {}

    @property
    def max_position_embeddings(self) -> int:
        return self.cfg["text"]["max_pos"]

    def _pack(self, dev: torch.device) -> dict:
        if dev in self._packed:
            return self._packed[dev]
        sd, v, dt = self._sd, self.cfg["vision"], self.compute_dtype
        f32 = lambda t: t.to(dev, torch.float32).contiguous()
        pre = _ns_norm(sd, "vision_model.pre_layrnorm", v["eps"])
        self._packed[dev] = dict(
            patch=_Lin(sd["vision_model.embeddings.patch_embedding.weight"], None, dev, dt),
            cls=f32(sd["vision_model.embeddings.class_embedding"]),
            pos=f32(sd["vision_model.embeddings.position_embedding.weight"]),
            pre=_Norm(pre, dev), post=_Norm(_ns_norm(sd, "vision_model.post_layernorm", v["eps"]), dev),
            layers=[_Layer(l, dev, dt) for l in _ns_layers(sd, "vision_model", v)],
            vproj=_Lin(sd["visual_projection.weight"], None, dev, dt),
            tproj=_Lin(sd["text_projection.weight"], None, dev, dt))
        return self._packed[dev]

    def taps(self, H: int, W: int, dev: torch.device) -> torch.Tensor:
        """pf_clip_prep_taps(H, W) on `dev`, computed once per size."""
        key = (H, W, dev)
        if key not in self._taps:
            l = _lib.lib()
            n = int(l.pf_clip_prep_taps_ints(H, W))
            host = torch.empty(n, dtype=torch.int32)
            _lib.check(l.pf_clip_prep_taps(H, W, C.c_void_p(host.data_ptr())))
            self._taps[key] = host.to(dev)
        return self._taps[key]

    @torch.no_grad()
    def prep(self, imgs: torch.Tensor, out_dtype: torch.dtype = torch.float16) -> torch.Tensor:
        """uint8 or fp32 [B, 3, H, W] CUDA images -> the normalised 224^2 crops as patch rows [B * 196, 768]."""
        _lib.require_cuda(imgs)
        if imgs.dim() != 4 or imgs.shape[1] != 3:
            raise ValueError(f"expected images [B, 3, H, W], got {tuple(imgs.shape)}")
        if imgs.dtype not in (torch.uint8, torch.float32):
            raise ValueError(f"expected uint8 or float32 images, got {imgs.dtype}")
        B, _, H, W = imgs.shape
        imgs = imgs.contiguous()
        taps = self.taps(H, W, imgs.device)
        out = torch.empty(B * GRID * GRID, 3 * PATCH * PATCH, device=imgs.device, dtype=out_dtype)
        ops._count(1)
        _lib.check(_lib.lib().pf_clip_prep(C.c_void_p(imgs.data_ptr()), int(imgs.dtype == torch.uint8), B, H, W,
                                           C.c_void_p(taps.data_ptr()), C.c_void_p(out.data_ptr()),
                                           _lib.dtype_code(out_dtype), C.c_void_p(_lib.stream_ptr())))
        return out

    @torch.no_grad()
    def encode_image(self, imgs: torch.Tensor) -> torch.Tensor:
        """get_image_features: uint8 or fp32 [0, 1] [B, 3, H, W] CUDA images -> fp32 [B, projection_dim]."""
        dev = imgs.device
        with torch.cuda.device(dev):
            w, v, dt = self._pack(dev), self.cfg["vision"], self.compute_dtype
            C_ = v["hidden"]
            patches = self.prep(imgs, dt)
            B = imgs.shape[0]
            pe = ops.gemm_taps(patches, w["patch"].w, torch.empty(B * GRID * GRID, C_, device=dev, dtype=torch.float32),
                               M=B * GRID * GRID, Kc=w["patch"].k)
            x = torch.empty(B * TOKENS, C_, device=dev, dtype=dt)
            st = torch.empty(B * TOKENS, 2, 2, device=dev, dtype=torch.float32)
            Cv = C.c_void_p
            ops._count(1)
            _lib.check(_lib.lib().pf_clip_embed(
                Cv(pe.data_ptr()), Cv(w["cls"].data_ptr()), Cv(w["pos"].data_ptr()), Cv(w["pre"].g.data_ptr()),
                Cv(w["pre"].b.data_ptr()), C.c_float(w["pre"].eps), B, C_, Cv(x.data_ptr()), _lib.dtype_code(dt),
                Cv(st.data_ptr()), Cv(_lib.stream_ptr())))
            x = encoder_layers(x, st, w["layers"], B, TOKENS, v["heads"], ACTIVATIONS[v["act"]])
            cls = x.view(B, TOKENS * C_)[:, :C_]  # the CLS rows, a strided view
            h = ops.layernorm(cls, w["post"].g, w["post"].b, w["post"].eps)
            return ops.gemm_taps(h, w["vproj"].w, torch.empty(B, w["vproj"].n, device=dev, dtype=torch.float32),
                                 M=B, Kc=C_)

    @torch.no_grad()
    def encode_text(self, input_ids: torch.Tensor, device: torch.device) -> torch.Tensor:
        """get_text_features: int64 [B, L] token ids (L <= max_position_embeddings) -> fp32 [B, projection_dim]. The
        attention mask is not needed: padding follows the EOS row and the mask is causal."""
        with torch.cuda.device(device):
            w = self._pack(device)
            hid = self._text(input_ids.to(device))  # packs on first use; final_layer_norm on all rows
            B = hid.shape[0]
            rows = (torch.arange(B) * hid.shape[1] + eos_rows(input_ids)).to(device)
            h = hid.reshape(-1, hid.shape[-1]).index_select(0, rows)
            return ops.gemm_taps(h, w["tproj"].w, torch.empty(B, w["tproj"].n, device=device, dtype=torch.float32),
                                 M=B, Kc=w["tproj"].k)


def _token_ids(tokenizer: Callable, text: list[str]) -> torch.Tensor:
    out = tokenizer(text, padding=True, return_tensors="pt")
    if not torch.is_tensor(out):
        out = out.input_ids if hasattr(out, "input_ids") else out["input_ids"]
    return torch.as_tensor(out, dtype=torch.int64)


class CLIPScore(nn.Module):
    """torchmetrics' CLIPScore on the GPU: update(images, text), compute() -> 0-d fp32 CUDA tensor
    max(score / n_samples, 0), reset(). `clip=` shares one packed CLIPEncoder between metrics; `tokenizer` is any
    callable(list[str], padding=True, return_tensors="pt") returning input_ids (default: transformers' CLIPTokenizer
    from the local model directory, local_files_only=True). States `score` (fp64) and `n_samples` (int64) are
    non-persistent buffers: .to(device) moves them and a sum all-reduce merges ranks."""

    higher_is_better = True
    is_differentiable = False
    full_state_update = True

    def __init__(self, model_name_or_path="openai/clip-vit-base-patch16", *, clip: Optional[CLIPEncoder] = None,
                 tokenizer: Optional[Callable] = None, device: torch.device | str | None = None):
        super().__init__()
        if clip is None:
            clip = CLIPEncoder(model_name_or_path)
        elif not isinstance(clip, CLIPEncoder):
            raise ValueError(f"clip must be a CLIPEncoder, got {type(clip).__name__}")
        self.clip = clip
        if tokenizer is None:
            if clip.path is None:
                raise ValueError("tokenizer=None loads CLIPTokenizer from the model's local directory; this CLIPEncoder "
                                 "was built from a state dict, so pass tokenizer=")
            from transformers import CLIPTokenizer
            tokenizer = CLIPTokenizer.from_pretrained(str(clip.path), local_files_only=True)
        self.tokenizer = tokenizer
        self.register_buffer("score", torch.zeros((), dtype=torch.float64), persistent=False)
        self.register_buffer("n_samples", torch.zeros((), dtype=torch.int64), persistent=False)
        self._update_called = False
        if device is not None:
            self.to(device)

    def reset(self) -> None:
        self.score.zero_()
        self.n_samples.zero_()
        self._update_called = False

    def token_ids(self, text: list[str]) -> torch.Tensor:
        """Tokenise with padding, then truncate to max_position_embeddings with a warning, as torchmetrics does."""
        ids = _token_ids(self.tokenizer, text)
        L = self.clip.max_position_embeddings
        if ids.shape[-1] > L:
            warnings.warn(f"Encountered caption longer than max_position_embeddings={L}. Will truncate captions to this "
                          "length. If longer captions are needed, initialize argument `model_name_or_path` with a model "
                          "that supports longer sequences", UserWarning)
            ids = ids[..., :L]
        return ids

    @torch.no_grad()
    def update(self, images, text) -> None:
        if not isinstance(images, list):
            batch = images if images.ndim == 4 else None
            images = [images] if images.ndim == 3 else list(images)
        else:
            batch = None
        if not all(i.ndim == 3 for i in images):
            raise ValueError("Expected all images to be 3d but found image that has either more or less")
        if not isinstance(text, list):
            text = [text]
        if len(text) != len(images):
            raise ValueError(f"Expected the number of images and text examples to be the same but got {len(images)} "
                             f"and {len(text)}")
        dev = self.score.device
        for i in images:
            if i.device != dev:
                raise ValueError(f"images are on {i.device} but the metric's states on {dev}; move the metric with "
                                 ".to(device)")
            _lib.require_cuda(i)
        ids = self.token_ids(text)
        with torch.cuda.device(dev):
            if batch is not None:
                img = self.clip.encode_image(batch)
            else:
                # consecutive images of one shape and dtype go through the towers together
                parts, k = [], 0
                while k < len(images):
                    j = k + 1
                    while j < len(images) and images[j].shape == images[k].shape and images[j].dtype == images[k].dtype:
                        j += 1
                    parts.append(self.clip.encode_image(torch.stack(images[k:j])))
                    k = j
                img = torch.cat(parts)
            txt = self.clip.encode_text(ids, dev)
            scores = torch.empty(len(images), device=dev, dtype=torch.float32)
            ops._count(1)
            _lib.check(_lib.lib().pf_clip_score(C.c_void_p(img.data_ptr()), C.c_void_p(txt.data_ptr()), len(images),
                                                img.shape[1], C.c_void_p(scores.data_ptr()),
                                                C.c_void_p(self.score.data_ptr()), C.c_void_p(_lib.stream_ptr())))
        self.n_samples.add_(len(images))
        self.last_scores = scores
        self._update_called = True

    def compute(self) -> torch.Tensor:
        return torch.clamp(self.score / self.n_samples, min=0).float()
