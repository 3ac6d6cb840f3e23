"""HorizonNet's layout network (the `net` of models/horizonnet/HorizonNet.py, external/HorizonNet/model.py
HorizonNet('resnet50', use_rnn=True)) on the sm_90a kernels.

    pf_hnet_prep             _prepare_x: (x[:, :3] - mean) / std in fp32, rounded once to fp16 [B, 512, 1024, 16]
    pf_hnet_conv             the ResNet-50 encoder (stem, 16 bottlenecks, residual added before the ReLU) and the 16
                             ConvCompressH layers: BN folded in fp64, rows zero-padded, columns wrapped (wrap_lr_pad)
    pf_pool2d_nhwc           the stem's MaxPool2d(3, 2, 1) (-inf padding, no wrap)
    pf_hnet_height_upsample  GlobalHeightConv's tail, written straight into the (t, b) rows of the LSTM input
    pf_gemm_taps             each LSTM layer's input projections of both directions (fp32 out, b_ih + b_hh)
    pf_lstm_bidir            each LSTM layer's recurrence, both directions in one launch
    pf_hnet_head             Linear(1024, 12) and the reference's permutation into bon / cor

The host post-processing (horizon_to_manhattan_layout, LayoutIoU) stays the reference's and reads this module's
outputs. Batches above MAX_BATCH are run in chunks.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import torch
from torch import nn

from . import _lib, ops
from .inception import MAX

BN_EPS = 1e-5
H, W, T = 512, 1024, 256
PREP_C = 16
MAX_BATCH = 16  # pf_lstm_bidir's limit per launch
ENC = "feature_extractor.encoder."
LAYERS = [(3, 64, 1), (4, 128, 2), (6, 256, 2), (3, 512, 2)]  # torchvision resnet50: blocks, width, first stride
SCALE_C = (256, 512, 1024, 2048)


def _convs() -> list[tuple]:
    """(name, weight key, BN prefix, conv bias key, Cin, Cout, k, (stride_h, stride_w)) of every convolution."""
    out = [("stem", f"{ENC}conv1.1.weight", f"{ENC}bn1", None, 3, 64, 7, (2, 2))]
    cin = 64
    for li, (n, width, s) in enumerate(LAYERS, 1):
        for j in range(n):
            p = f"{ENC}layer{li}.{j}."
            st = (s, s) if j == 0 else (1, 1)
            out.append((f"l{li}_{j}_c1", p + "conv1.weight", p + "bn1", None, cin, width, 1, (1, 1)))
            out.append((f"l{li}_{j}_c2", p + "conv2.1.weight", p + "bn2", None, width, width, 3, st))
            out.append((f"l{li}_{j}_c3", p + "conv3.weight", p + "bn3", None, width, 4 * width, 1, (1, 1)))
            if j == 0:
                out.append((f"l{li}_{j}_ds", p + "downsample.0.weight", p + "downsample.1", None, cin, 4 * width, 1,
                            st))
            cin = 4 * width
    for s, c in enumerate(SCALE_C):
        chans = [c, c // 2, c // 2, c // 4, c // 8]
        for l in range(4):
            p = f"reduce_height_module.ghc_lst.{s}.layer.{l}.layers."
            out.append((f"h{s}_{l}", p + "0.1.weight", p + "1", p + "0.1.bias", chans[l], chans[l + 1], 3, (2, 1)))
    return out


CONVS = {c[0]: c[1:] for c in _convs()}


def _lstm_key(name: str, layer: int, reverse: bool) -> str:
    return f"bi_rnn.{name}_l{layer}" + ("_reverse" if reverse else "")


def state_shapes() -> dict[str, tuple]:
    """Every key the network reads and its shape (num_batches_tracked is not read)."""
    want = {}
    for _n, (wk, bp, bk, ci, co, k, _s) in CONVS.items():
        want[wk] = (co, ci, k, k)
        if bk:
            want[bk] = (co,)
        for p in ("weight", "bias", "running_mean", "running_var"):
            want[f"{bp}.{p}"] = (co,)
    for layer in (0, 1):
        for rev in (False, True):
            want[_lstm_key("weight_ih", layer, rev)] = (2048, 1024)
            want[_lstm_key("weight_hh", layer, rev)] = (2048, 512)
            want[_lstm_key("bias_ih", layer, rev)] = (2048,)
            want[_lstm_key("bias_hh", layer, rev)] = (2048,)
    want["linear.weight"] = (12, 1024)
    want["linear.bias"] = (12,)
    return want


def load_state(state) -> dict[str, torch.Tensor]:
    """A reference HorizonNetModule state dict (wrap_lr_pad's key names), the Lightning checkpoint LayoutConsistency
    loads (a path or its loaded dict: ['state_dict'] with a `net.` prefix), or a live reference nn.Module, checked:
    every key the network reads must be present with its shape, else ValueError naming it."""
    if isinstance(state, nn.Module):
        state = state.state_dict()
    elif isinstance(state, (str, bytes, Path)):
        state = torch.load(state, map_location="cpu", weights_only=True)
    state = dict(state)
    if isinstance(state.get("state_dict"), dict):
        state = state["state_dict"]
    if any(k.startswith("net.") for k in state):
        state = {k[4:]: v for k, v in state.items() if k.startswith("net.")}
    sd = {k: v.detach().cpu() for k, v in state.items() if torch.is_tensor(v)}
    for k, shape in state_shapes().items():
        if k not in sd:
            raise ValueError(f"HorizonNet state dict: missing key {k!r}")
        if tuple(sd[k].shape) != shape:
            raise ValueError(f"HorizonNet state dict: {k!r} has shape {tuple(sd[k].shape)}, expected {shape}")
    return sd


def fold_bn(sd: dict, name: str) -> tuple[torch.Tensor, torch.Tensor]:
    """Convolution `name` with its eval-mode BatchNorm folded in, fp64: w' = w s, b' = (b - mu) s + beta with
    s = gamma / sqrt(var + eps) and b the conv bias (ConvCompressH) or 0."""
    wk, bp, bk, *_ = CONVS[name]
    w = sd[wk].double()
    s = sd[f"{bp}.weight"].double() / torch.sqrt(sd[f"{bp}.running_var"].double() + BN_EPS)
    b = sd[bk].double() if bk else torch.zeros(w.shape[0], dtype=torch.float64)
    return w * s[:, None, None, None], (b - sd[f"{bp}.running_mean"].double()) * s + sd[f"{bp}.bias"].double()


def pack_weight(w: torch.Tensor, cin_pad: int) -> torch.Tensor:
    """[Cout, Cin, k, k] -> pf_hnet_conv's fp16 [k*k][Cin_pad][Cout] (tap-major ky, kx; zero rows past Cin)."""
    cout, cin, kh, kw = w.shape
    p = torch.zeros(kh * kw, cin_pad, cout, dtype=torch.float64)
    p[:, :cin] = w.permute(2, 3, 1, 0).reshape(kh * kw, cin, cout)
    return p.half()


def pack_whh(w: torch.Tensor) -> torch.Tensor:
    """W_hh [2048, 512] -> pf_lstm_bidir's [16][128][512]: CTA r's row (q, u) is W_hh[q * 512 + 32 r + u]."""
    return w.reshape(4, 16, 32, 512).permute(1, 0, 2, 3).reshape(16, 128, 512)


class HorizonNetModule(nn.Module):
    """The reference HorizonNetModule's forward(x) -> (bon fp32 [B, 2, 1024], cor fp32 [B, 1, 1024]) on the GPU for
    fp32 CUDA images [B, C >= 3, 512, 1024] (other sizes raise NotImplementedError, as the reference does). `state`:
    see load_state. The packed weights are non-persistent buffers, so .to(device) moves them."""

    def __init__(self, state, device: torch.device | str | None = None):
        super().__init__()
        sd = load_state(state)
        for name, (_wk, _bp, _bk, cin, _co, _k, _s) in CONVS.items():
            w, b = fold_bn(sd, name)
            self.register_buffer(f"{name}_w", pack_weight(w, PREP_C if cin == 3 else cin), persistent=False)
            self.register_buffer(f"{name}_b", b.float(), persistent=False)
        for layer in (0, 1):
            wih = torch.cat([sd[_lstm_key("weight_ih", layer, r)] for r in (False, True)])
            bias = torch.cat([sd[_lstm_key("bias_ih", layer, r)].double() + sd[_lstm_key("bias_hh", layer, r)].double()
                              for r in (False, True)])
            whh = torch.stack([pack_whh(sd[_lstm_key("weight_hh", layer, r)]) for r in (False, True)])
            self.register_buffer(f"wih{layer}", wih.half().contiguous(), persistent=False)
            self.register_buffer(f"bias{layer}", bias.float(), persistent=False)
            self.register_buffer(f"whh{layer}", whh.half().contiguous(), persistent=False)
        self.register_buffer("head_w", sd["linear.weight"].float().contiguous(), persistent=False)
        self.register_buffer("head_b", sd["linear.bias"].float().contiguous(), persistent=False)
        if device is not None:
            self.to(device)

    # ---- launches ----
    def _conv(self, name, x, relu=True, residual=None):
        _wk, _bp, _bk, _ci, cout, k, (sh, sw) = CONVS[name]
        B, Hi, Wi, cin = x.shape
        p = k // 2
        out = torch.empty(B, (Hi + 2 * p - k) // sh + 1, (Wi + 2 * p - k) // sw + 1, cout, device=x.device,
                          dtype=torch.float16)
        _lib.check(self._l.pf_hnet_conv(
            C.c_void_p(x.data_ptr()), B, Hi, Wi, cin, C.c_void_p(getattr(self, f"{name}_w").data_ptr()),
            C.c_void_p(getattr(self, f"{name}_b").data_ptr()), cout, k, sh, sw, int(relu),
            C.c_void_p(residual.data_ptr() if residual is not None else 0), C.c_void_p(out.data_ptr()), _lib.PF_F16,
            C.c_void_p(self._st)))
        return out

    def _encoder(self, x):
        B = x.shape[0]
        x = self._conv("stem", x)
        y = torch.empty(B, x.shape[1] // 2, x.shape[2] // 2, 64, device=x.device, dtype=torch.float16)
        _lib.check(self._l.pf_pool2d_nhwc(C.c_void_p(x.data_ptr()), B, x.shape[1], x.shape[2], 64, MAX, 2, 1,
                                          C.c_void_p(y.data_ptr()), 64, 0, C.c_void_p(self._st)))
        feats = []
        for li, (n, _w, _s) in enumerate(LAYERS, 1):
            for j in range(n):
                idt = self._conv(f"l{li}_{j}_ds", y, relu=False) if j == 0 else y
                t = self._conv(f"l{li}_{j}_c2", self._conv(f"l{li}_{j}_c1", y))
                y = self._conv(f"l{li}_{j}_c3", t, residual=idt)
            feats.append(y)
        return feats

    def _lstm_input(self, feats):
        B = feats[0].shape[0]
        out = torch.empty(T * B, 1024, device=feats[0].device, dtype=torch.float16)
        off = 0
        for s, y in enumerate(feats):
            for l in range(4):
                y = self._conv(f"h{s}_{l}", y)
            _B, h, w, c = y.shape
            _lib.check(self._l.pf_hnet_height_upsample(C.c_void_p(y.data_ptr()), B, h, w, c, T,
                                                       C.c_void_p(out.data_ptr()), off, C.c_void_p(self._st)))
            off += c * h
        return out

    def _lstm(self, x, layer, B):
        xproj = torch.empty(T * B, 4096, device=x.device, dtype=torch.float32)
        ops.gemm_taps(x, getattr(self, f"wih{layer}"), xproj, M=T * B, Kc=1024, bias=getattr(self, f"bias{layer}"),
                      block_n=128, k_splits=1)
        out = torch.empty(T * B, 1024, device=x.device, dtype=torch.float16)
        _lib.check(self._l.pf_lstm_bidir(C.c_void_p(xproj.data_ptr()), C.c_void_p(getattr(self, f"whh{layer}").data_ptr()),
                                         T, B, C.c_void_p(out.data_ptr()), C.c_void_p(self._st)))
        return out

    def _head(self, y, B):
        bon = torch.empty(B, 2, 4 * T, device=y.device, dtype=torch.float32)
        cor = torch.empty(B, 1, 4 * T, device=y.device, dtype=torch.float32)
        _lib.check(self._l.pf_hnet_head(C.c_void_p(y.data_ptr()), T, B, C.c_void_p(self.head_w.data_ptr()),
                                        C.c_void_p(self.head_b.data_ptr()), C.c_void_p(bon.data_ptr()),
                                        C.c_void_p(cor.data_ptr()), C.c_void_p(self._st)))
        return bon, cor

    def _chunk(self, x):
        B = x.shape[0]
        p = torch.empty(B, H, W, PREP_C, device=x.device, dtype=torch.float16)
        _lib.check(self._l.pf_hnet_prep(C.c_void_p(x.data_ptr()), B, x.shape[1], H, W, C.c_void_p(p.data_ptr()),
                                        C.c_void_p(self._st)))
        y = self._lstm_input(self._encoder(p))
        y = self._lstm(self._lstm(y, 0, B), 1, B)
        return self._head(y, B)

    @torch.no_grad()
    def forward(self, x: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
        if x.shape[2] != H or x.shape[3] != W:
            raise NotImplementedError()
        _lib.require_cuda(x)
        if x.device != self.head_w.device:
            raise ValueError(f"images are on {x.device} but the network's weights on {self.head_w.device}; "
                             "move the module with .to(device)")
        if x.dtype != torch.float32 or x.dim() != 4 or x.shape[1] < 3:
            raise ValueError(f"expected fp32 images [B, C >= 3, 512, 1024], got {x.dtype} {tuple(x.shape)}")
        x = x.contiguous()
        with torch.cuda.device(x.device):
            self._l, self._st = _lib.lib(), _lib.stream_ptr()
            outs = [self._chunk(c) for c in x.split(MAX_BATCH)]
        if len(outs) == 1:
            return outs[0]
        return torch.cat([o[0] for o in outs]), torch.cat([o[1] for o in outs])
