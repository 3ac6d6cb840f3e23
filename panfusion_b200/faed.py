"""FAED, the Fréchet AutoEncoder Distance of PanFusion (models/faed/FAED.py:50-103), on the sm_90a kernels.

`FAEDEncoder` runs the FAED encoder (models/faed/modules.py:176-264) on `pf_conv_circ` with eval-mode BatchNorm folded
into the convolutions (fp64 on the host, packed once) and returns the latitude-weighted features of FAED.py:69-78.
`FrechetAutoEncoderDistance` keeps the reference metric's fp64 states under the reference's names (a sum all-reduce
merges ranks) and computes the distance with `pf_frechet_fp64`. Both are `nn.Module`s: they are built on the CPU like
the reference metric, go into an `nn.ModuleDict` like `EvalPanoGen`'s, and `.to(device)` moves the packed weights and
the states (non-persistent buffers, as torchmetrics keeps its states out of the state dict).

Deviation: H and W must be multiples of 32 (the reference floors the odd rows and columns away in its stride-2 layers);
anything else raises ValueError.
"""
from __future__ import annotations

import ctypes as C
import math

import torch
from torch import nn

from . import _lib

BN_EPS = 1e-5
# (name, Cin, Cout, k, stride, pad) in Encoder.forward order; ResBlocks are (name, C, C, k, 1, k // 2)
CONVS = [("downconv1_rgb", 3, 32, 9, 1, 4)]
RES = {"downres1_rgb": (32, 9), "downres2_rgb": (64, 7), "downres3_rgb": (128, 5), "downres4_rgb": (128, 3),
       "downres5_rgb": (128, 3)}
DOWN = {"downconv2_rgb": (32, 64), "downconv3_rgb": (64, 128), "downconv4_rgb": (128, 128),
        "downconv5_rgb": (128, 128), "downconv6_rgb": (128, 128)}
ORDER = ["downconv1_rgb", "downres1_rgb", "downconv2_rgb", "downres2_rgb", "downconv3_rgb", "downres3_rgb",
         "downconv4_rgb", "downres4_rgb", "downconv5_rgb", "downres5_rgb", "downconv6_rgb", "fuse"]
PREP_C = 16  # pf_faed_prep's channel count: 3 image channels and 13 zeros


def _state_dict(encoder) -> dict[str, torch.Tensor]:
    sd = encoder.state_dict() if hasattr(encoder, "state_dict") else dict(encoder)
    return {k: v.detach().cpu() for k, v in sd.items()}


def fold_conv(sd: dict, conv: str, bn: str | None) -> tuple[torch.Tensor, torch.Tensor]:
    """Weight [Cout, Cin, k, k] and bias [Cout] of `conv` (a modules.Conv2d prefix) with the eval-mode BatchNorm `bn`
    folded in, in fp64: w * g / sqrt(var + eps), (b - mean) * g / sqrt(var + eps) + beta."""
    w = sd[f"{conv}.conv2d.weight"].double()
    b = sd[f"{conv}.conv2d.bias"].double()
    if bn is not None:
        s = sd[f"{bn}.weight"].double() / torch.sqrt(sd[f"{bn}.running_var"].double() + BN_EPS)
        w = w * s[:, None, None, None]
        b = (b - sd[f"{bn}.running_mean"].double()) * s + sd[f"{bn}.bias"].double()
    return w, b


def _layers(sd: dict) -> list[tuple]:
    """(folded w, folded b, k, stride, pad, relu, residual role) for every convolution in forward order; role is
    'save' (ResBlock input kept for the add), 'add' (ResBlock conv2) or None."""
    out = []
    for name in ORDER:
        if name == "downconv1_rgb":
            out.append((*fold_conv(sd, name, None), 9, 1, 4, False, None))
        elif name == "fuse":
            out.append((*fold_conv(sd, name, None), 3, 1, 1, False, None))
        elif name in DOWN:
            out.append((*fold_conv(sd, f"{name}.conv1", f"{name}.batchnorm1"), 4, 2, 1, True, None))
        else:
            k = RES[name][1]
            out.append((*fold_conv(sd, f"{name}.conv1", f"{name}.batchnorm1"), k, 1, k // 2, True, "save"))
            out.append((*fold_conv(sd, f"{name}.conv2", f"{name}.batchnorm2"), k, 1, k // 2, False, "add"))
    return out


def pack_weight(w: torch.Tensor, cin_pad: int, dtype: torch.dtype) -> torch.Tensor:
    """[Cout, Cin, k, k] -> pf_conv_circ's [k*k][Cin_pad][Cout] (tap-major ky, kx; zero rows for padded channels)."""
    cout, cin, k, _ = w.shape
    p = torch.zeros(k * k, cin_pad, cout, dtype=torch.float64)
    p[:, :cin] = w.permute(2, 3, 1, 0).reshape(k * k, cin, cout)
    return p.to(dtype)


def latitude_weight(h: int) -> torch.Tensor:
    """cos(torch.linspace(pi/2, -pi/2, h)) in fp32, as FAED.py:73-75 computes it."""
    return torch.cos(torch.linspace(math.pi / 2, -math.pi / 2, h, dtype=torch.float32))


class FAEDEncoder(nn.Module):
    """The FAED encoder on `pf_conv_circ`. `encoder` is the reference `Encoder` module or a state dict with its names
    (`downconv1_rgb.conv2d.weight`, `downres1_rgb.batchnorm1.running_var`, ...). fp16 operands: the same 10-bit
    mantissa as the TF32 convolutions cuDNN runs for the reference. The packed weights are buffers `w{i}` / `b{i}`."""

    def __init__(self, encoder, device: torch.device | str | None = None):
        super().__init__()
        self.layers = []
        for i, (w, b, k, s, p, relu, role) in enumerate(_layers(_state_dict(encoder))):
            cin = PREP_C if w.shape[1] == 3 else w.shape[1]
            self.register_buffer(f"w{i}", pack_weight(w, cin, torch.float16), persistent=False)
            self.register_buffer(f"b{i}", b.float(), persistent=False)
            self.layers.append(dict(cin=cin, cout=w.shape[0], k=k, s=s, p=p, relu=relu, role=role))
        self._lat: dict[tuple, torch.Tensor] = {}
        if device is not None:
            self.to(device)

    def _latitude(self, h: int, device: torch.device) -> torch.Tensor:
        key = (h, device)
        if key not in self._lat:
            self._lat[key] = latitude_weight(h).to(device)
        return self._lat[key]

    @torch.no_grad()
    def forward(self, imgs: torch.Tensor) -> torch.Tensor:
        """uint8 (or float) images [B, C >= 3, H, W] on the GPU -> fp32 features [B, 128 * H / 32] (FAED.py:69-78)."""
        _lib.require_cuda(imgs)
        if self.w0.device != imgs.device:
            raise ValueError(f"images are on {imgs.device} but the encoder's weights on {self.w0.device}; "
                             "move the module with .to(device)")
        if imgs.dim() != 4 or imgs.shape[1] < 3:
            raise ValueError(f"expected images [B, C >= 3, H, W], got {tuple(imgs.shape)}")
        B, Cimg, H, W = imgs.shape
        if H % 32 or W % 32:
            raise ValueError(f"FAED needs H and W that are multiples of 32, got {H}x{W}")
        if imgs.dtype == torch.uint8:
            is_u8 = 1
        elif imgs.dtype == torch.float32:
            is_u8 = 0
        else:
            raise ValueError(f"images must be uint8 or float32, got {imgs.dtype}")
        imgs = imgs.contiguous()
        with torch.cuda.device(imgs.device):
            l, st = _lib.lib(), _lib.stream_ptr()
            x = torch.empty(B, H, W, PREP_C, device=imgs.device, dtype=torch.float16)
            _lib.check(l.pf_faed_prep(C.c_void_p(imgs.data_ptr()), is_u8, B, Cimg, H, W, C.c_void_p(x.data_ptr()),
                                      C.c_void_p(st)))
            saved = None
            for i, L in enumerate(self.layers):
                h, w = x.shape[1], x.shape[2]
                ho, wo = (h + 2 * L["p"] - L["k"]) // L["s"] + 1, (w + 2 * L["p"] - L["k"]) // L["s"] + 1
                last = i == len(self.layers) - 1
                y = torch.empty(B, ho, wo, L["cout"], device=imgs.device,
                                dtype=torch.float32 if last else torch.float16)
                if L["role"] == "save":
                    saved = x
                res = saved if L["role"] == "add" else None
                _lib.check(l.pf_conv_circ(C.c_void_p(x.data_ptr()), B, h, w, L["cin"],
                                          C.c_void_p(getattr(self, f"w{i}").data_ptr()),
                                          C.c_void_p(getattr(self, f"b{i}").data_ptr()), L["cout"], L["k"], L["s"],
                                          L["p"], int(L["relu"]), C.c_void_p(_lib.ptr(res)), C.c_void_p(y.data_ptr()),
                                          _lib.PF_F32 if last else _lib.PF_F16, C.c_void_p(st)))
                x = y
            h, w = x.shape[1], x.shape[2]
            feats = torch.empty(B, 128 * h, device=imgs.device, dtype=torch.float32)
            _lib.check(l.pf_faed_pool(C.c_void_p(x.data_ptr()), B, h, w, 128,
                                      C.c_void_p(self._latitude(h, imgs.device).data_ptr()),
                                      C.c_void_p(feats.data_ptr()), C.c_void_p(st)))
        return feats


def load_encoder_state(ckpt_path: str) -> dict[str, torch.Tensor]:
    """The encoder's state dict from the FAED Lightning checkpoint: `state_dict` entries under `net.encoder.`."""
    ck = torch.load(ckpt_path, map_location="cpu", weights_only=False)
    sd = ck.get("state_dict", ck)
    pre = "net.encoder."
    out = {k[len(pre):]: v for k, v in sd.items() if k.startswith(pre)}
    if not out:
        raise ValueError(f"{ckpt_path}: no `net.encoder.` entries in its state_dict")
    return out


def frechet_distance(sum1, cov_sum1, n1: int, sum2, cov_sum2, n2: int, return_sweeps: bool = False):
    """pf_frechet_fp64 on fp64 CUDA statistics -> 0-d fp64 CUDA tensor (and, with return_sweeps, the sweep counts of
    the Jacobi iterations on S1, S2 and L1^T L2)."""
    _lib.require_cuda(sum1, cov_sum1, sum2, cov_sum2)
    d = sum1.numel()
    for t in (sum1, cov_sum1, sum2, cov_sum2):
        if t.dtype != torch.float64 or not t.is_contiguous():
            raise ValueError("statistics must be contiguous fp64 tensors")
        if t.device != sum1.device:
            raise ValueError("statistics are on different devices")
    if cov_sum1.shape != (d, d) or cov_sum2.shape != (d, d) or sum2.numel() != d:
        raise ValueError("statistics shapes disagree")
    l = _lib.lib()
    l.pf_frechet_ws_doubles.restype = C.c_longlong
    sweeps = (C.c_int * 3)()
    with torch.cuda.device(sum1.device):
        ws = torch.empty(l.pf_frechet_ws_doubles(d), device=sum1.device, dtype=torch.float64)
        out = torch.empty((), device=sum1.device, dtype=torch.float64)
        _lib.check(l.pf_frechet_fp64(C.c_void_p(sum1.data_ptr()), C.c_void_p(cov_sum1.data_ptr()), C.c_longlong(n1),
                                     C.c_void_p(sum2.data_ptr()), C.c_void_p(cov_sum2.data_ptr()), C.c_longlong(n2),
                                     d, C.c_void_p(ws.data_ptr()), C.c_void_p(out.data_ptr()), sweeps,
                                     C.c_void_p(_lib.stream_ptr())))
    return (out, list(sweeps)) if return_sweeps else out


class FrechetAutoEncoderDistance(nn.Module):
    """models/faed/FAED.py:50-103 on the GPU: update(imgs, real), compute() -> 0-d fp64 CUDA tensor, reset().
    Built on `device` (the CPU by default, like the reference); `.to(device)` moves weights and states together."""

    higher_is_better = False

    def __init__(self, pano_height: int, encoder=None, ckpt_path: str = "weights/faed.ckpt",
                 device: torch.device | str | None = None):
        super().__init__()
        self.pano_height = pano_height
        if encoder is None:
            encoder = load_encoder_state(ckpt_path)
        self.encoder = encoder if isinstance(encoder, FAEDEncoder) else FAEDEncoder(encoder)
        d = pano_height * 4
        self.num_features = d
        for side in ("real", "fake"):
            self.register_buffer(f"{side}_features_sum", torch.zeros(d, dtype=torch.float64), persistent=False)
            self.register_buffer(f"{side}_features_cov_sum", torch.zeros(d, d, dtype=torch.float64),
                                 persistent=False)
            self.register_buffer(f"{side}_features_num_samples", torch.zeros((), dtype=torch.int64),
                                 persistent=False)
        self._update_called = False
        if device is not None:
            self.to(device)

    def reset(self) -> None:
        for side in ("real", "fake"):
            for k in ("sum", "cov_sum", "num_samples"):
                getattr(self, f"{side}_features_{k}").zero_()
        self._update_called = False

    @torch.no_grad()
    def update(self, imgs: torch.Tensor, real: bool) -> None:
        _lib.require_cuda(imgs)
        if imgs.device != self.real_features_sum.device:
            raise ValueError(f"images are on {imgs.device} but the metric's states on "
                             f"{self.real_features_sum.device}; move the metric with .to(device)")
        if imgs.dim() != 4 or imgs.shape[2] != self.pano_height:
            raise ValueError(f"expected panoramas [B, C, {self.pano_height}, W], got {tuple(imgs.shape)}")
        feats = self.encoder(imgs)
        side = "real" if real else "fake"
        s, c = getattr(self, f"{side}_features_sum"), getattr(self, f"{side}_features_cov_sum")
        with torch.cuda.device(imgs.device):
            _lib.check(_lib.lib().pf_faed_stats(C.c_void_p(feats.data_ptr()), feats.shape[0], feats.shape[1],
                                                C.c_void_p(s.data_ptr()), C.c_void_p(c.data_ptr()),
                                                C.c_void_p(_lib.stream_ptr())))
        getattr(self, f"{side}_features_num_samples").add_(imgs.shape[0])
        self._update_called = True

    def compute(self) -> torch.Tensor:
        n1, n2 = int(self.real_features_num_samples), int(self.fake_features_num_samples)
        if n1 < 2 or n2 < 2:
            raise RuntimeError("More than one sample is required for both the real and fake distributed to compute FID")
        return frechet_distance(self.real_features_sum, self.real_features_cov_sum, n1,
                                self.fake_features_sum, self.fake_features_cov_sum, n2)
