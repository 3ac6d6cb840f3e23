"""FID and Inception Score (torchmetrics' FrechetInceptionDistance / InceptionScore, as models/pano/EvalPanoGen.py:30-49
builds them) on the sm_90a kernels.

`InceptionV3` is torch-fidelity's FeatureExtractorInceptionV3, the network behind torchmetrics' NoTrainInceptionV3: the
TF1-style resize to 299x299 (`pf_inception_prep`), 94 BasicConv2d layers on the implicit-GEMM convolution shared with
FAED (`pf_conv2d_nhwc`, BN folded in fp64 on the host and packed once), the 3x3 pools (`pf_pool2d_nhwc`) and the
pool3 / logits head (`pf_inception_head`). Each branch writes straight into its slice of the block's concat buffer.
`FrechetInceptionDistance` accumulates pool3 with `pf_faed_stats` into fp64 states under torchmetrics' names and
computes the distance with `faed.frechet_distance`; `InceptionScore` keeps the logits and reduces them with
`pf_inception_score`. All three are `nn.Module`s built on the CPU; `.to(device)` moves the packed weights and the states.
"""
from __future__ import annotations

import ctypes as C

import torch
from torch import nn

from . import _lib
from .faed import frechet_distance

BN_EPS = 1e-3
SIZE = 299
PREP_C = 16  # pf_inception_prep's channel count: 3 image channels and 13 zeros
FEATURES = 2048
CLASSES = 1008
MAX, AVG = 0, 1  # PF_POOL_MAX, PF_POOL_AVG_EXCL_PAD
WEIGHTS = "weights/pt_inception-2015-12-05-6726825d.pth"  # torch-fidelity's FID InceptionV3 weights


def _conv_table() -> dict[str, tuple]:
    """BasicConv2d name -> (Cin, Cout, kh, kw, stride, ph, pw), in forward order (torchvision's Inception3 topology)."""
    T = {}

    def c(name, cin, cout, k=(1, 1), s=1, p=(0, 0)):
        T[name] = (cin, cout, *k, s, *p)

    c("Conv2d_1a_3x3", 3, 32, (3, 3), 2)
    c("Conv2d_2a_3x3", 32, 32, (3, 3))
    c("Conv2d_2b_3x3", 32, 64, (3, 3), p=(1, 1))
    c("Conv2d_3b_1x1", 64, 80)
    c("Conv2d_4a_3x3", 80, 192, (3, 3))
    for blk, cin, pool in (("Mixed_5b", 192, 32), ("Mixed_5c", 256, 64), ("Mixed_5d", 288, 64)):
        c(f"{blk}.branch1x1", cin, 64)
        c(f"{blk}.branch5x5_1", cin, 48)
        c(f"{blk}.branch5x5_2", 48, 64, (5, 5), p=(2, 2))
        c(f"{blk}.branch3x3dbl_1", cin, 64)
        c(f"{blk}.branch3x3dbl_2", 64, 96, (3, 3), p=(1, 1))
        c(f"{blk}.branch3x3dbl_3", 96, 96, (3, 3), p=(1, 1))
        c(f"{blk}.branch_pool", cin, pool)
    c("Mixed_6a.branch3x3", 288, 384, (3, 3), 2)
    c("Mixed_6a.branch3x3dbl_1", 288, 64)
    c("Mixed_6a.branch3x3dbl_2", 64, 96, (3, 3), p=(1, 1))
    c("Mixed_6a.branch3x3dbl_3", 96, 96, (3, 3), 2)
    row, col = ((1, 7), (0, 3)), ((7, 1), (3, 0))
    for blk, c7 in (("Mixed_6b", 128), ("Mixed_6c", 160), ("Mixed_6d", 160), ("Mixed_6e", 192)):
        c(f"{blk}.branch1x1", 768, 192)
        c(f"{blk}.branch7x7_1", 768, c7)
        c(f"{blk}.branch7x7_2", c7, c7, row[0], p=row[1])
        c(f"{blk}.branch7x7_3", c7, 192, col[0], p=col[1])
        c(f"{blk}.branch7x7dbl_1", 768, c7)
        c(f"{blk}.branch7x7dbl_2", c7, c7, col[0], p=col[1])
        c(f"{blk}.branch7x7dbl_3", c7, c7, row[0], p=row[1])
        c(f"{blk}.branch7x7dbl_4", c7, c7, col[0], p=col[1])
        c(f"{blk}.branch7x7dbl_5", c7, 192, row[0], p=row[1])
        c(f"{blk}.branch_pool", 768, 192)
    c("Mixed_7a.branch3x3_1", 768, 192)
    c("Mixed_7a.branch3x3_2", 192, 320, (3, 3), 2)
    c("Mixed_7a.branch7x7x3_1", 768, 192)
    c("Mixed_7a.branch7x7x3_2", 192, 192, row[0], p=row[1])
    c("Mixed_7a.branch7x7x3_3", 192, 192, col[0], p=col[1])
    c("Mixed_7a.branch7x7x3_4", 192, 192, (3, 3), 2)
    for blk, cin in (("Mixed_7b", 1280), ("Mixed_7c", 2048)):
        c(f"{blk}.branch1x1", cin, 320)
        c(f"{blk}.branch3x3_1", cin, 384)
        c(f"{blk}.branch3x3_2a", 384, 384, (1, 3), p=(0, 1))
        c(f"{blk}.branch3x3_2b", 384, 384, (3, 1), p=(1, 0))
        c(f"{blk}.branch3x3dbl_1", cin, 448)
        c(f"{blk}.branch3x3dbl_2", 448, 384, (3, 3), p=(1, 1))
        c(f"{blk}.branch3x3dbl_3a", 384, 384, (1, 3), p=(0, 1))
        c(f"{blk}.branch3x3dbl_3b", 384, 384, (3, 1), p=(1, 0))
        c(f"{blk}.branch_pool", cin, 192)
    return T


CONVS = _conv_table()


def load_state(state) -> dict[str, torch.Tensor]:
    """A state dict with torch-fidelity's key names (or the path of pt_inception-2015-12-05-6726825d.pth), checked:
    every key the network reads must be present with its shape, else ValueError naming it."""
    if isinstance(state, (str, bytes)) or hasattr(state, "__fspath__"):
        state = torch.load(state, map_location="cpu", weights_only=True)
    sd = {k: v.detach().cpu() for k, v in dict(state).items()}
    want = {"fc.weight": (CLASSES, FEATURES)}
    for name, (cin, cout, kh, kw, *_rest) in CONVS.items():
        want[f"{name}.conv.weight"] = (cout, cin, kh, kw)
        for p in ("weight", "bias", "running_mean", "running_var"):
            want[f"{name}.bn.{p}"] = (cout,)
    for k, shape in want.items():
        if k not in sd:
            raise ValueError(f"InceptionV3 state dict: missing key {k!r}")
        if tuple(sd[k].shape) != shape:
            raise ValueError(f"InceptionV3 state dict: {k!r} has shape {tuple(sd[k].shape)}, expected {shape}")
    return sd


def fold_bn(sd: dict, name: str) -> tuple[torch.Tensor, torch.Tensor]:
    """BasicConv2d `name` with its eval-mode BatchNorm (eps 1e-3) folded in, in fp64: weight [Cout, Cin, kh, kw] and
    bias [Cout]."""
    w = sd[f"{name}.conv.weight"].double()
    s = sd[f"{name}.bn.weight"].double() / torch.sqrt(sd[f"{name}.bn.running_var"].double() + BN_EPS)
    b = sd[f"{name}.bn.bias"].double() - sd[f"{name}.bn.running_mean"].double() * s
    return w * s[:, None, None, None], b


def packed_cout(cout: int) -> int:
    """pf_conv2d_packed_cout: the zero-padded width of a packed weight / bias."""
    return 32 if cout <= 32 else (cout + 63) // 64 * 64


def pack_weight(w: torch.Tensor, cin_pad: int) -> torch.Tensor:
    """[Cout, Cin, kh, kw] -> pf_conv2d_nhwc's fp16 [kh*kw][Cin_pad][Cw] (tap-major ky, kx; zero rows and columns)."""
    cout, cin, kh, kw = w.shape
    p = torch.zeros(kh * kw, cin_pad, packed_cout(cout), dtype=torch.float64)
    p[:, :cin, :cout] = w.permute(2, 3, 1, 0).reshape(kh * kw, cin, cout)
    return p.half()


def _key(name: str) -> str:
    return name.replace(".", "_")


class InceptionV3(nn.Module):
    """torch-fidelity's FeatureExtractorInceptionV3 on the GPU: forward(uint8 [B, 3, H, W]) -> (pool3 fp32 [B, 2048],
    logits_unbiased fp32 [B, 1008]). `state` is a state dict with torch-fidelity's key names or the path of its
    weights file; nothing is downloaded. The packed weights are non-persistent buffers `{layer}_w` / `{layer}_b` and
    `fc_w`."""

    def __init__(self, state, device: torch.device | str | None = None):
        super().__init__()
        sd = load_state(state)
        for name, (cin, cout, *_rest) in CONVS.items():
            w, b = fold_bn(sd, name)
            bias = torch.zeros(packed_cout(cout), dtype=torch.float32)
            bias[:cout] = b.float()
            self.register_buffer(f"{_key(name)}_w", pack_weight(w, PREP_C if cin == 3 else cin), persistent=False)
            self.register_buffer(f"{_key(name)}_b", bias, persistent=False)
        self.register_buffer("fc_w", sd["fc.weight"].float().contiguous(), persistent=False)
        if device is not None:
            self.to(device)

    # ---- launches ----
    def _conv(self, name, x, out=None, off=0, f32=False):
        cin, cout, kh, kw, s, ph, pw = CONVS[name]
        B, H, W, c = x.shape
        ho, wo = (H + 2 * ph - kh) // s + 1, (W + 2 * pw - kw) // s + 1
        if out is None:
            out = torch.empty(B, ho, wo, cout, device=x.device, dtype=torch.float32 if f32 else torch.float16)
        _lib.check(self._l.pf_conv2d_nhwc(
            C.c_void_p(x.data_ptr()), B, H, W, c, C.c_void_p(getattr(self, f"{_key(name)}_w").data_ptr()),
            C.c_void_p(getattr(self, f"{_key(name)}_b").data_ptr()), cout, kh, kw, s, ph, pw, 1,
            C.c_void_p(out.data_ptr()), _lib.PF_F32 if out.dtype == torch.float32 else _lib.PF_F16, out.shape[-1], off,
            C.c_void_p(self._st)))
        return out

    def _pool(self, x, mode, stride, pad, out=None, off=0):
        B, H, W, c = x.shape
        ho, wo = (H + 2 * pad - 3) // stride + 1, (W + 2 * pad - 3) // stride + 1
        if out is None:
            out = torch.empty(B, ho, wo, c, device=x.device, dtype=torch.float16)
        _lib.check(self._l.pf_pool2d_nhwc(C.c_void_p(x.data_ptr()), B, H, W, c, mode, stride, pad,
                                          C.c_void_p(out.data_ptr()), out.shape[-1], off, C.c_void_p(self._st)))
        return out

    def _cat(self, x, hw, c, f32=False):
        return torch.empty(x.shape[0], hw, hw, c, device=x.device, dtype=torch.float32 if f32 else torch.float16)

    def _mixed_a(self, blk, x):
        out = self._cat(x, 35, 224 + CONVS[f"{blk}.branch_pool"][1])
        self._conv(f"{blk}.branch1x1", x, out, 0)
        self._conv(f"{blk}.branch5x5_2", self._conv(f"{blk}.branch5x5_1", x), out, 64)
        d = self._conv(f"{blk}.branch3x3dbl_2", self._conv(f"{blk}.branch3x3dbl_1", x))
        self._conv(f"{blk}.branch3x3dbl_3", d, out, 128)
        self._conv(f"{blk}.branch_pool", self._pool(x, AVG, 1, 1), out, 224)
        return out

    def _mixed_6a(self, x):
        out = self._cat(x, 17, 768)
        self._conv("Mixed_6a.branch3x3", x, out, 0)
        d = self._conv("Mixed_6a.branch3x3dbl_2", self._conv("Mixed_6a.branch3x3dbl_1", x))
        self._conv("Mixed_6a.branch3x3dbl_3", d, out, 384)
        self._pool(x, MAX, 2, 0, out, 480)
        return out

    def _mixed_c(self, blk, x):
        out = self._cat(x, 17, 768)
        self._conv(f"{blk}.branch1x1", x, out, 0)
        t = self._conv(f"{blk}.branch7x7_2", self._conv(f"{blk}.branch7x7_1", x))
        self._conv(f"{blk}.branch7x7_3", t, out, 192)
        d = self._conv(f"{blk}.branch7x7dbl_1", x)
        for i in (2, 3, 4):
            d = self._conv(f"{blk}.branch7x7dbl_{i}", d)
        self._conv(f"{blk}.branch7x7dbl_5", d, out, 384)
        self._conv(f"{blk}.branch_pool", self._pool(x, AVG, 1, 1), out, 576)
        return out

    def _mixed_7a(self, x):
        out = self._cat(x, 8, 1280)
        self._conv("Mixed_7a.branch3x3_2", self._conv("Mixed_7a.branch3x3_1", x), out, 0)
        t = self._conv("Mixed_7a.branch7x7x3_1", x)
        for i in (2, 3):
            t = self._conv(f"Mixed_7a.branch7x7x3_{i}", t)
        self._conv("Mixed_7a.branch7x7x3_4", t, out, 320)
        self._pool(x, MAX, 2, 0, out, 512)
        return out

    def _mixed_e(self, blk, x, last):
        out = self._cat(x, 8, 2048, f32=last)  # Mixed_7c is fp32, so pool3 and the logits come from fp32
        self._conv(f"{blk}.branch1x1", x, out, 0)
        t = self._conv(f"{blk}.branch3x3_1", x)
        self._conv(f"{blk}.branch3x3_2a", t, out, 320)
        self._conv(f"{blk}.branch3x3_2b", t, out, 704)
        d = self._conv(f"{blk}.branch3x3dbl_2", self._conv(f"{blk}.branch3x3dbl_1", x))
        self._conv(f"{blk}.branch3x3dbl_3a", d, out, 1088)
        self._conv(f"{blk}.branch3x3dbl_3b", d, out, 1472)
        self._conv(f"{blk}.branch_pool", self._pool(x, MAX if last else AVG, 1, 1), out, 1856)
        return out

    @torch.no_grad()
    def forward(self, imgs: torch.Tensor, normalize: bool = False) -> tuple[torch.Tensor, torch.Tensor]:
        """uint8 [B, 3, H, W] CUDA images of any H, W (with normalize=True: fp32 in [0, 1], converted as
        `(imgs * 255).byte()` inside the prep kernel) -> (pool3 [B, 2048], logits_unbiased [B, 1008]), fp32."""
        _lib.require_cuda(imgs)
        if self.fc_w.device != imgs.device:
            raise ValueError(f"images are on {imgs.device} but the network's weights on {self.fc_w.device}; "
                             "move the module with .to(device)")
        if imgs.dim() != 4 or imgs.shape[1] != 3:
            raise ValueError(f"expected images [B, 3, H, W], got {tuple(imgs.shape)}")
        want = torch.float32 if normalize else torch.uint8
        if imgs.dtype != want:
            raise ValueError(f"expected {want} images (normalize={normalize}), got {imgs.dtype}")
        B, _, H, W = imgs.shape
        imgs = imgs.contiguous()
        with torch.cuda.device(imgs.device):
            self._l, self._st = _lib.lib(), _lib.stream_ptr()
            x = torch.empty(B, SIZE, SIZE, PREP_C, device=imgs.device, dtype=torch.float16)
            _lib.check(self._l.pf_inception_prep(C.c_void_p(imgs.data_ptr()), int(not normalize), B, H, W,
                                                 C.c_void_p(x.data_ptr()), C.c_void_p(self._st)))
            for name in ("Conv2d_1a_3x3", "Conv2d_2a_3x3", "Conv2d_2b_3x3"):
                x = self._conv(name, x)
            x = self._pool(x, MAX, 2, 0)
            x = self._conv("Conv2d_4a_3x3", self._conv("Conv2d_3b_1x1", x))
            x = self._pool(x, MAX, 2, 0)
            for blk in ("Mixed_5b", "Mixed_5c", "Mixed_5d"):
                x = self._mixed_a(blk, x)
            x = self._mixed_6a(x)
            for blk in ("Mixed_6b", "Mixed_6c", "Mixed_6d", "Mixed_6e"):
                x = self._mixed_c(blk, x)
            x = self._mixed_e("Mixed_7b", self._mixed_7a(x), last=False)
            x = self._mixed_e("Mixed_7c", x, last=True)
            pool3 = torch.empty(B, FEATURES, device=imgs.device, dtype=torch.float32)
            logits = torch.empty(B, CLASSES, device=imgs.device, dtype=torch.float32)
            _lib.check(self._l.pf_inception_head(C.c_void_p(x.data_ptr()), B, 64, FEATURES,
                                                 C.c_void_p(self.fc_w.data_ptr()), CLASSES,
                                                 C.c_void_p(pool3.data_ptr()), C.c_void_p(logits.data_ptr()),
                                                 C.c_void_p(self._st)))
        return pool3, logits


def _network(inception, weights_path) -> InceptionV3:
    if inception is None:
        return InceptionV3(weights_path)
    if not isinstance(inception, InceptionV3):
        raise ValueError(f"inception must be an InceptionV3, got {type(inception).__name__}")
    return inception


def _check_images(net: InceptionV3, imgs: torch.Tensor, normalize: bool) -> None:
    want = torch.float32 if normalize else torch.uint8
    if imgs.dtype != want:
        raise ValueError(f"expected {want} images (normalize={normalize}), got {imgs.dtype}")
    _lib.require_cuda(imgs)
    if imgs.device != net.fc_w.device:
        raise ValueError(f"images are on {imgs.device} but the metric's states on {net.fc_w.device}; "
                         "move the metric with .to(device)")


def _check_features(f: torch.Tensor, width: int, device: torch.device) -> None:
    _lib.require_cuda(f)
    if f.dtype != torch.float32 or f.dim() != 2 or f.shape[1] != width:
        raise ValueError(f"expected fp32 features [n, {width}], got {f.dtype} {tuple(f.shape)}")
    if f.device != device:
        raise ValueError(f"features are on {f.device} but the metric's states on {device}; "
                         "move the metric with .to(device)")


class FrechetInceptionDistance(nn.Module):
    """torchmetrics' FrechetInceptionDistance(feature=2048) on the GPU: update(imgs, real), compute() -> 0-d fp32 CUDA
    tensor, reset(). `inception=` shares one packed network between metric objects."""

    higher_is_better = False

    def __init__(self, feature: int = 2048, normalize: bool = False, inception: InceptionV3 | None = None,
                 weights_path: str = WEIGHTS, device: torch.device | str | None = None):
        super().__init__()
        if feature != FEATURES:
            raise ValueError(f"only feature=2048 (pool3) is supported, got {feature!r}")
        self.normalize = normalize
        self.inception = _network(inception, weights_path)
        for side in ("real", "fake"):
            self.register_buffer(f"{side}_features_sum", torch.zeros(FEATURES, dtype=torch.float64), persistent=False)
            self.register_buffer(f"{side}_features_cov_sum", torch.zeros(FEATURES, FEATURES, dtype=torch.float64),
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
        _check_images(self.inception, imgs, self.normalize)
        if imgs.device != self.real_features_sum.device:
            raise ValueError(f"images are on {imgs.device} but the metric's states on "
                             f"{self.real_features_sum.device}; move the metric with .to(device)")
        feats, _ = self.inception(imgs, normalize=self.normalize)
        self.update_features(feats, real)

    @torch.no_grad()
    def update_features(self, pool3: torch.Tensor, real: bool) -> None:
        """update() from pool3 features [n, 2048] fp32 (CUDA) that the caller took from this metric's network, so one
        forward can feed several metrics."""
        _check_features(pool3, FEATURES, self.real_features_sum.device)
        pool3 = pool3.contiguous()
        side = "real" if real else "fake"
        s, c = getattr(self, f"{side}_features_sum"), getattr(self, f"{side}_features_cov_sum")
        with torch.cuda.device(pool3.device):
            _lib.check(_lib.lib().pf_faed_stats(C.c_void_p(pool3.data_ptr()), pool3.shape[0], FEATURES,
                                                C.c_void_p(s.data_ptr()), C.c_void_p(c.data_ptr()),
                                                C.c_void_p(_lib.stream_ptr())))
        getattr(self, f"{side}_features_num_samples").add_(pool3.shape[0])
        self._update_called = True

    def compute(self) -> torch.Tensor:
        n1, n2 = int(self.real_features_num_samples), int(self.fake_features_num_samples)
        if n1 < 2 or n2 < 2:
            raise RuntimeError("More than one sample is required for both the real and fake distributed to compute FID")
        return frechet_distance(self.real_features_sum, self.real_features_cov_sum, n1,
                                self.fake_features_sum, self.fake_features_cov_sum, n2).float()


class InceptionScore(nn.Module):
    """torchmetrics' InceptionScore(feature='logits_unbiased') on the GPU: update(imgs), compute() -> (mean, std) as
    0-d fp32 CUDA tensors, reset(). The logits are kept in the list `features`; compute draws torch.randperm(n) from
    the global CPU generator, as torchmetrics does, and reduces on the device."""

    higher_is_better = True

    def __init__(self, feature: str = "logits_unbiased", splits: int = 10, normalize: bool = False,
                 inception: InceptionV3 | None = None, weights_path: str = WEIGHTS,
                 device: torch.device | str | None = None):
        super().__init__()
        if feature != "logits_unbiased":
            raise ValueError(f"only feature='logits_unbiased' is supported, got {feature!r}")
        if not isinstance(splits, int) or splits < 1:
            raise ValueError(f"splits must be a positive int, got {splits!r}")
        self.splits = splits
        self.normalize = normalize
        self.inception = _network(inception, weights_path)
        self.features: list[torch.Tensor] = []
        self._update_called = False
        if device is not None:
            self.to(device)

    def reset(self) -> None:
        self.features = []
        self._update_called = False

    @torch.no_grad()
    def update(self, imgs: torch.Tensor) -> None:
        _check_images(self.inception, imgs, self.normalize)
        self.update_logits(self.inception(imgs, normalize=self.normalize)[1])

    @torch.no_grad()
    def update_logits(self, logits: torch.Tensor) -> None:
        """update() from logits_unbiased [n, 1008] fp32 (CUDA) that the caller took from this metric's network. Rows
        are kept in call order, which compute()'s randperm indexes."""
        _check_features(logits, CLASSES, self.inception.fc_w.device)
        self.features.append(logits)
        self._update_called = True

    def compute(self) -> tuple[torch.Tensor, torch.Tensor]:
        if not self.features:
            raise RuntimeError("InceptionScore.compute() called before update()")
        f = torch.cat(self.features).contiguous()
        n = f.shape[0]
        idx = torch.randperm(n)
        l = _lib.lib()
        l.pf_inception_score_ws_doubles.restype = C.c_longlong
        with torch.cuda.device(f.device):
            perm = idx.to(f.device)
            ws = torch.empty(l.pf_inception_score_ws_doubles(n, CLASSES, self.splits), device=f.device,
                             dtype=torch.float64)
            out = torch.empty(2, device=f.device, dtype=torch.float32)
            _lib.check(l.pf_inception_score(C.c_void_p(f.data_ptr()), C.c_void_p(perm.data_ptr()), n, CLASSES,
                                            self.splits, C.c_void_p(ws.data_ptr()), C.c_void_p(out.data_ptr()),
                                            C.c_void_p(_lib.stream_ptr())))
        return out[0], out[1]
