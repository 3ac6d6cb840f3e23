"""Train the FAED autoencoder (models/faed/FAED.py:13-33: AutoEncoder, L1 loss, Adam, ExponentialLR) on the sm_90a
kernels of csrc/faed_train.cu, and write the Lightning checkpoint `FrechetAutoEncoderDistance` loads.

`FAEDTrainer.training_step` runs the training-mode forward (convolutions on the pf_conv_circ core with bias, BatchNorm
with batch statistics), the L1 loss, the backward (BatchNorm, ReLU and residual gradients, convolution data gradients
on the same core, tensor-core weight gradients, bilinear-upsample gathers) and Adam without a host synchronisation.
Parameters, their gradients and Adam's moments are flat fp32 device buffers in the reference's parameter order; the
fp16 packed weights are rewritten from them by the device after every step.

Activation gradients carry a power-of-two loss scale S with torch.cuda.amp.GradScaler's policy: a step whose loss or
gradients are not finite changes no parameter, moment, running statistic or step count and halves S; S doubles after
2000 clean steps. The reference never skips; `skipped_steps` counts the skips.
"""
from __future__ import annotations

import ctypes as C
import math
from collections import OrderedDict

import torch
import torch.nn.functional as F
from torch import nn

from . import _lib

BETAS = (0.9, 0.999)
ADAM_EPS = 1e-8
INIT_SCALE = 1.0  # seed magnitude 1: the activation gradients of this network stay well inside fp16's range
F16, F32 = _lib.PF_F16, _lib.PF_F32


# --------------------------------------------------------------------------------------------------------------------
# The module tree with the reference's names and construction order (so torch.manual_seed(seed) gives the same
# default initialisation as the reference's AutoEncoder()). Also the fp64 restatement the tests compare against.
# --------------------------------------------------------------------------------------------------------------------
def circular_pad(x: torch.Tensor, p: int) -> torch.Tensor:
    """CircularPadding: rows zero-padded, columns wrapped, corners zero."""
    if p == 0:
        return x
    x = F.pad(x, (0, 0, p, p))
    return torch.cat([x[..., -p:], x, x[..., :p]], dim=-1)


class CircConv2d(nn.Module):
    def __init__(self, cin, cout, k, stride, pad):
        super().__init__()
        self.pad = pad
        self.conv2d = nn.Conv2d(cin, cout, k, stride, padding=0)

    def forward(self, x):
        return self.conv2d(circular_pad(x, self.pad))


class ResBlock(nn.Module):
    def __init__(self, c, k):
        super().__init__()
        self.conv1 = CircConv2d(c, c, k, 1, k // 2)
        self.batchnorm1 = nn.BatchNorm2d(c)
        self.conv2 = CircConv2d(c, c, k, 1, k // 2)
        self.batchnorm2 = nn.BatchNorm2d(c)

    def forward(self, x):
        return self.batchnorm2(self.conv2(F.relu(self.batchnorm1(self.conv1(x))))) + x


class ConvBlock(nn.Module):
    def __init__(self, cin, cout, k, stride, pad):
        super().__init__()
        self.conv1 = CircConv2d(cin, cout, k, stride, pad)
        self.batchnorm1 = nn.BatchNorm2d(cout)

    def forward(self, x):
        return F.relu(self.batchnorm1(self.conv1(x)))


def _up(x):
    return F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=False)


# Encoder / Decoder forward order: ("conv" | "cb" | "rb" | "up", attribute, args)
ENC = [("conv", "downconv1_rgb", (3, 32, 9, 1, 4)), ("rb", "downres1_rgb", (32, 9)),
       ("cb", "downconv2_rgb", (32, 64, 4, 2, 1)), ("rb", "downres2_rgb", (64, 7)),
       ("cb", "downconv3_rgb", (64, 128, 4, 2, 1)), ("rb", "downres3_rgb", (128, 5)),
       ("cb", "downconv4_rgb", (128, 128, 4, 2, 1)), ("rb", "downres4_rgb", (128, 3)),
       ("cb", "downconv5_rgb", (128, 128, 4, 2, 1)), ("rb", "downres5_rgb", (128, 3)),
       ("cb", "downconv6_rgb", (128, 128, 4, 2, 1)), ("conv", "fuse", (128, 128, 3, 1, 1))]
DEC = [("up", None, None), ("cb", "upconv2_rgb", (128, 128, 3, 1, 1)), ("rb", "upres2_rgb", (128, 3)),
       ("up", None, None), ("cb", "upconv3_rgb", (128, 128, 3, 1, 1)), ("rb", "upres3_rgb", (128, 5)),
       ("up", None, None), ("cb", "upconv4_rgb", (128, 64, 3, 1, 1)), ("rb", "upres4_rgb", (64, 7)),
       ("up", None, None), ("cb", "upconv5_rgb", (64, 32, 3, 1, 1)), ("rb", "upres5_rgb", (32, 9)),
       ("up", None, None), ("conv", "outconv_rgb", (32, 3, 9, 1, 4))]
# construction order of modules.py's __init__s (it fixes the default initialisation's RNG draws)
ENC_INIT = ["downconv1_rgb", "downconv2_rgb", "downconv3_rgb", "downconv4_rgb", "downconv5_rgb", "downconv6_rgb",
            "downres1_rgb", "downres2_rgb", "downres3_rgb", "downres4_rgb", "downres5_rgb", "fuse"]
DEC_INIT = ["upconv2_rgb", "upconv3_rgb", "upconv4_rgb", "upconv5_rgb", "outconv_rgb", "upres2_rgb", "upres3_rgb",
            "upres4_rgb", "upres5_rgb"]


class _Stack(nn.Module):
    def __init__(self, plan, init_order):
        super().__init__()
        self.plan = plan
        spec = {name: (kind, args) for kind, name, args in plan if name}
        for name in init_order:
            kind, args = spec[name]
            mod = {"conv": CircConv2d, "cb": ConvBlock, "rb": ResBlock}[kind](*args)
            self.add_module(name, mod)

    def forward(self, x):
        for kind, name, _ in self.plan:
            x = _up(x) if kind == "up" else getattr(self, name)(x)
        return x


class AutoEncoder(nn.Module):
    """models/faed/modules.py's AutoEncoder restated: the same parameter names, shapes and initialisation order."""

    def __init__(self):
        super().__init__()
        self.encoder = _Stack(ENC, ENC_INIT)
        self.decoder = _Stack(DEC, DEC_INIT)

    def forward(self, x):
        return torch.tanh(self.decoder(self.encoder(x)))


def init_state(seed: int = 0) -> OrderedDict:
    """The state dict of the reference's `torch.manual_seed(seed); AutoEncoder()` (the global RNG is left as it was)."""
    with torch.random.fork_rng(devices=[]):
        torch.manual_seed(seed)
        return AutoEncoder().state_dict()


# --------------------------------------------------------------------------------------------------------------------
# The trainer
# --------------------------------------------------------------------------------------------------------------------
def _vp(t):
    return C.c_void_p(0 if t is None else t.data_ptr())


class _Conv:
    """One circular convolution: flat-buffer offsets of its weight / bias and its packed fp16 operands."""

    def __init__(self, prefix, cin, cout, k, s, p, off, dev, dgrad):
        self.prefix, self.cin, self.cout, self.k, self.s, self.p = prefix, cin, cout, k, s, p
        self.w_off, self.b_off = off[f"{prefix}.conv2d.weight"], off[f"{prefix}.conv2d.bias"]
        self.x_c = 16 if cin == 3 else cin  # channels of the stored input
        self.dy_c = 16 if cout == 3 else cout  # channels of the stored output gradient
        self.out_c = 4 if cout == 3 else cout  # channels of the stored output
        self.cw = max(cout, 32)
        self.fwd = torch.empty(k * k, self.x_c, self.cw, device=dev, dtype=torch.float16)
        self.dg = torch.empty(k * k, self.dy_c, cin, device=dev, dtype=torch.float16) if dgrad else None


class FAEDTrainer:
    """FAED.training_step + Adam + ExponentialLR on the GPU. `state`: a reference AutoEncoder state dict
    (`encoder.*` / `decoder.*`), a Lightning checkpoint dict or its path; None gives `torch.manual_seed(seed);
    AutoEncoder()`'s initialisation."""

    def __init__(self, state=None, lr: float = 1e-4, lr_decay: float = 0.99, seed: int = 0, device="cuda"):
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise _lib.PFError("FAEDTrainer runs on CUDA devices only")
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.lr0, self.lr, self.lr_decay = float(lr), float(lr), float(lr_decay)
        self.epoch, self.global_step = 0, 0
        ref = AutoEncoder()
        self.param_names = [n for n, _ in ref.named_parameters()]
        self.param_shapes = {n: tuple(p.shape) for n, p in ref.named_parameters()}
        self.bn_names = [n[: -len(".running_mean")] for n, _ in ref.named_buffers() if n.endswith(".running_mean")]
        self.off, o = {}, 0
        for n in self.param_names:
            self.off[n] = o
            o += math.prod(self.param_shapes[n])
        self.n_params = o
        self.bn_off, o = {}, 0
        for n in self.bn_names:
            self.bn_off[n] = o
            o += 2 * self.param_shapes[f"{n}.weight"][0]
        self.n_running = o
        dev = self.device
        f32 = dict(device=dev, dtype=torch.float32)
        self.params = torch.zeros(self.n_params, **f32)
        self.grads = torch.zeros(self.n_params, **f32)
        self.exp_avg = torch.zeros(self.n_params, **f32)
        self.exp_avg_sq = torch.zeros(self.n_params, **f32)
        self.running = torch.zeros(self.n_running, **f32)
        self.pending = torch.zeros(self.n_running, **f32)
        self.num_batches = torch.zeros((), device=dev, dtype=torch.int64)
        self.ctl = torch.tensor([self.lr, INIT_SCALE], device=dev, dtype=torch.float64)  # lr, loss scale
        self.ictl = torch.zeros(4, device=dev, dtype=torch.int32)  # step, growth tracker, skipped, non-finite flag
        self.zero_bias = torch.zeros(128, **f32)
        self.out_bias = torch.zeros(4, **f32)
        self.convs = {}
        for stack, plan in (("encoder", ENC), ("decoder", DEC)):
            for kind, name, args in plan:
                if kind == "conv":
                    self._add_conv(f"{stack}.{name}", *args, dgrad=name != "downconv1_rgb")
                elif kind == "cb":
                    self._add_conv(f"{stack}.{name}.conv1", *args)
                elif kind == "rb":
                    c, k = args
                    self._add_conv(f"{stack}.{name}.conv1", c, c, k, 1, k // 2)
                    self._add_conv(f"{stack}.{name}.conv2", c, c, k, 1, k // 2)
        self._ws = {}
        if state is None:
            state = init_state(seed)
        self.load_state(state)

    def _add_conv(self, prefix, cin, cout, k, s, p, dgrad=True):
        self.convs[prefix] = _Conv(prefix, cin, cout, k, s, p, self.off, self.device, dgrad)

    # ---- views -------------------------------------------------------------------------------------------------------
    def _param(self, name, flat=None):
        flat = self.params if flat is None else flat
        o = self.off[name]
        return flat[o: o + math.prod(self.param_shapes[name])].view(self.param_shapes[name])

    def _bn(self, name):
        c = self.param_shapes[f"{name}.weight"][0]
        o, ob = self.off[f"{name}.weight"], self.off[f"{name}.bias"]
        r = self.bn_off[name]
        return dict(C=c, gamma=self.params[o: o + c], beta=self.params[ob: ob + c], dgamma=self.grads[o: o + c],
                    dbeta=self.grads[ob: ob + c], running=self.running[r: r + 2 * c],
                    pending=self.pending[r: r + 2 * c])

    def _scratch(self, key, n, dtype=torch.float32):
        t = self._ws.get(key)
        if t is None or t.numel() < n:
            t = torch.empty(max(int(n), 1), device=self.device, dtype=dtype)
            self._ws[key] = t
        return t

    def _repack(self, st):
        l = _lib.lib()
        for cv in self.convs.values():
            w = self._param(f"{cv.prefix}.conv2d.weight")
            _lib.check(l.pf_faedt_pack(_vp(w), cv.cout, cv.cin, cv.k, cv.s, _vp(cv.fwd), cv.x_c, cv.cw, _vp(cv.dg),
                                       cv.dy_c, cv.cin, C.c_void_p(st)))
        ob = self.off["decoder.outconv_rgb.conv2d.bias"]
        self.out_bias[:3].copy_(self.params[ob: ob + 3])

    # ---- state -------------------------------------------------------------------------------------------------------
    def load_state(self, state) -> None:
        """Load a reference AutoEncoder state dict, a `net.`-prefixed Lightning state dict, or a checkpoint (dict or
        path; its optimizer, scheduler and loss-scale state too)."""
        ck = None
        if isinstance(state, str):
            state = torch.load(state, map_location="cpu", weights_only=False)
        if "state_dict" in state:
            ck, state = state, state["state_dict"]
        sd = {(k[4:] if k.startswith("net.") else k): v for k, v in state.items()}
        missing = [n for n in self.param_names if n not in sd]
        if missing:
            raise ValueError(f"state dict lacks {missing[:3]}... ({len(missing)} parameters)")
        with torch.no_grad():
            for n in self.param_names:
                self._param(n).copy_(sd[n].reshape(self.param_shapes[n]))
            for n in self.bn_names:
                b = self._bn(n)
                b["running"][: b["C"]].copy_(sd[f"{n}.running_mean"])
                b["running"][b["C"]:].copy_(sd[f"{n}.running_var"])
            self.num_batches.fill_(int(sd[f"{self.bn_names[0]}.num_batches_tracked"]))
            if ck is not None:
                self._load_training_state(ck)
        self._repack(_lib.stream_ptr())

    def _load_training_state(self, ck) -> None:
        self.epoch, self.global_step = int(ck.get("epoch", 0)), int(ck.get("global_step", 0))
        hp = ck.get("hyper_parameters", {})
        self.lr0, self.lr_decay = float(hp.get("lr", self.lr0)), float(hp.get("lr_decay", self.lr_decay))
        step = 0
        if ck.get("optimizer_states"):
            opt = ck["optimizer_states"][0]
            self.lr = float(opt["param_groups"][0]["lr"])
            for i, n in enumerate(self.param_names):
                s = opt["state"].get(i)
                if s is None:
                    continue
                self._param(n, self.exp_avg).copy_(s["exp_avg"])
                self._param(n, self.exp_avg_sq).copy_(s["exp_avg_sq"])
                step = int(s["step"])
        extra = ck.get("faed_train", {})
        self.ctl.copy_(torch.tensor([self.lr, float(extra.get("loss_scale", INIT_SCALE))], dtype=torch.float64))
        self.ictl.copy_(torch.tensor([step, int(extra.get("growth_tracker", 0)), int(extra.get("skipped_steps", 0)),
                                      0], dtype=torch.int32))

    def state_dict(self) -> OrderedDict:
        """The reference FAED LightningModule's state dict: `net.`-prefixed parameters, running statistics and
        num_batches_tracked, on the CPU."""
        nbt = self.num_batches.cpu().clone()
        out = OrderedDict()
        ref = AutoEncoder().state_dict()
        for k in ref:
            if k.endswith(".running_mean") or k.endswith(".running_var"):
                b = self._bn(k.rsplit(".", 1)[0])
                r = b["running"][: b["C"]] if k.endswith("mean") else b["running"][b["C"]:]
                out[f"net.{k}"] = r.detach().cpu().clone()
            elif k.endswith(".num_batches_tracked"):
                out[f"net.{k}"] = nbt.clone()
            else:
                out[f"net.{k}"] = self._param(k).detach().cpu().clone()
        return out

    def optimizer_state_dict(self) -> dict:
        """torch.optim.Adam(lr=lr0)'s state_dict format, with the scheduler's `initial_lr`."""
        step = float(self.ictl[0].item())
        state = {}
        if step > 0:
            for i, n in enumerate(self.param_names):
                state[i] = {"step": torch.tensor(step), "exp_avg": self._param(n, self.exp_avg).cpu().clone(),
                            "exp_avg_sq": self._param(n, self.exp_avg_sq).cpu().clone()}
        group = torch.optim.Adam([torch.zeros(1)], lr=self.lr0).state_dict()["param_groups"][0]
        group.update(lr=self.lr, initial_lr=self.lr0, params=list(range(len(self.param_names))))
        return {"state": state, "param_groups": [group]}

    @property
    def skipped_steps(self) -> int:
        return int(self.ictl[2].item())

    @property
    def loss_scale(self) -> float:
        return float(self.ctl[1].item())

    def save_checkpoint(self, path) -> None:
        """Lightning's checkpoint layout; `faed.load_encoder_state` reads its `net.encoder.` entries."""
        ck = {
            "epoch": self.epoch,
            "global_step": self.global_step,
            "state_dict": self.state_dict(),
            "optimizer_states": [self.optimizer_state_dict()],
            "lr_schedulers": [{"gamma": self.lr_decay, "base_lrs": [self.lr0], "last_epoch": self.epoch,
                               "_step_count": self.epoch + 1, "_is_initial": False,
                               "_get_lr_called_within_step": False, "_last_lr": [self.lr]}],
            "hyper_parameters": {"lr": self.lr0, "lr_decay": self.lr_decay},
            "faed_train": {"loss_scale": self.loss_scale, "growth_tracker": int(self.ictl[1].item()),
                           "skipped_steps": self.skipped_steps},
        }
        torch.save(ck, path)

    def load_checkpoint(self, path) -> None:
        self.load_state(path)

    def on_train_epoch_end(self) -> None:
        """ExponentialLR.step(): lr *= gamma."""
        self.epoch += 1
        self.lr = self.lr * self.lr_decay
        self.ctl[0:1].fill_(self.lr)

    # ---- forward / backward ------------------------------------------------------------------------------------------
    def _conv(self, cv, x, B, H, W, out_dtype=F16):
        ho, wo = (H + 2 * cv.p - cv.k) // cv.s + 1, (W + 2 * cv.p - cv.k) // cv.s + 1
        dt = torch.float32 if out_dtype == F32 else torch.float16
        y = torch.empty(B, ho, wo, cv.out_c, device=self.device, dtype=dt)
        bias = self.out_bias if cv.cout == 3 else self.params[cv.b_off: cv.b_off + cv.cout]
        _lib.check(_lib.lib().pf_faedt_conv(_vp(x), B, H, W, cv.x_c, _vp(cv.fwd), _vp(bias), cv.out_c, cv.cw, cv.k,
                                            cv.k, cv.s, cv.p, cv.p, ho, wo, None, _vp(y), cv.out_c, out_dtype,
                                            C.c_void_p(self._st)))
        return y

    def _dgrad(self, cv, g, B, H, W, residual=None):
        """Gradient of the conv input [B, H, W, cin] from g [B, Ho, Wo, dy_c] (+ residual)."""
        l, st = _lib.lib(), C.c_void_p(self._st)
        ho, wo = g.shape[1], g.shape[2]
        dx = torch.empty(B, H, W, cv.cin, device=self.device, dtype=torch.float16)
        if cv.s == 1:
            _lib.check(l.pf_faedt_conv(_vp(g), B, ho, wo, cv.dy_c, _vp(cv.dg), _vp(self.zero_bias), cv.cin, cv.cin,
                                       cv.k, cv.k, 1, cv.p, cv.p, H, W, _vp(residual), _vp(dx), cv.cin, F16, st))
            return dx
        # stride 2, k 4, pad 1: four 2x2 phase convolutions of g, interleaved
        ph = torch.empty(4, B, ho, wo, cv.cin, device=self.device, dtype=torch.float16)
        for r in range(2):
            for c in range(2):
                i = 2 * r + c
                _lib.check(l.pf_faedt_conv(_vp(g), B, ho, wo, cv.dy_c, _vp(cv.dg[4 * i: 4 * i + 4]),
                                           _vp(self.zero_bias), cv.cin, cv.cin, 2, 2, 1, 1 - r, 1 - c, ho, wo, None,
                                           _vp(ph[i]), cv.cin, F16, st))
        _lib.check(l.pf_faedt_interleave(_vp(ph), B, H, W, cv.cin, _vp(dx), st))
        return dx

    def _wgrad(self, cv, x, g, B, H, W):
        l = _lib.lib()
        ho, wo = g.shape[1], g.shape[2]
        ws = self._scratch("wgrad", l.pf_faedt_wgrad_ws_floats(B, ho, wo, cv.x_c, cv.dy_c, cv.k))
        _lib.check(l.pf_faedt_wgrad(_vp(x), B, H, W, cv.x_c, _vp(g), ho, wo, cv.dy_c, cv.cin, cv.cout, cv.k, cv.s, cv.p,
                                    _vp(ws), _vp(self.ctl[1:]), C.c_double(self._inv_n),
                                    _vp(self.grads[cv.w_off:]), _vp(self.grads[cv.b_off:]), _vp(self.ictl[3:]),
                                    C.c_void_p(self._st)))

    def _bn_fwd(self, name, z, relu, residual, train):
        bn = self._bn(name)
        P, c = z.numel() // bn["C"], bn["C"]
        l, st = _lib.lib(), C.c_void_p(self._st)
        if train:
            stats = torch.empty(3 * c, device=self.device, dtype=torch.float32)
            ws = self._scratch("bn", l.pf_faedt_bn_ws_floats(C.c_longlong(P), c))
            _lib.check(l.pf_faedt_bn_stats(_vp(z), C.c_longlong(P), c, _vp(ws), _vp(stats), _vp(bn["pending"]), st))
        else:  # eval mode: the running statistics
            rm, rv = bn["running"][:c], bn["running"][c:]
            stats = torch.cat([rm, torch.rsqrt(rv + 1e-5), rv])
        out = torch.empty_like(z)
        _lib.check(l.pf_faedt_bn_apply(_vp(z), C.c_longlong(P), c, _vp(stats), _vp(bn["gamma"]), _vp(bn["beta"]),
                                       int(relu), _vp(residual), _vp(out), st))
        return out, stats

    def _bn_bwd(self, name, g, mask, z, stats):
        bn = self._bn(name)
        P, c = z.numel() // bn["C"], bn["C"]
        l = _lib.lib()
        ws = self._scratch("bn", l.pf_faedt_bn_ws_floats(C.c_longlong(P), c))
        dz = torch.empty_like(z)
        _lib.check(l.pf_faedt_bn_bwd(_vp(g), _vp(mask), _vp(z), C.c_longlong(P), c, _vp(stats), _vp(bn["gamma"]),
                                     _vp(ws), _vp(self.ctl[1:]), C.c_double(self._inv_n), _vp(bn["dgamma"]),
                                     _vp(bn["dbeta"]), _vp(self.ictl[3:]), _vp(dz), C.c_void_p(self._st)))
        return dz

    def _forward(self, x, train):
        """Runs AutoEncoder.forward up to outconv (fp32 [B, H, W, 4]); returns it and the saved tape."""
        tape = []
        for stack, plan in (("encoder", ENC), ("decoder", DEC)):
            for kind, name, _ in plan:
                B, H, W = x.shape[0], x.shape[1], x.shape[2]
                pre = f"{stack}.{name}"
                if kind == "up":
                    y = torch.empty(B, 2 * H, 2 * W, x.shape[3], device=self.device, dtype=torch.float16)
                    _lib.check(_lib.lib().pf_faedt_upsample(_vp(x), B, H, W, x.shape[3], _vp(y),
                                                            C.c_void_p(self._st)))
                    tape.append(("up", None, (B, H, W)))
                elif kind == "conv":
                    last = name == "outconv_rgb"
                    y = self._conv(self.convs[pre], x, B, H, W, F32 if last else F16)
                    tape.append(("conv", pre, (x, B, H, W)))
                elif kind == "cb":
                    z = self._conv(self.convs[f"{pre}.conv1"], x, B, H, W)
                    y, s = self._bn_fwd(f"{pre}.batchnorm1", z, True, None, train)
                    tape.append(("cb", pre, (x, B, H, W, z, y, s)))
                else:
                    z1 = self._conv(self.convs[f"{pre}.conv1"], x, B, H, W)
                    a1, s1 = self._bn_fwd(f"{pre}.batchnorm1", z1, True, None, train)
                    z2 = self._conv(self.convs[f"{pre}.conv2"], a1, B, H, W)
                    y, s2 = self._bn_fwd(f"{pre}.batchnorm2", z2, False, x, train)
                    tape.append(("rb", pre, (x, B, H, W, z1, a1, s1, z2, s2)))
                x = y
        return x, tape

    def _backward(self, g, tape):
        for kind, pre, saved in reversed(tape):
            if kind == "up":
                B, H, W = saved
                dx = torch.empty(B, H, W, g.shape[3], device=self.device, dtype=torch.float16)
                _lib.check(_lib.lib().pf_faedt_upsample_bwd(_vp(g), B, H, W, g.shape[3], _vp(dx),
                                                            C.c_void_p(self._st)))
                g = dx
            elif kind == "conv":
                x, B, H, W = saved
                cv = self.convs[pre]
                self._wgrad(cv, x, g, B, H, W)
                g = self._dgrad(cv, g, B, H, W) if cv.dg is not None else None
            elif kind == "cb":
                x, B, H, W, z, y, s = saved
                cv = self.convs[f"{pre}.conv1"]
                gz = self._bn_bwd(f"{pre}.batchnorm1", g, y, z, s)
                self._wgrad(cv, x, gz, B, H, W)
                g = self._dgrad(cv, gz, B, H, W)
            else:
                x, B, H, W, z1, a1, s1, z2, s2 = saved
                c1, c2 = self.convs[f"{pre}.conv1"], self.convs[f"{pre}.conv2"]
                gz2 = self._bn_bwd(f"{pre}.batchnorm2", g, None, z2, s2)
                self._wgrad(c2, a1, gz2, B, H, W)
                ga1 = self._dgrad(c2, gz2, B, H, W)
                gz1 = self._bn_bwd(f"{pre}.batchnorm1", ga1, a1, z1, s1)
                self._wgrad(c1, x, gz1, B, H, W)
                g = self._dgrad(c1, gz1, B, H, W, residual=g)

    @staticmethod
    def _check_pano(pano):
        _lib.require_cuda(pano)
        if pano.dim() == 5 and pano.shape[1] == 1:
            pano = pano[:, 0]
        if pano.dim() != 4 or pano.shape[1] != 3 or pano.dtype != torch.float32:
            raise ValueError(f"expected fp32 panoramas [B, 1, 3, H, W] or [B, 3, H, W], got {tuple(pano.shape)} "
                             f"{pano.dtype}")
        B, _, H, W = pano.shape
        if H % 32 or W % 32 or B * H * W < 2:
            raise ValueError(f"FAED needs H and W that are multiples of 32, got {H}x{W}")
        return pano.contiguous()

    def _prep(self, pano):
        B, _, H, W = pano.shape
        x = torch.empty(B, H, W, 16, device=self.device, dtype=torch.float16)
        _lib.check(_lib.lib().pf_faedt_prep(_vp(pano), B, H, W, _vp(x), C.c_void_p(self._st)))
        return x

    def training_step(self, pano: torch.Tensor) -> torch.Tensor:
        """One FAED.training_step and optimizer step; returns the 0-d fp32 CUDA loss without synchronising."""
        pano = self._check_pano(pano)
        if pano.device != self.device:
            raise ValueError(f"panoramas on {pano.device}, trainer on {self.device}")
        B, _, H, W = pano.shape
        l = _lib.lib()
        with torch.cuda.device(self.device):
            self._st = _lib.stream_ptr()
            st = C.c_void_p(self._st)
            self._inv_n = 1.0 / (3.0 * B * H * W)
            o, tape = self._forward(self._prep(pano), True)
            loss = torch.empty((), device=self.device, dtype=torch.float32)
            seed = torch.empty(B, H, W, 16, device=self.device, dtype=torch.float16)
            ws = self._scratch("loss", l.pf_faedt_loss_ws_floats())
            _lib.check(l.pf_faedt_loss(_vp(o), _vp(pano), B, H, W, _vp(self.ctl[1:]), _vp(ws), _vp(loss), None,
                                       _vp(seed), _vp(self.ictl[3:]), st))
            self._backward(seed, tape)
            _lib.check(l.pf_faedt_adam(_vp(self.params), _vp(self.grads), _vp(self.exp_avg), _vp(self.exp_avg_sq),
                                       C.c_longlong(self.n_params), _vp(self.running), _vp(self.pending),
                                       C.c_longlong(self.n_running), _vp(self.ctl), _vp(self.ictl),
                                       _vp(self.num_batches), C.c_double(BETAS[0]), C.c_double(BETAS[1]),
                                       C.c_double(ADAM_EPS), st))
            self._repack(self._st)
        self.global_step += 1
        return loss

    @torch.no_grad()
    def reconstruct(self, pano: torch.Tensor) -> torch.Tensor:
        """AutoEncoder.forward in eval mode (BatchNorm from the running statistics): fp32 [B, 3, H, W]."""
        pano = self._check_pano(pano)
        B, _, H, W = pano.shape
        l = _lib.lib()
        with torch.cuda.device(self.device):
            self._st = _lib.stream_ptr()
            o, _ = self._forward(self._prep(pano), False)
            pred = torch.empty(B, 3, H, W, device=self.device, dtype=torch.float32)
            ws = self._scratch("loss", l.pf_faedt_loss_ws_floats())
            scratch_loss = torch.empty((), device=self.device, dtype=torch.float32)
            seed = torch.empty(B, H, W, 16, device=self.device, dtype=torch.float16)
            flag = torch.zeros((), device=self.device, dtype=torch.int32)
            _lib.check(l.pf_faedt_loss(_vp(o), None, B, H, W, _vp(self.ctl[1:]), _vp(ws), _vp(scratch_loss),
                                       _vp(pred), _vp(seed), _vp(flag), C.c_void_p(self._st)))
        return pred

    def encoder_state(self) -> dict[str, torch.Tensor]:
        """The encoder's state dict (reference names without `net.encoder.`), as `faed.load_encoder_state` returns."""
        pre = "net.encoder."
        return {k[len(pre):]: v for k, v in self.state_dict().items() if k.startswith(pre)}
