"""HorizonNet oracle: a torch restatement of the layout network of models/horizonnet/HorizonNet.py (`net`, i.e.
external/HorizonNet/model.py HorizonNet('resnet50', use_rnn=True)) in fp64, seeded non-degenerate weights, and
`python -m oracle.horizonnet`, which mints tests/golden/horizonnet.npz by executing the reference's own
external/HorizonNet/model.py, loaded by path (build container only; it needs torch, torchvision and numpy).

The golden holds the weight seed and a SHA-256 of the weight bytes (not the weights), the SHA-256 of the three input
images, the reference's fp64 `bon` / `cor`, subsamples of the [B, 1024, 256] LSTM input and of layer 1's LSTM output,
and per-gate statistics of both LSTM layers' pre-activations. Image 2 went through LayoutConsistency's composition
(imgs * 2 - 1, then mask_and_normalize: / 2 + 0.5 and rows [:135], [-135:] zeroed).
"""
from __future__ import annotations

import hashlib
import importlib.util
import math
from pathlib import Path

import numpy as np
import torch
import torch.nn.functional as F

GOLDEN = Path(__file__).resolve().parent.parent / "tests" / "golden" / "horizonnet.npz"
REF_MODEL = Path("/root/reference/external/HorizonNet/model.py")
SEED = 20250
BN_EPS = 1e-5
H, W, T = 512, 1024, 256
MEAN = torch.tensor([0.485, 0.456, 0.406], dtype=torch.float32)
STD = torch.tensor([0.229, 0.224, 0.225], dtype=torch.float32)
ENC = "feature_extractor.encoder."
# torchvision resnet50: (blocks, width, stride of the first block) per layer
LAYERS = [(3, 64, 1), (4, 128, 2), (6, 256, 2), (3, 512, 2)]
SCALE_C = (256, 512, 1024, 2048)  # encoder output channels per scale
BN3_GAMMA = 0.25  # keeps the residual stream of 16 bottlenecks from growing


def encoder_convs():
    """(conv weight key, BN prefix, Cin, Cout, k, stride) of every encoder convolution in forward order; the stem and
    3x3 keys carry wrap_lr_pad's `.1`."""
    out = [(f"{ENC}conv1.1.weight", f"{ENC}bn1", 3, 64, 7, 2)]
    cin = 64
    for li, (n, width, s) in enumerate(LAYERS, 1):
        for j in range(n):
            p = f"{ENC}layer{li}.{j}."
            st = s if j == 0 else 1
            out.append((p + "conv1.weight", p + "bn1", cin, width, 1, 1))
            out.append((p + "conv2.1.weight", p + "bn2", width, width, 3, st))
            out.append((p + "conv3.weight", p + "bn3", width, 4 * width, 1, 1))
            if j == 0:
                out.append((p + "downsample.0.weight", p + "downsample.1", cin, 4 * width, 1, st))
            cin = 4 * width
    return out


def height_convs():
    """(conv prefix, BN prefix, Cin, Cout) of the 4 x 4 ConvCompressH layers (3x3, stride (2, 1), with bias)."""
    out = []
    for s, c in enumerate(SCALE_C):
        chans = [c, c // 2, c // 2, c // 4, c // 8]
        for l in range(4):
            p = f"reduce_height_module.ghc_lst.{s}.layer.{l}.layers."
            out.append((p + "0.1", p + "1", chans[l], chans[l + 1]))
    return out


def lstm_keys(layer: int, reverse: bool) -> dict[str, str]:
    sfx = f"l{layer}" + ("_reverse" if reverse else "")
    return {n: f"bi_rnn.{n}_{sfx}" for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")}


def state_shapes() -> dict[str, tuple]:
    """Every key the network reads (num_batches_tracked excluded) and its shape."""
    want = {}

    def bn(p, c):
        for n in ("weight", "bias", "running_mean", "running_var"):
            want[f"{p}.{n}"] = (c,)

    for wk, bp, ci, co, k, _s in encoder_convs():
        want[wk] = (co, ci, k, k)
        bn(bp, co)
    for cp, bp, ci, co in height_convs():
        want[cp + ".weight"] = (co, ci, 3, 3)
        want[cp + ".bias"] = (co,)
        bn(bp, co)
    for layer in (0, 1):
        for rev in (False, True):
            k = lstm_keys(layer, rev)
            want[k["weight_ih"]] = (2048, 1024)
            want[k["weight_hh"]] = (2048, 512)
            want[k["bias_ih"]] = (2048,)
            want[k["bias_hh"]] = (2048,)
    want["linear.weight"] = (12, 1024)
    want["linear.bias"] = (12,)
    return want


# ---------------------------------------------------------------------------------------------------------------------
# restatement (fp64 unless the input is fp32)
# ---------------------------------------------------------------------------------------------------------------------
def circular_cols(x: torch.Tensor, p: int) -> torch.Tensor:
    """LR_PAD(p): columns -p .. W+p-1 taken modulo W."""
    w = x.shape[-1]
    return x[..., torch.arange(-p, w + p) % w]


def conv(x, w, b, k, stride):
    """wrap_lr_pad's LR_PAD(k // 2) + Conv2d(padding=(k // 2, 0))."""
    p = k // 2
    return F.conv2d(circular_cols(x, p) if p else x, w, b, stride=stride, padding=(p, 0))


def fold_bn(sd, wkey, bp, bkey=None):
    """Conv weight and bias with the eval-mode BatchNorm `bp` folded in, fp64: b' = (b - mu) s + beta."""
    w = sd[wkey].double()
    s = sd[f"{bp}.weight"].double() / torch.sqrt(sd[f"{bp}.running_var"].double() + BN_EPS)
    b = sd[bkey].double() if bkey else torch.zeros(w.shape[0], dtype=torch.float64)
    return w * s[:, None, None, None], (b - sd[f"{bp}.running_mean"].double()) * s + sd[f"{bp}.bias"].double()


def _bn_conv(sd, wkey, bp, x, k, stride, bkey=None, calibrate=False):
    if calibrate:  # running statistics of this BN = the batch's, rounded to fp16 so they regenerate bit-identically
        y = conv(x, sd[wkey].double(), sd[bkey].double() if bkey else None, k, stride)
        sd[f"{bp}.running_mean"] = y.mean((0, 2, 3)).half().float()
        sd[f"{bp}.running_var"] = y.var((0, 2, 3), unbiased=False).clamp_min(1e-4).half().float()
    w, b = fold_bn(sd, wkey, bp, bkey)
    return conv(x, w.to(x.dtype), b.to(x.dtype), k, stride)


def prepare(x: torch.Tensor) -> torch.Tensor:
    """_prepare_x: (x[:, :3] - mean) / std with the fp32 constants."""
    return (x[:, :3] - MEAN.to(x.dtype)[None, :, None, None]) / STD.to(x.dtype)[None, :, None, None]


def encoder(sd, x, calibrate=False):
    specs = encoder_convs()
    y = _bn_conv(sd, *specs[0][:2], x, 7, 2, calibrate=calibrate).relu()
    y = F.max_pool2d(y, 3, 2, 1)
    feats, i = [], 1
    for n, _w, _s in LAYERS:
        for j in range(n):
            c1, c2, c3 = specs[i:i + 3]
            i += 3
            idt = y
            if j == 0:
                ds = specs[i]
                i += 1
                idt = _bn_conv(sd, ds[0], ds[1], y, 1, ds[5], calibrate=calibrate)
            t = _bn_conv(sd, c1[0], c1[1], y, 1, 1, calibrate=calibrate).relu()
            t = _bn_conv(sd, c2[0], c2[1], t, 3, c2[5], calibrate=calibrate).relu()
            y = (_bn_conv(sd, c3[0], c3[1], t, 1, 1, calibrate=calibrate) + idt).relu()
        feats.append(y)
    return feats


def height_tail(x: torch.Tensor, out_w: int) -> torch.Tensor:
    """GlobalHeightConv's tail restated: column t of the result is l0 * xp[x0] + l1 * xp[x0 + 1] of the circularly
    extended xp = x[..., (p - 1) mod w], with src = (t + f + 0.5) / f - 0.5, x0 = floor(src), l1 = src - x0."""
    w = x.shape[-1]
    f = out_w // w
    t = torch.arange(out_w, dtype=torch.float64)
    src = (t + f + 0.5) / f - 0.5
    x0 = src.floor().long()
    l1 = (src - x0).to(x.dtype)
    l0 = 1 - l1
    return l0 * x[..., (x0 - 1) % w] + l1 * x[..., x0 % w]


def height_stage(sd, feats, calibrate=False):
    convs = height_convs()
    outs = []
    for s, y in enumerate(feats):
        for cp, bp, _ci, _co in convs[4 * s:4 * s + 4]:
            y = _bn_conv(sd, cp + ".weight", bp, y, 3, (2, 1), bkey=cp + ".bias", calibrate=calibrate).relu()
        outs.append(height_tail(y, T).reshape(y.shape[0], -1, T))
    return torch.cat(outs, 1)


def lstm_layer(sd, layer, x, pre=None):
    """One bidirectional layer: x [T, B, 1024] -> [T, B, 1024] = [fwd | bwd]; pre (a list) collects the gate
    pre-activations [T, B, 2048] of both directions."""
    outs = []
    for rev in (False, True):
        k = lstm_keys(layer, rev)
        wih, whh = sd[k["weight_ih"]].to(x.dtype), sd[k["weight_hh"]].to(x.dtype)
        b = (sd[k["bias_ih"]].double() + sd[k["bias_hh"]].double()).to(x.dtype)
        xp = x @ wih.T + b
        h = x.new_zeros(x.shape[1], 512)
        c = x.new_zeros(x.shape[1], 512)
        hs = [None] * x.shape[0]
        g_all = [None] * x.shape[0]
        for t in (range(x.shape[0] - 1, -1, -1) if rev else range(x.shape[0])):
            g = xp[t] + h @ whh.T
            g_all[t] = g
            i, f, gg, o = g.split(512, 1)
            c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(gg)
            h = torch.sigmoid(o) * torch.tanh(c)
            hs[t] = h
        outs.append(torch.stack(hs))
        if pre is not None:
            pre.append(torch.stack(g_all))
    return torch.cat(outs, 2)


def head(sd, y):
    """Linear(1024, 12) + view(T, B, 3, 4).permute(1, 2, 0, 3) -> (bon [B, 2, 4T], cor [B, 1, 4T])."""
    o = y @ sd["linear.weight"].to(y.dtype).T + sd["linear.bias"].to(y.dtype)
    o = o.view(o.shape[0], o.shape[1], 3, 4).permute(1, 2, 0, 3).reshape(o.shape[1], 3, -1)
    return o[:, 1:], o[:, :1]


def forward(sd, x: torch.Tensor, inter: dict | None = None):
    """The network on fp32 images [B, C >= 3, 512, 1024], computed in fp64 -> (bon, cor). `inter` (a dict) receives
    the LSTM input `feature` [B, 1024, 256], layer 1's output `lstm1` [T, B, 1024] and the gate pre-activations."""
    x = prepare(x.double())
    feature = height_stage(sd, encoder(sd, x))
    pre = []
    y1 = lstm_layer(sd, 0, feature.permute(2, 0, 1), pre)
    y2 = lstm_layer(sd, 1, y1, pre)
    if inter is not None:
        inter.update(feature=feature, lstm1=y1, pre=pre)
    return head(sd, y2)


# ---------------------------------------------------------------------------------------------------------------------
# seeded weights and inputs
# ---------------------------------------------------------------------------------------------------------------------
def synth_state(seed: int = SEED) -> dict[str, torch.Tensor]:
    """Seeded weights with the reference's state-dict names: He-initialised convolutions, BN running statistics from
    an fp64 calibration pass over one 512 x 1024 noise image (so every BN output is about N(0, 1)), bn3 scaled by 0.25,
    PyTorch's default LSTM / Linear initialisation and the reference's head bias fills."""
    g = torch.Generator().manual_seed(seed)
    sd = {}

    def bn(p, c, gamma=1.0):
        sd[f"{p}.weight"] = gamma * (0.8 + 0.4 * torch.rand(c, generator=g))
        sd[f"{p}.bias"] = 0.1 * torch.randn(c, generator=g)
        sd[f"{p}.running_mean"] = torch.zeros(c)
        sd[f"{p}.running_var"] = torch.ones(c)
        sd[f"{p}.num_batches_tracked"] = torch.tensor(0)

    for wk, bp, ci, co, k, _s in encoder_convs():
        sd[wk] = torch.randn(co, ci, k, k, generator=g) * math.sqrt(2.0 / (ci * k * k))
        bn(bp, co, BN3_GAMMA if bp.endswith("bn3") else 1.0)
    for cp, bp, ci, co in height_convs():
        sd[cp + ".weight"] = torch.randn(co, ci, 3, 3, generator=g) * math.sqrt(2.0 / (ci * 9))
        sd[cp + ".bias"] = 0.1 * torch.randn(co, generator=g)
        bn(bp, co)
    kr = 1.0 / math.sqrt(512)
    for layer in (0, 1):
        for rev in (False, True):
            for name, key in lstm_keys(layer, rev).items():
                shape = {"weight_ih": (2048, 1024), "weight_hh": (2048, 512)}.get(name, (2048,))
                sd[key] = (torch.rand(shape, generator=g) * 2 - 1) * kr
    sd["linear.weight"] = (torch.rand(12, 1024, generator=g) * 2 - 1) / 32
    sd["linear.bias"] = torch.tensor([-1.0] * 4 + [-0.478] * 4 + [0.425] * 4)
    calib = prepare(torch.rand(1, 3, H, W, generator=g)).double()
    with torch.no_grad():
        height_stage(sd, encoder(sd, calib, calibrate=True), calibrate=True)
    return sd


def state_sha256(sd) -> str:
    h = hashlib.sha256()
    for k in sorted(sd):
        h.update(k.encode())
        h.update(sd[k].detach().cpu().contiguous().numpy().tobytes())
    return h.hexdigest()


def images(seed: int = SEED) -> torch.Tensor:
    """Three fp32 [3, 512, 1024] images in [0, 1]: uniform noise, a smooth room-like pattern with noise, and the same
    pattern through LayoutConsistency's composition."""
    g = torch.Generator().manual_seed(seed + 1)
    yy = np.linspace(0, 1, H)[:, None]
    xx = np.linspace(0, 2 * math.pi, W + 1)[:-1][None, :]
    base = np.stack([0.5 + 0.3 * np.sin(3 * xx + c) * np.cos(4 * math.pi * yy) for c in (0.0, 1.0, 2.0)])
    # 8-bit levels computed in fp64: a last-ulp difference of sin / cos between CPUs never changes a level
    base = torch.from_numpy(np.round(base * 255)).float() / 255
    smooth = (base + 0.1 * torch.rand(3, H, W, generator=g)).clamp(0, 1)
    comp = smooth * 2 - 1
    comp = comp / 2 + 0.5
    border = (H - int((85 / 180) * H)) // 2
    comp[..., :border, :] = 0
    comp[..., -border:, :] = 0
    return torch.stack([torch.rand(3, H, W, generator=g), smooth, comp]).contiguous()


def images_sha256(x: torch.Tensor) -> str:
    return hashlib.sha256(x.contiguous().numpy().tobytes()).hexdigest()


# subsampling of the stored intermediates
FEAT_CH, FEAT_T = slice(0, 1024, 4), slice(0, 256, 8)
LSTM_T, LSTM_U = slice(0, 256, 8), slice(0, 1024, 4)


def gate_stats(pre) -> np.ndarray:
    """[layer, direction, gate (i f g o), (mean, std)] of the LSTM gate pre-activations."""
    out = np.zeros((2, 2, 4, 2))
    for n, g in enumerate(pre):
        for q, part in enumerate(g.split(512, 2)):
            out[n // 2, n % 2, q] = (part.mean().item(), part.std().item())
    return out


def mint() -> None:
    """Run the reference's model.py in fp64 on images() and write GOLDEN."""
    spec = importlib.util.spec_from_file_location("hn_reference_model", REF_MODEL)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    sd = synth_state(SEED)
    net = mod.HorizonNet("resnet50", True)
    net.load_state_dict(sd, strict=True)
    net = net.double().eval()
    x = images(SEED)
    got = {}
    net.reduce_height_module.register_forward_hook(lambda m, i, o: got.__setitem__("feature", o))
    with torch.no_grad():
        bon, cor = net(x.double())
        feature = got["feature"]
        pre = []
        y1 = lstm_layer(sd, 0, feature.permute(2, 0, 1), pre)
        lstm_layer(sd, 1, y1, pre)
        # layer 1 through torch's own LSTM, so the stored output is the reference's, not the restatement's
        ref = torch.nn.LSTM(1024, 512, bidirectional=True).double()
        ref.load_state_dict({k: sd[f"bi_rnn.{k}"].double() for k in ref.state_dict()})
        y1_ref, _ = ref(feature.permute(2, 0, 1))
    np.savez_compressed(
        GOLDEN, seed=np.int64(SEED), weights_sha256=np.str_(state_sha256(sd)),
        images_sha256=np.str_(images_sha256(x)), bon=bon.numpy(), cor=cor.numpy(),
        feature_sub=feature[:, FEAT_CH, FEAT_T].float().numpy(),
        lstm1_sub=y1_ref[LSTM_T, :, LSTM_U].float().numpy(), gate_stats=gate_stats(pre))
    print(f"wrote {GOLDEN} ({GOLDEN.stat().st_size} bytes)")


if __name__ == "__main__":
    mint()
