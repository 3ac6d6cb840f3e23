"""FAED autoencoder training oracle: an fp64 functional restatement of models/faed/modules.py's AutoEncoder in
training mode (Conv2d = CircularPadding + unpadded conv, ResBlock, ConvBlock, BatchNorm2d with batch statistics and
running-statistics updates, bilinear 2x upsampling, tanh), FAED.training_step's L1 loss, its backward (torch
autograd) and torch.optim.Adam's single-tensor update restated op by op.

`python -m oracle.faed_train` mints tests/golden/faed_train.npz by running the reference's own modules.py (loaded
through oracle/ref_loader.py) and torch.optim.Adam in fp64 for STEPS steps at B = 2, 64x128 from
`torch.manual_seed(SEED); AutoEncoder()` on seeded panoramas. It stores digests, not tensors: the init SHA-256 and key
list, the per-step loss, per-parameter gradient sum, norm and a seeded sample of 64 entries, and the running
statistics after each step.
"""
from __future__ import annotations

import hashlib
import importlib
from pathlib import Path

import numpy as np
import torch
import torch.nn.functional as F

GOLDEN = Path(__file__).resolve().parent.parent / "tests" / "golden" / "faed_train.npz"
SEED = 0
STEPS = 3
B, H, W = 2, 64, 128
LR, BETAS, EPS = 1e-4, (0.9, 0.999), 1e-8
N_SAMPLE = 64

# forward plans: ("conv" | "cb" | "rb" | "up", module name, (Cin, Cout, k, stride, pad) or (C, k))
ENCODER = [("conv", "downconv1_rgb", (3, 32, 9, 1, 4)), ("rb", "downres1_rgb", (32, 9)),
           ("cb", "downconv2_rgb", (32, 64, 4, 2, 1)), ("rb", "downres2_rgb", (64, 7)),
           ("cb", "downconv3_rgb", (64, 128, 4, 2, 1)), ("rb", "downres3_rgb", (128, 5)),
           ("cb", "downconv4_rgb", (128, 128, 4, 2, 1)), ("rb", "downres4_rgb", (128, 3)),
           ("cb", "downconv5_rgb", (128, 128, 4, 2, 1)), ("rb", "downres5_rgb", (128, 3)),
           ("cb", "downconv6_rgb", (128, 128, 4, 2, 1)), ("conv", "fuse", (128, 128, 3, 1, 1))]
DECODER = [("up", None, None), ("cb", "upconv2_rgb", (128, 128, 3, 1, 1)), ("rb", "upres2_rgb", (128, 3)),
           ("up", None, None), ("cb", "upconv3_rgb", (128, 128, 3, 1, 1)), ("rb", "upres3_rgb", (128, 5)),
           ("up", None, None), ("cb", "upconv4_rgb", (128, 64, 3, 1, 1)), ("rb", "upres4_rgb", (64, 7)),
           ("up", None, None), ("cb", "upconv5_rgb", (64, 32, 3, 1, 1)), ("rb", "upres5_rgb", (32, 9)),
           ("up", None, None), ("conv", "outconv_rgb", (32, 3, 9, 1, 4))]


def circular_pad(x, p):
    """modules.py CircularPadding: zero pad, then the columns wrap (corners stay zero)."""
    if p == 0:
        return x
    x = F.pad(x, (p, p, p, p), "constant", 0)
    x[:, :, :, 0:p] = x[:, :, :, -2 * p:-p]
    x[:, :, :, -p:] = x[:, :, :, p:2 * p]
    return x


def _conv(sd, pre, x, stride, pad):
    return F.conv2d(circular_pad(x, pad), sd[f"{pre}.conv2d.weight"], sd[f"{pre}.conv2d.bias"], stride)


def _bn(sd, bufs, pre, x):
    """BatchNorm2d training mode, eps 1e-5, momentum 0.1 (updates bufs' running statistics in place)."""
    bufs[f"{pre}.num_batches_tracked"] += 1
    return F.batch_norm(x, bufs[f"{pre}.running_mean"], bufs[f"{pre}.running_var"], sd[f"{pre}.weight"],
                        sd[f"{pre}.bias"], True, 0.1, 1e-5)


def forward(sd, bufs, x):
    """AutoEncoder.forward in training mode; sd holds the parameters, bufs the BatchNorm buffers."""
    for stack, plan in (("encoder", ENCODER), ("decoder", DECODER)):
        for kind, name, args in plan:
            pre = f"{stack}.{name}"
            if kind == "up":
                x = F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=False)
            elif kind == "conv":
                x = _conv(sd, pre, x, args[3], args[4])
            elif kind == "cb":
                x = F.relu(_bn(sd, bufs, f"{pre}.batchnorm1", _conv(sd, f"{pre}.conv1", x, args[3], args[4])))
            else:
                p = args[1] // 2
                out = F.relu(_bn(sd, bufs, f"{pre}.batchnorm1", _conv(sd, f"{pre}.conv1", x, 1, p)))
                out = _bn(sd, bufs, f"{pre}.batchnorm2", _conv(sd, f"{pre}.conv2", out, 1, p))
                out += x
                x = out
    return torch.tanh(x)


def adam_step(params, grads, state, step, lr=LR):
    """torch.optim.Adam's single-tensor update (no weight decay, bias correction), op by op."""
    b1, b2 = BETAS
    for n, p in params.items():
        g = grads[n]
        m, v = state[n]
        m.lerp_(g, 1 - b1)
        v.mul_(b2).addcmul_(g, g, value=1 - b2)
        bc1, bc2 = 1 - b1 ** step, 1 - b2 ** step
        denom = (v.sqrt() / bc2 ** 0.5).add_(EPS)
        p.addcdiv_(m, denom, value=-(lr / bc1))


def panos(step: int) -> torch.Tensor:
    g = torch.Generator().manual_seed(1000 + step)
    return torch.rand(B, 3, H, W, generator=g, dtype=torch.float64) * 2 - 1


def state_sha256(sd) -> str:
    h = hashlib.sha256()
    for k, v in sd.items():
        h.update(k.encode())
        h.update(v.detach().contiguous().numpy().tobytes())
    return h.hexdigest()


def sample_index(name: str, numel: int) -> torch.Tensor:
    g = torch.Generator().manual_seed(int(hashlib.sha256(name.encode()).hexdigest()[:8], 16))
    return torch.randint(0, numel, (N_SAMPLE,), generator=g)


def digests(named_grads, bufs) -> dict:
    out = {}
    for n, g in named_grads:
        g = g.detach().reshape(-1)
        out[f"grad_sum/{n}"] = g.sum().item()
        out[f"grad_norm/{n}"] = g.norm().item()
        out[f"grad_sample/{n}"] = g[sample_index(n, g.numel())].numpy()
    for k, v in bufs.items():
        if "running" in k:
            out[f"{k}"] = v.detach().numpy().copy()
    return out


def init_state(seed: int = SEED) -> dict:
    """`torch.manual_seed(seed); AutoEncoder()`'s state dict without the module: PyTorch's default initialisation
    (kaiming_uniform(a=sqrt(5)) weights, uniform(+-1/sqrt(fan_in)) biases, BN ones / zeros) drawn in modules.py's
    construction order."""
    import math
    init_order = {"encoder": ["downconv1_rgb", "downconv2_rgb", "downconv3_rgb", "downconv4_rgb", "downconv5_rgb",
                              "downconv6_rgb", "downres1_rgb", "downres2_rgb", "downres3_rgb", "downres4_rgb",
                              "downres5_rgb", "fuse"],
                  "decoder": ["upconv2_rgb", "upconv3_rgb", "upconv4_rgb", "upconv5_rgb", "outconv_rgb",
                              "upres2_rgb", "upres3_rgb", "upres4_rgb", "upres5_rgb"]}
    plans = {"encoder": {n: (k, a) for k, n, a in ENCODER if n}, "decoder": {n: (k, a) for k, n, a in DECODER if n}}
    sd = {}

    def conv(pre, ci, co, k):
        w, b = torch.empty(co, ci, k, k), torch.empty(co)
        bound = 1 / math.sqrt(ci * k * k)
        torch.nn.init.kaiming_uniform_(w, a=math.sqrt(5))
        torch.nn.init.uniform_(b, -bound, bound)
        sd[f"{pre}.conv2d.weight"], sd[f"{pre}.conv2d.bias"] = w, b

    def bn(pre, c):
        sd[f"{pre}.weight"], sd[f"{pre}.bias"] = torch.ones(c), torch.zeros(c)
        sd[f"{pre}.running_mean"], sd[f"{pre}.running_var"] = torch.zeros(c), torch.ones(c)
        sd[f"{pre}.num_batches_tracked"] = torch.tensor(0)

    with torch.random.fork_rng(devices=[]):
        torch.manual_seed(seed)
        for stack in ("encoder", "decoder"):
            for name in init_order[stack]:
                kind, a = plans[stack][name]
                pre = f"{stack}.{name}"
                if kind == "conv":
                    conv(pre, a[0], a[1], a[2])
                elif kind == "cb":
                    conv(f"{pre}.conv1", a[0], a[1], a[2])
                    bn(f"{pre}.batchnorm1", a[1])
                else:
                    conv(f"{pre}.conv1", a[0], a[0], a[1])
                    bn(f"{pre}.batchnorm1", a[0])
                    conv(f"{pre}.conv2", a[0], a[0], a[1])
                    bn(f"{pre}.batchnorm2", a[0])
    return sd


def restated_run(sd0: dict, steps: int = STEPS) -> dict:
    """STEPS training steps of the restatement from state dict sd0 -> the golden's keys (losses, gradient digests,
    running statistics)."""
    params = {k: v.detach().double().clone().requires_grad_(True) for k, v in sd0.items()
              if not (k.endswith("running_mean") or k.endswith("running_var") or k.endswith("num_batches_tracked"))}
    bufs = {k: v.detach().clone().double() if v.is_floating_point() else v.detach().clone()
            for k, v in sd0.items() if k not in params}
    state = {n: (torch.zeros_like(p), torch.zeros_like(p)) for n, p in params.items()}
    out = {}
    for s in range(steps):
        x = panos(s)
        pred = forward(params, bufs, x)
        loss = F.l1_loss(pred.unsqueeze(1), x.unsqueeze(1))
        gd = dict(zip(params, torch.autograd.grad(loss, list(params.values()))))
        with torch.no_grad():
            adam_step(params, gd, state, s + 1)
        out[f"step{s}/loss"] = np.float64(loss.item())
        for k, v in digests(gd.items(), {f"step{s}/{k}": v for k, v in bufs.items()}).items():
            out[k if k.startswith("step") else f"step{s}/{k}"] = np.asarray(v)
    return out


def max_rel_error(gold, run) -> tuple[float, str]:
    """Largest |run - gold| over the golden's numeric step entries, relative to the entry's magnitude; gradient
    digests of a parameter are relative to that parameter's gradient norm (a pre-BN bias's true gradient is zero)."""
    worst, where = 0.0, ""
    for k in gold:
        if not k.startswith("step"):
            continue
        g, r = np.asarray(gold[k], dtype=np.float64), np.asarray(run[k], dtype=np.float64)
        if "/grad_" in k:
            s, rest = k.split("/", 1)
            name = rest.split("/", 1)[1]
            w = name.rsplit(".", 1)[0] + ".weight"
            scale = max(float(gold[f"{s}/grad_norm/{name}"]), float(gold.get(f"{s}/grad_norm/{w}", 0.0)))
        else:
            scale = float(np.abs(g).max())
        e = float(np.abs(g - r).max()) / max(scale, 1e-300)
        if e > worst:
            worst, where = e, k
    return worst, where


# ---- minting ------------------------------------------------------------------------------------------------------

def _load_reference():
    from oracle import ref_loader
    ref_loader.load()
    return importlib.import_module("models.faed.modules")


def mint() -> dict:
    mods = _load_reference()
    torch.manual_seed(SEED)
    net = mods.AutoEncoder()
    sd0 = net.state_dict()
    gold = {"seed": np.int64(SEED), "init_sha256": np.array(state_sha256(sd0)), "keys": np.array(list(sd0))}
    net = net.double().train()
    opt = torch.optim.Adam(net.parameters(), lr=LR, foreach=False)
    names = [n for n, _ in net.named_parameters()]
    for s in range(STEPS):
        x = panos(s)
        opt.zero_grad()
        pano_pred = net(x.unsqueeze(1).squeeze(1)).unsqueeze(1)  # FAED.training_step
        loss = F.l1_loss(pano_pred, x.unsqueeze(1))
        loss.backward()
        grads = [(n, p.grad.clone()) for n, p in zip(names, net.parameters())]
        opt.step()
        gold[f"step{s}/loss"] = np.float64(loss.item())
        bufs = {f"step{s}/{k}": v for k, v in net.state_dict().items() if "running" in k}
        for k, v in digests(grads, bufs).items():
            gold[k if k.startswith("step") else f"step{s}/{k}"] = np.asarray(v)
    return gold


if __name__ == "__main__":
    gold = mint()
    np.savez_compressed(GOLDEN, **gold)
    print(GOLDEN, GOLDEN.stat().st_size, "bytes")
    sd0 = init_state()
    assert state_sha256(sd0) == str(gold["init_sha256"]), "restated init differs from the reference's"
    print("restatement vs reference: max rel err %.3e at %s" % max_rel_error(gold, restated_run(sd0)))
