"""GPU: FAED autoencoder training (panfusion_b200.faed_train on csrc/faed_train.cu) against the fp64 restatement
`faed_train.AutoEncoder` (identical to the reference's models/faed/modules.py, checked on the CPU in
tests/test_faed_train.py) run by torch autograd, and Adam against torch.optim.Adam. The panoramas are rounded to fp16
first, so both sides see the same input operand."""
import math

import pytest
import torch

from panfusion_b200 import faed, faed_train as ft

pytestmark = pytest.mark.gpu


def _pano(B, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    x = (torch.rand(B, 3, H, W, generator=g) * 2 - 1).half().float()
    # smooth content, as a real panorama has, plus noise
    yy, xx = torch.meshgrid(torch.linspace(0, 3, H), torch.linspace(0, 2 * math.pi, W), indexing="ij")
    x = (0.6 * torch.sin(xx + yy)[None, None] + 0.4 * x).clamp(-1, 1).half().float()
    return x


def _ref_step(net, pano):
    net.zero_grad(set_to_none=True)
    loss = (net(pano) - pano).abs().mean()
    loss.backward()
    return loss


def _is_prebn_bias(name):
    return name.endswith("conv2d.bias") and "batchnorm" not in name and (".conv1." in name or ".conv2." in name)


def _grad_errors(tr, net):
    out = {}
    for n, p in net.named_parameters():
        g = tr._param(n, tr.grads).double()
        r = p.grad
        if _is_prebn_bias(n):  # mathematically zero: both sides return rounding noise of sum(dz)
            out[n] = ("abs", (g - r).abs().max().item())
        else:
            out[n] = ("rel", ((g - r).norm() / r.norm().clamp_min(1e-300)).item())
    return out


@pytest.mark.parametrize("B,H,W", [(2, 64, 128), (2, 64, 96), (4, 512, 1024)])
def test_one_step_gradients_match_fp64(B, H, W, cuda_device):
    sd = ft.init_state(0)
    tr = ft.FAEDTrainer(sd, device=cuda_device)
    net = ft.AutoEncoder().to(cuda_device).double()
    net.load_state_dict(sd)
    net.train()
    pano = _pano(B, H, W, 1).to(cuda_device)
    loss = tr.training_step(pano)
    # the reference's own precision: fp32 with TF32 convolutions (cuDNN's default), same weights and input
    n32 = ft.AutoEncoder().to(cuda_device)
    n32.load_state_dict(sd)
    n32.train()
    _ref_step(n32, pano)
    g32 = {n: p.grad for n, p in n32.named_parameters()}
    ref = _ref_step(net, pano.double())
    lerr = abs(loss.item() - ref.item()) / ref.item()
    errs = _grad_errors(tr, net)
    rel32 = {n: ((g32[n].double() - p.grad).norm() / p.grad.norm()).item() for n, p in net.named_parameters()}
    worst_rel = max(v for k, v in errs.values() if k == "rel")
    worst_abs = max(v for k, v in errs.values() if k == "abs")
    worst_ratio = max(v / max(rel32[n], 1e-3) for n, (k, v) in errs.items() if k == "rel")
    print(f"\n{B}x{H}x{W}: loss rel err {lerr:.2e}, worst grad rel Frobenius {worst_rel:.2e} "
          f"(fp32/TF32 eager: {max(rel32.values()):.2e}), worst ours/TF32 {worst_ratio:.2f}, "
          f"worst pre-BN bias abs {worst_abs:.2e}")
    for n, (k, v) in errs.items():
        print(f"  {n}: {k} {v:.2e} tf32 {rel32[n]:.2e}")
    # measured on an H100: loss 9.0e-4, worst parameter 0.28 (<= 2.9x the fp32/TF32 eager error of the same
    # parameter), pre-BN biases 5.1e-4 absolute; at 512x1024 B = 4: 8.0e-5, 0.18 (2.0x), 2.3e-4
    assert lerr < 2e-3
    assert worst_rel < 0.55, errs
    assert worst_ratio < 6.0, errs
    assert worst_abs < 1e-3
    # running statistics (momentum 0.1, unbiased var) against the fp64 module's
    sd_mine = tr.state_dict()
    rs = net.state_dict()
    run_err = max(((sd_mine[f"net.{k}"].double() - rs[k].cpu()).abs().max() /
                   rs[k].abs().max()).item() for k in rs if "running" in k)
    print(f"  running stats max rel err {run_err:.2e}")
    assert run_err < 1e-2  # measured 4.0e-3
    assert all(int(sd_mine[f"net.{k}"]) == 1 for k in rs if k.endswith("num_batches_tracked"))


def test_adam_matches_torch(cuda_device):
    sd = ft.init_state(3)
    tr = ft.FAEDTrainer(sd, device=cuda_device)
    p0 = tr.params.clone()
    pano = _pano(2, 32, 64, 2).to(cuda_device)
    ps, opt = None, None
    for step in range(3):
        before = tr.params.clone()
        tr.training_step(pano)
        g = tr.grads.clone()
        if ps is None:
            ps = torch.nn.Parameter(p0.clone())
            opt = torch.optim.Adam([ps], lr=1e-4, foreach=False)
        ps.data.copy_(before)  # same starting point each step; moments carried by the optimizer
        ps.grad = g
        opt.step()
        # in ulps of the larger operand of the update (a result near zero after cancellation has tiny ulps)
        ref_mag = torch.maximum(before.abs(), ps.data.abs()).clamp_min(1e-30)
        ulp = (tr.params - ps.data).abs() / torch.finfo(torch.float32).eps / ref_mag
        diff = (tr.params != ps.data).sum().item()
        print(f"\nstep {step + 1}: {diff} of {ps.numel()} params differ, max {ulp.max().item():.2f} ulp")
        assert diff == 0, ulp.max().item()  # pf_faedt_adam rounds as torch's single-tensor Adam does
    st = opt.state[ps]
    assert torch.equal(tr.exp_avg, st["exp_avg"]) or (tr.exp_avg - st["exp_avg"]).abs().max() <= \
        1.2e-7 * st["exp_avg"].abs().max()


def test_trajectory_matches_fp64(cuda_device):
    sd = ft.init_state(0)
    tr = ft.FAEDTrainer(sd, device=cuda_device)
    net = ft.AutoEncoder().to(cuda_device).double()
    net.load_state_dict(sd)
    net.train()
    n32 = ft.AutoEncoder().to(cuda_device)
    n32.load_state_dict(sd)
    n32.train()
    opt = torch.optim.Adam(net.parameters(), lr=1e-4)
    opt32 = torch.optim.Adam(n32.parameters(), lr=1e-4)
    worst, worst32 = 0.0, 0.0
    for i in range(5):
        pano = _pano(2, 64, 128, 10 + i).to(cuda_device)
        loss = tr.training_step(pano).item()
        ref = _ref_step(net, pano.double()).item()
        l32 = _ref_step(n32, pano).item()
        opt.step()
        opt32.step()
        worst = max(worst, abs(loss - ref) / ref)
        worst32 = max(worst32, abs(l32 - ref) / ref)
        print(f"\nstep {i}: loss {loss:.6f} fp64 {ref:.6f} fp32/TF32 {l32:.6f}")
    print(f"worst loss rel err over 5 steps {worst:.2e} (fp32/TF32 eager {worst32:.2e})")
    # measured on an H100: 0.16, fp32/TF32 eager 0.08 (near-zero gradients flip Adam's +-lr step either way)
    assert worst < 0.32
    assert tr.skipped_steps == 0


def test_repeat_and_resume_are_bit_identical(cuda_device, tmp_path):
    panos = [_pano(2, 32, 64, 20 + i).to(cuda_device) for i in range(4)]
    a = ft.FAEDTrainer(seed=5, device=cuda_device)
    b = ft.FAEDTrainer(seed=5, device=cuda_device)
    la = [a.training_step(p) for p in panos]
    lb = [b.training_step(p) for p in panos[:2]]
    b.on_train_epoch_end()
    b.save_checkpoint(tmp_path / "r.ckpt")
    c = ft.FAEDTrainer(str(tmp_path / "r.ckpt"), device=cuda_device)
    a2 = ft.FAEDTrainer(seed=5, device=cuda_device)
    for p in panos[:2]:
        a2.training_step(p)
    a2.on_train_epoch_end()
    lc = lb + [c.training_step(p) for p in panos[2:]]
    la2 = [a2.training_step(p) for p in panos[2:]]
    assert all(torch.equal(x, y) for x, y in zip(la[:2], lc[:2]))
    assert torch.equal(a2.params, c.params) and torch.equal(a2.exp_avg_sq, c.exp_avg_sq)
    assert torch.equal(a2.running, c.running) and all(torch.equal(x, y) for x, y in zip(la2, lc[2:]))
    assert c.epoch == 1 and c.global_step == 4 and c.lr == pytest.approx(1e-4 * 0.99)


def test_nonfinite_input_is_skipped(cuda_device):
    tr = ft.FAEDTrainer(seed=1, device=cuda_device)
    tr.training_step(_pano(2, 32, 64, 0).to(cuda_device))
    before = [t.clone() for t in (tr.params, tr.exp_avg, tr.exp_avg_sq, tr.running, tr.num_batches)]
    bad = _pano(2, 32, 64, 1)
    bad[0, 1, 5, 7] = float("nan")
    scale = tr.loss_scale
    loss = tr.training_step(bad.to(cuda_device))
    assert not torch.isfinite(loss)
    after = (tr.params, tr.exp_avg, tr.exp_avg_sq, tr.running, tr.num_batches)
    assert all(torch.equal(x, y) for x, y in zip(before, after))
    assert tr.skipped_steps == 1 and tr.loss_scale == scale / 2 and int(tr.ictl[0]) == 1
    assert torch.isfinite(tr.training_step(_pano(2, 32, 64, 2).to(cuda_device)))
    assert int(tr.ictl[0]) == 2 and tr.skipped_steps == 1


def test_checkpoint_feeds_the_faed_metric(cuda_device, tmp_path):
    tr = ft.FAEDTrainer(seed=2, device=cuda_device)
    for i in range(2):
        tr.training_step(_pano(2, 64, 128, 30 + i).to(cuda_device))
    path = tmp_path / "faed.ckpt"
    tr.save_checkpoint(path)
    metric = faed.FrechetAutoEncoderDistance(64, ckpt_path=str(path), device=cuda_device)
    direct = faed.FAEDEncoder(tr.encoder_state(), cuda_device)
    imgs = (torch.rand(3, 3, 64, 128, generator=torch.Generator().manual_seed(4)) * 255).to(torch.uint8)
    imgs = imgs.to(cuda_device)
    assert torch.equal(metric.encoder(imgs), direct(imgs))
    ck = torch.load(path, weights_only=False)
    assert set(ck) >= {"state_dict", "optimizer_states", "lr_schedulers", "epoch", "global_step",
                       "hyper_parameters"}
    assert list(ck["state_dict"]) == [f"net.{k}" for k in ft.init_state(0)]


def test_reconstruct_matches_fp64_eval(cuda_device):
    tr = ft.FAEDTrainer(seed=3, device=cuda_device)
    for i in range(2):
        tr.training_step(_pano(2, 64, 128, 40 + i).to(cuda_device))
    net = ft.AutoEncoder().to(cuda_device).double()
    net.load_state_dict({k[4:]: v for k, v in tr.state_dict().items()})
    net.eval()
    pano = _pano(2, 64, 128, 50).to(cuda_device)
    got = tr.reconstruct(pano)
    with torch.no_grad():
        ref = net(pano.double())
    err = (got.double() - ref).abs().max().item()
    print(f"\nreconstruct max abs err {err:.2e}")
    assert err < 1e-4  # measured 5.0e-5


def test_cli_trains_and_writes_a_metric_checkpoint(cuda_device, tmp_path, capsys):
    import numpy as np
    from PIL import Image

    from panfusion_b200 import train_faed
    for i in range(8):
        Image.fromarray(((_pano(1, 64, 128, 60 + i)[0].permute(1, 2, 0).numpy() + 1) * 127.5).astype(np.uint8)).save(
            tmp_path / f"p{i}.png")
    out = tmp_path / "w" / "faed.ckpt"
    args = ["--images", str(tmp_path / "*.png"), "--pano-height", "32", "--batch-size", "2", "--out", str(out)]
    train_faed.main(args + ["--epochs", "3"])
    train_faed.main(args + ["--epochs", "5", "--resume"])
    lines = [ln for ln in capsys.readouterr().out.splitlines() if ln.startswith("epoch")]
    losses = [float(ln.split("train/loss ")[1].split()[0]) for ln in lines]
    print(losses)
    assert len(losses) == 5 and losses[-1] < losses[0] and "skipped 0" in lines[-1]
    metric = faed.FrechetAutoEncoderDistance(32, ckpt_path=str(out), device=cuda_device)
    assert torch.load(out, weights_only=False)["global_step"] == 20
    assert metric.encoder(torch.zeros(1, 3, 32, 64, dtype=torch.uint8, device=cuda_device)).shape == (1, 128)
