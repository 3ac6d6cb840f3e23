"""-m gpu: forward half of the training step (SURVEY.md 8f rank 4; models/pano/PanFusion.py:78-97) — add_noise, the joint
forward and the two MSE terms — against the oracle. The backward is not built and must say so."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def test_add_noise_bit_exact(cuda_device):
    """pf_add_noise == the eager fp32 ops of diffusers' add_noise (sqrt, two products, one sum, each rounded)."""
    from oracle import sampler as osamp, training as otr
    from panfusion_b200 import ops
    g = torch.Generator().manual_seed(0)
    abar = osamp.DDIM().alphas_cumprod
    for shape in [(3, 8, 4, 16, 16), (2, 1, 4, 16, 32), (5, 7)]:
        x0, eps = torch.randn(*shape, generator=g), torch.randn(*shape, generator=g)
        t = torch.randint(0, 1000, (shape[0],), generator=g)
        t[0], t[-1] = 0, 999
        got = ops.add_noise(x0.to(cuda_device), eps.to(cuda_device), t.to(cuda_device), abar.to(cuda_device))
        assert torch.equal(got.cpu(), otr.add_noise(x0, eps, t, abar))


def test_add_noise_rejects_wrong_timestep_count(cuda_device):
    """one timestep per sample is required (an out-of-table timestep traps on the device like torch raises IndexError)."""
    from panfusion_b200 import ops
    x = torch.zeros(1, 4, device=cuda_device)
    with pytest.raises(AssertionError):
        ops.add_noise(x, x, torch.zeros(2, dtype=torch.int64, device=cuda_device), torch.ones(10, device=cuda_device))


@pytest.mark.parametrize("n", [1, 255, 4096, 2 * 8 * 4 * 64 * 64 + 3])
def test_mse_loss_matches_torch_and_is_deterministic(cuda_device, n):
    from panfusion_b200 import ops
    g = torch.Generator().manual_seed(n)
    a, b = torch.randn(n, generator=g), torch.randn(n, generator=g)
    ref = torch.nn.functional.mse_loss(a.double(), b.double()).item()
    got1 = ops.mse_loss(a.to(cuda_device), b.to(cuda_device))
    got2 = ops.mse_loss(a.to(cuda_device), b.to(cuda_device))  # the re-armed counter works, same bits
    assert got1.shape == () and torch.equal(got1, got2)
    assert abs(got1.item() - ref) <= 2e-6 * max(1.0, abs(ref))


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_training_loss_vs_oracle(cuda_device, dtype):
    """TrainingStep.loss on the tiny two-branch model == the oracle's restatement of PanFusion.py:78-97 on the same draws
    (b = 2 samples with different timesteps, 2 views): the shared noise field and the noised latents exactly, the losses to
    1e-4 (fp16) / 3e-4 (bf16) — the forward's 16-bit storage rounding averaged over the outputs."""
    from oracle import synth, training as otr, unet as ou
    from test_gpu_mvgen import _build_mine
    from panfusion_b200.training import TrainingStep
    cfg = ou.TINY_CONFIG
    orc, mine = _build_mine(cuda_device, cfg, dtype)
    inp = synth.step_inputs(2, (16, 32), (16, 16), cfg["cross_attention_dim"], seed=3, batch=2)
    g = torch.Generator().manual_seed(5)
    latents = torch.randn(2, 2, 4, 16, 16, generator=g)
    pano_latent = torch.randn(2, 1, 4, 16, 32, generator=g)
    pano_noise = torch.randn(2, 1, 4, 16, 32, generator=g)
    t = torch.tensor([17, 801])
    ref = otr.training_loss(orc, latents, pano_latent, t, inp["prompt_embd"], inp["pano_prompt_embd"], inp["cameras"], pano_noise)
    step = TrainingStep(mine)
    dev = lambda x: x.to(cuda_device)
    cams = {k: dev(v) for k, v in inp["cameras"].items()}
    # the shared noise field: every view's noise is the nearest-neighbour e2p of the panorama noise (PanFusion.py:30-43)
    from panfusion_b200 import geometry
    c1 = {k: v.flatten(0, 1) for k, v in cams.items()}
    noise = geometry.e2p(dev(pano_noise)[:, 0], c1["FoV"], c1["theta"], c1["phi"], (16, 16), mode="nearest",
                         views_per_image=2).reshape(2, 2, 4, 16, 16)
    assert torch.equal(noise.cpu(), ref["noise"])
    assert torch.equal(step.add_noise(dev(latents), noise, dev(t)).cpu(), ref["noise_z"])
    out = step.loss(dev(latents), dev(pano_latent), dev(inp["prompt_embd"]), dev(inp["pano_prompt_embd"]), cams, t=dev(t),
                    noise=noise, pano_noise=dev(pano_noise))
    torch.cuda.synchronize()
    # measured on an H100: |loss - oracle| <= 5.5e-5 (fp16 and bf16) on losses of 1.1 / 1.1 / 2.2
    lim = {torch.float16: 1e-4, torch.bfloat16: 3e-4}[dtype]
    for k in ("loss_pers", "loss_pano", "loss"):
        got, want = out[k].item(), ref[k].item()
        print(f"[parity] training {k} {dtype}: {got:.6f} vs oracle {want:.6f}")
        assert abs(got - want) <= lim * max(1.0, abs(want)), (k, got, want)
    assert abs(out["loss"].item() - (out["loss_pers"].item() + out["loss_pano"].item())) < 1e-6
    # random draws path: runs, finite, and different draws give a different loss
    g1 = torch.Generator(device=cuda_device).manual_seed(1)
    r1 = step.loss(dev(latents), dev(pano_latent), dev(inp["prompt_embd"]), dev(inp["pano_prompt_embd"]), cams, generator=g1)
    assert torch.isfinite(r1["loss"]) and r1["t"].shape == (2,) and r1["noise"].shape == latents.shape
    with pytest.raises(NotImplementedError):
        step.training_step()
