"""-m gpu: MVDiffusion's denoiser (panfusion_b200.mvdiffusion) — the three CPAttn kernels one by one, one CPAttn and the
whole step (tiny and SD-2 width), the sampler loop and the panorama stitching against the goldens minted by executing
the reference's own files (oracle/mvdiffusion.py).

The whole-step gates are PanFusion's (tests/test_gpu_mvgen.py): fp16 max 4e-3 / mean 5e-4, bf16 2.5e-2 / 4e-3 of
max|ref|; the single-block gates compare the residual update alone, like test_gpu_mvgen's WarpAttn test.
"""
from pathlib import Path

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
GOLD = Path(__file__).parent / "golden"
LIMITS = {torch.float16: (4e-3, 5e-4), torch.bfloat16: (2.5e-2, 4e-3)}
UPDATE_LIMITS = {torch.float16: (1.5e-2, 1e-3), torch.bfloat16: (1e-1, 6e-3)}


def _check(name, got, ref, dtype, limits):
    scale = ref.abs().max().item()
    d = (got.float().cpu() - ref).abs()
    mx, mean = d.max().item() / scale, d.mean().item() / scale
    lim = limits[dtype]
    print(f"[parity] {name} {dtype}: max {mx:.3e} mean {mean:.3e} (of max|ref|) limits {lim}")
    assert mx <= lim[0] and mean <= lim[1], (name, mx, mean)


def _tables(dev, h, img):
    from oracle import mvdiffusion as omv
    from panfusion_b200 import ops
    from panfusion_b200.mvdiffusion import homographies
    K, R = omv.horizon_cameras(8)
    hl, hr = homographies(K, R)
    return ops.cpattn_tables(hl.to(dev).contiguous(), hr.to(dev).contiguous(), h, h, img)


@pytest.mark.parametrize("level", [8, 64])
def test_tables_match_reference_golden(cuda_device, level):
    from oracle import mvdiffusion as omv
    img = dict(omv.TABLE_LEVELS)[level]
    g = np.load(GOLD / "mvdiff_tables.npz")
    pos, mask = _tables(cuda_device, level, img)
    sel = omv._table_rows(level)
    keep = lambda t: t[0].reshape(8, level, level, *t.shape[3:])[:, sel, sel].cpu()
    pos, mask = keep(pos), keep(mask)
    gp, gm, gr = (torch.from_numpy(g[f"{k}_{level}"]) for k in ("pos", "mask", "rel"))
    assert (pos[..., :2] - gp).abs().max() <= 1e-4
    # masks exact, except where the golden's rescaled coordinate lies within 1e-3 px of a bound
    s = img // level
    sc = (gp + 0.5) * s
    near = ((sc.abs() < 1e-3) | ((sc - img).abs() < 1e-3)).any(-1)
    assert torch.equal(mask.bool()[~near], gm.bool()[~near])
    exact = (pos[..., 2:] == gr).float().mean().item()
    print(f"[tables {level}^2] xy_rel bit-identical fraction {exact:.5f}, in-image keys {gm.float().mean():.3f}")
    assert (pos[..., 2:] - gr).abs().max() <= 1e-4
    # key PE of the kernel's arguments against the golden's, for every in-image key (what the gather adds)
    freq = (2.0 ** torch.arange(80, dtype=torch.float32)).to(cuda_device)
    pe = lambda r: torch.cat([torch.sin(r[..., :, None] * freq), torch.cos(r[..., :, None] * freq)], -2).flatten(-2)
    live = gm.bool().to(cuda_device)
    d = (pe(pos[..., 2:].to(cuda_device)) - pe(gr.to(cuda_device)))[live]
    assert d.abs().max().item() <= 2e-6


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_gather_matches_grid_sample_restatement(cuda_device, dtype):
    from oracle import mvdiffusion as omv
    from panfusion_b200 import ops
    from panfusion_b200.mvdiffusion import _PosEmbedding
    B, m, C, h, img = 2, 8, 320, 16, 512
    x = torch.randn(B, m, C, h, h, generator=torch.Generator().manual_seed(3)).to(dtype).float()
    freq = _PosEmbedding(C // 4).freq_bands
    K, R = omv.horizon_cameras(m, batch=B)
    pos, mask, rel = omv.tables(K, R, h, img)
    want = omv.gather_keys(x, pos, mask, rel, freq).reshape(-1, C)
    tp, tm = _tables(cuda_device, h, img)
    tok = x.permute(0, 1, 3, 4, 2).reshape(-1, C).to(cuda_device, dtype).contiguous()
    keys, st = ops.cpattn_gather(tok, B, m, h, h, tp, tm, freq.reshape(-1).to(cuda_device).contiguous())
    torch.testing.assert_close(keys.float().cpu(), want, rtol=1e-2 if dtype == torch.bfloat16 else 2e-3, atol=2e-3)
    kf = keys.float()
    torch.testing.assert_close(st[:, 0, 0], kf.sum(1), rtol=1e-4, atol=1e-3)
    torch.testing.assert_close(st[:, 0, 1], (kf * kf).sum(1), rtol=1e-4, atol=1e-3)
    assert (st[:, 1] == 0).all()
    assert (keys.float().abs().sum(1) == 0).any() and (keys.float().abs().sum(1) > 0).any()


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_attention_matches_softmax_restatement(cuda_device, dtype):
    from panfusion_b200 import ops
    T, C = 1000, 320
    g = torch.Generator().manual_seed(5)
    q = torch.randn(T, C, generator=g).to(cuda_device, dtype)
    kv = torch.randn(T * 18, 2 * C, generator=g).to(cuda_device, dtype)
    out = ops.cpattn_attn(q, kv, torch.empty(T, C, dtype=dtype, device=cuda_device), 32 ** -0.5)
    qh = q.float().reshape(T, 1, 10, 32).transpose(1, 2)
    k = kv[:, :C].float().reshape(T, 18, 10, 32).transpose(1, 2)
    v = kv[:, C:].float().reshape(T, 18, 10, 32).transpose(1, 2)
    ref = (torch.softmax(qh @ k.transpose(-1, -2) * 32 ** -0.5, -1) @ v).transpose(1, 2).reshape(T, C)
    tol = 1e-3 if dtype == torch.float16 else 1e-2
    torch.testing.assert_close(out.float(), ref, rtol=tol, atol=tol)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_cpattn_matches_reference_golden(cuda_device, dtype):
    from oracle import mvdiffusion as omv
    from panfusion_b200.mvdiffusion import CPAttn
    orc, x, K, R = omv.cpattn_case(omv.CPAttn)
    mine = CPAttn(320, flag360=True)
    mine.load_state_dict(orc.state_dict())
    gold = torch.from_numpy(np.load(GOLD / "mvdiff_cpattn.npz")["out"])
    y = mine.to(cuda_device)(x.to(cuda_device), None, 512, 512, R, K, 8, compute_dtype=dtype)
    _check("CPAttn(320) update", y.float().cpu() - x, gold - x, dtype, UPDATE_LIMITS)


def _tiny(cuda_device, dtype):
    from oracle import mvdiffusion as omv, unet as ou
    from panfusion_b200.mvdiffusion import MultiViewBaseModel
    orc = omv.build_model(omv.MultiViewBaseModel, ou.TINY_CONFIG)
    mine = MultiViewBaseModel(orc.unet, compute_dtype=dtype)
    mine.load_state_dict(orc.state_dict())
    mine.prepare(cuda_device, dtype)
    inp = omv.step_inputs_cfg(8, 16, ou.TINY_CONFIG["cross_attention_dim"])
    cu = dict(inp, latents=inp["latents"].to(cuda_device), timestep=inp["timestep"].to(cuda_device),
              prompt_embd=inp["prompt_embd"].to(cuda_device))
    return orc, mine, inp, cu


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_tiny_step_matches_reference_golden(cuda_device, dtype):
    _, mine, _, cu = _tiny(cuda_device, dtype)
    s = mine(**cu)
    _check("MVDiffusion tiny step", s, torch.from_numpy(np.load(GOLD / "mvdiff_tiny.npz")["sample"]), dtype, LIMITS)


def test_step_is_deterministic_and_graph_replay_is_bit_exact(cuda_device):
    _, mine, _, cu = _tiny(cuda_device, torch.float16)
    a = mine(**cu).clone()
    b = mine(**cu).clone()
    assert torch.equal(a, b)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        with torch.cuda.graph(g, stream=side):
            out = mine(**cu)
    torch.cuda.current_stream().wait_stream(side)
    out.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, a)


def test_single_view_skips_the_cp_blocks(cuda_device, monkeypatch):
    """m = 1: MVGenModel.py:82,105,142 run no CP block; the step equals the oracle's plain UNet walk."""
    from panfusion_b200.mvdiffusion import CPAttn
    orc, mine, inp, cu = _tiny(cuda_device, torch.float16)

    def boom(*a, **k):
        raise AssertionError("CP block called with one view")

    monkeypatch.setattr(CPAttn, "forward_tokens", boom)
    one = dict(latents=inp["latents"][:, :1], timestep=inp["timestep"][:, :1], prompt_embd=inp["prompt_embd"][:, :1],
               meta={k: v[:, :1] for k, v in inp["meta"].items()})
    with torch.no_grad():
        ref = orc(**one)
    s = mine(**dict(one, latents=one["latents"].to(cuda_device), timestep=one["timestep"].to(cuda_device),
                    prompt_embd=one["prompt_embd"].to(cuda_device)))
    _check("MVDiffusion m=1 step", s, ref, torch.float16, LIMITS)


def test_mp2e_matches_reference_golden(cuda_device):
    """pf_mp2e against the executed mp2e.py (golden): within one level, fraction of differing pixels reported."""
    from oracle import mvdiffusion as omv
    from panfusion_b200 import ops
    imgs, fov, theta, phi = omv.mp2e_inputs()
    got = ops.mp2e(torch.from_numpy(imgs).to(cuda_device), fov, theta, phi, omv.MP2E_CASE["out_hw"]).cpu()
    gold = torch.from_numpy(np.load(GOLD / "mvdiff_mp2e.npz")["pano"])
    d = (got.int() - gold.int()).abs()
    print(f"[mp2e] max |diff| {d.max().item()} levels, differing pixels {(d > 0).float().mean().item():.5f}")
    assert got.shape == gold.shape and d.max().item() <= 1


def test_five_sampler_steps_match_oracle_loop(cuda_device):
    """MvDiffusionSampler (CFG pair, DDIM-50 schedule, one captured graph) for its first five steps vs the oracle's
    restatement of MvDiffusion.inference's loop on the same initial latents."""
    from oracle import mvdiffusion as omv, unet as ou
    from panfusion_b200.mvdiffusion import MvDiffusionSampler
    orc, mine, inp, _ = _tiny(cuda_device, torch.float16)
    lat0 = torch.randn(1, 8, 4, 16, 16, generator=torch.Generator().manual_seed(21))
    K, R = inp["meta"]["K"][:1], inp["meta"]["R"][:1]
    with torch.no_grad():
        ref = omv.sample_loop(orc, lat0, inp["prompt_embd"], K, R, num_steps=5)
    smp = MvDiffusionSampler(mine)
    got = smp.denoise(lat0.to(cuda_device), inp["prompt_embd"].to(cuda_device), K, R, num_steps=5)
    assert len(smp._graphs) == 1 and all(getattr(g, "_pf_tables", None) for g in smp._graphs.values())
    _check("MVDiffusion 5 sampler steps", got, ref, torch.float16, LIMITS)
    # a second image of the same shapes replays the same graph on the new inputs
    again = smp.denoise(lat0.to(cuda_device), inp["prompt_embd"].to(cuda_device), K, R, num_steps=5)
    assert torch.equal(again, got) and len(smp._graphs) == 1


def test_sd2_width_step_matches_reference_golden(cuda_device):
    """The default configuration's denoiser: SD-2 widths, 8 horizon views of 64^2 latents, CFG pair."""
    from oracle import mvdiffusion as omv, unet as ou
    from panfusion_b200.mvdiffusion import MultiViewBaseModel
    orc = omv.build_model(omv.MultiViewBaseModel, ou.SD2_CONFIG)
    for dtype in (torch.float16, torch.bfloat16):
        mine = MultiViewBaseModel(orc.unet, compute_dtype=dtype)
        mine.load_state_dict(orc.state_dict())
        mine.prepare(cuda_device, dtype)
        inp = omv.step_inputs_cfg(8, 64, ou.SD2_CONFIG["cross_attention_dim"])
        s = mine(**dict(inp, latents=inp["latents"].to(cuda_device), timestep=inp["timestep"].to(cuda_device),
                        prompt_embd=inp["prompt_embd"].to(cuda_device)))
        _check("MVDiffusion SD-2 8-view CFG step", s, torch.from_numpy(np.load(GOLD / "mvdiff_c2.npz")["sample"]), dtype,
               LIMITS)
        del mine, s
        torch.cuda.empty_cache()


def test_graph_holds_tables_after_eviction(cuda_device):
    """A captured step co-owns the camera tables it reads: evicting them from the LRU cache frees nothing it uses."""
    from panfusion_b200.mvdiffusion import MvDiffusionSampler
    _, mine, inp, _ = _tiny(cuda_device, torch.float16)
    lat0 = torch.randn(1, 8, 4, 16, 16, generator=torch.Generator().manual_seed(22))
    K, R = inp["meta"]["K"][:1], inp["meta"]["R"][:1]
    smp = MvDiffusionSampler(mine)
    a = smp.denoise(lat0.to(cuda_device), inp["prompt_embd"].to(cuda_device), K, R, num_steps=2)
    tables = mine.cp_blocks_mid.tables
    held = [t.data_ptr() for g in smp._graphs.values() for t in g._pf_tables]
    tables.clear()
    assert held and not tables.tensors_of(mine.last_camera_key)
    torch.cuda.empty_cache()
    b = smp.denoise(lat0.to(cuda_device), inp["prompt_embd"].to(cuda_device), K, R, num_steps=2)
    assert torch.equal(a, b)
