"""-m gpu: the drop-in modules (WarpAttn, MultiViewBaseModel) through the full CUDA path against
(a) the committed goldens minted by executing the reference's own files (oracle/make_golden.py) and
(b) the CPU oracle on the same seeded inputs.

Tolerances. The north star asks rtol 1e-3 / atol 1e-4 "fp16"; that bar is met per kernel (tests/test_gpu_gemm.py,
test_gpu_fmha.py, test_gpu_kernels.py, test_gpu_resample.py compare each kernel with an fp32 reference on
16-bit-rounded inputs). End to end the activations are ROUNDED TO 16 BIT between ~400 kernels, which the fp32
reference never does, so the whole-model comparison is bounded by accumulated storage rounding instead. The gates
are set at about TWICE the measured values (DESIGN.md "Parity" lists them), relative to max|ref|, so a 2x regression
of the end-to-end agreement fails. Measured on an H100:
fp16 (11-bit significand)  : max |err| <= 4e-3,   mean |err| <= 5e-4    (measured 1.2e-3 .. 1.8e-3 / 2.9e-4)
bf16 ( 8-bit significand)  : max |err| <= 2.5e-2, mean |err| <= 4e-3    (measured 8.9e-3 .. 1.3e-2 / 2.3e-3)
"""
import functools
from pathlib import Path

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
GOLD = Path(__file__).parent / "golden"


LIMITS = {torch.float16: (4e-3, 5e-4), torch.bfloat16: (2.5e-2, 4e-3)}


@functools.lru_cache(maxsize=2)
def _oracle_model(config_name: str):
    """The seeded oracle model (weights only are used on the GPU side); SD-2 size takes ~1 min of host RNG: shared."""
    from oracle import mvgen as om, synth, unet as ou
    return synth.build_model(om.MultiViewBaseModel, getattr(ou, config_name), seed=0)


def _err(got, ref):
    scale = ref.abs().max().item()
    d = (got - ref).abs()
    return d.max().item() / scale, d.mean().item() / scale


# the EPPA test compares the residual UPDATE alone (a few per cent of the activations' magnitude), so its relative error is
# larger than that of whole-model outputs: measured fp16 7.4e-3 / 4.0e-4, bf16 5.1e-2 / 2.8e-3 -> gates at 2x
UPDATE_LIMITS = {torch.float16: (1.5e-2, 1e-3), torch.bfloat16: (1e-1, 6e-3)}


def _check(name, got, ref, dtype, limits=None):
    mx, mean = _err(got.float().cpu(), ref)
    lim = (limits or LIMITS)[dtype]
    print(f"[parity] {name} {dtype}: max {mx:.3e} mean {mean:.3e} (of max|ref|) limits {lim}")
    assert mx <= lim[0] and mean <= lim[1], (name, mx, mean)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_warpattn_vs_reference_golden(cuda_device, dtype):
    """WarpAttn(320) on 2 batches x 2 views, 8x8 / 8x16 — golden = reference modules.py:8-59 output."""
    from oracle import eppa as oe, synth
    from panfusion_b200.eppa import WarpAttn
    torch.manual_seed(7)
    worc = oe.WarpAttn(320).eval()
    holder = torch.nn.Module()
    holder.cp_blocks = worc
    synth.randomize_zero_init(holder, 11)
    mine = WarpAttn(320).eval()
    mine.load_state_dict(worc.state_dict())
    g = torch.Generator().manual_seed(8)
    px, ex = torch.randn(4, 320, 8, 8, generator=g), torch.randn(2, 320, 8, 16, generator=g)
    c4 = dict(FoV=torch.full((4,), 90.0), theta=torch.tensor([0.0, 180.0, 0.0, 180.0]), phi=torch.zeros(4))
    gold = np.load(GOLD / "warpattn_320.npz")
    with torch.no_grad():
        op, oq = worc(px, ex, c4)
    # the oracle reproduces the reference golden (pins the oracle on this box too)
    torch.testing.assert_close(op, torch.from_numpy(gold["pers_out"]), rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(oq, torch.from_numpy(gold["equi_out"]), rtol=1e-5, atol=1e-5)
    gp, ge = mine.to(cuda_device)(px.to(cuda_device), ex.to(cuda_device), c4, compute_dtype=dtype)
    # the block is residual: compare the UPDATE it adds, which is what the kernels compute
    _check("WarpAttn pers update", gp.float().cpu() - px, torch.from_numpy(gold["pers_out"]) - px, dtype, UPDATE_LIMITS)
    _check("WarpAttn equi update", ge.float().cpu() - ex, torch.from_numpy(gold["equi_out"]) - ex, dtype, UPDATE_LIMITS)


def _build_mine(cuda_device, config, dtype):
    from oracle import unet as ou
    from panfusion_b200.mvgen import MultiViewBaseModel
    orc = _oracle_model("SD2_CONFIG" if config is ou.SD2_CONFIG else "TINY_CONFIG")
    mine = MultiViewBaseModel(orc.unet, orc.pano_unet, compute_dtype=dtype)
    mine.load_state_dict(orc.state_dict())
    mine.prepare(cuda_device, dtype)
    return orc, mine


def _run_mvgen(cuda_device, config, pano_hw, pers_hw, dtype):
    from oracle import synth
    orc, mine = _build_mine(cuda_device, config, dtype)
    inp = synth.step_inputs(2, pano_hw, pers_hw, config["cross_attention_dim"], seed=0)
    cu = {k: (v.to(cuda_device) if torch.is_tensor(v) else {kk: vv.to(cuda_device) for kk, vv in v.items()})
          for k, v in inp.items()}
    s, p = mine(**cu)
    torch.cuda.synchronize()
    return orc, inp, s, p


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_mvgen_tiny_vs_golden_and_oracle(cuda_device, dtype):
    from oracle import unet as ou
    orc, inp, s, p = _run_mvgen(cuda_device, ou.TINY_CONFIG, (16, 32), (16, 16), dtype)
    gold = np.load(GOLD / "mvgen_tiny.npz")
    with torch.no_grad():
        os_, op_ = orc(**inp)
    torch.testing.assert_close(os_, torch.from_numpy(gold["sample"]), rtol=1e-4, atol=1e-4)
    assert s.shape == os_.shape and p.shape == op_.shape
    _check("MultiViewBaseModel tiny sample", s, torch.from_numpy(gold["sample"]), dtype)
    _check("MultiViewBaseModel tiny pano", p, torch.from_numpy(gold["pano_sample"]), dtype)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_mvgen_c1_vs_reference_golden(cuda_device, dtype):
    """BASELINE config 1 (SD-2-size UNets, 1 pano 64x128 + 2 views 64x64): golden = the reference's own
    MultiViewBaseModel.forward executed on CPU in the build container."""
    from oracle import unet as ou
    _, _, s, p = _run_mvgen(cuda_device, ou.SD2_CONFIG, (64, 128), (64, 64), dtype)
    gold = np.load(GOLD / "mvgen_c1.npz")
    _check("MultiViewBaseModel C1 sample", s, torch.from_numpy(gold["sample"]), dtype)
    _check("MultiViewBaseModel C1 pano", p, torch.from_numpy(gold["pano_sample"]), dtype)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_mvgen_c2_vs_reference_golden(cuda_device, dtype):
    """BASELINE configs[1] — the BENCHMARKED configuration (SD-2 widths, 8 horizon views 64x64 + pano 64x128, the CFG
    pair b = 2 with prompts [null; text]): golden = the reference's own MultiViewBaseModel.forward (MVGenModel.py:38-297)
    executed on CPU in the build container (oracle/make_golden.py --only c2). Then the SAME step through the sharded
    code path: every rank of the 2x1 (N = 2) and 2x4 (N = 8) layouts runs on this GPU in turn (tests/_rank_replay.py) and
    the assembled result must equal the unsharded one."""
    from oracle import synth, unet as ou
    from _rank_replay import run_all_ranks, run_unsharded_recording
    cfg = ou.SD2_CONFIG
    _, mine = _build_mine(cuda_device, cfg, dtype)
    inp = _to_dev(synth.step_inputs_cfg(8, (64, 128), (64, 64), cfg["cross_attention_dim"], seed=0), cuda_device)
    from panfusion_b200 import ops
    (s, p), rec = run_unsharded_recording(mine, inp)
    torch.cuda.synchronize()
    gold = np.load(GOLD / "mvgen_c2.npz")
    _check("MultiViewBaseModel C2 sample", s, torch.from_numpy(gold["sample"]), dtype)
    _check("MultiViewBaseModel C2 pano", p, torch.from_numpy(gold["pano_sample"]), dtype)
    # CFG halves see different prompts: they must differ (a broken batch index would make them equal)
    assert (s[0] - s[1]).abs().max().item() > 1e-3
    assert len(rec) == 7
    # (1) default kernels: split-K partitions a few skinny convolutions by the rank's (smaller) M, so the sharded step
    # differs from the unsharded one by fp32 summation order only. 16-bit storage amplifies such a perturbation to the same
    # size as the deviation from the fp32 reference (measured fp16 1.4e-3, bf16 1.0e-2 of max): gated at the parity limit
    scale = s.abs().max().item()
    for layout in ((2, 1), (2, 4)):
        ss, sp, worst = run_all_ranks(mine, inp, *layout, rec)
        ds, dp = (ss - s).abs().max().item() / scale, (sp - p).abs().max().item() / scale
        print(f"[parity] C2 {dtype} layout {layout[0]}x{layout[1]} (split-K on): |sharded - unsharded| sample {ds:.3e} "
              f"pano {dp:.3e} of max, local K|V vs unsharded {worst:.3e}")
        assert ds <= LIMITS[dtype][0] and dp <= LIMITS[dtype][0]
    # (2) with the M-dependent K partition off, every kernel's arithmetic is independent of the batch size: EXACT equality
    keep = ops.SPLIT_K
    ops.SPLIT_K = False
    try:
        (s0, p0), rec0 = run_unsharded_recording(mine, inp)
        for layout in ((2, 1), (2, 4)):
            ss, sp, worst = run_all_ranks(mine, inp, *layout, rec0)
            ds, dp = (ss - s0).abs().max().item(), (sp - p0).abs().max().item()
            print(f"[parity] C2 {dtype} layout {layout[0]}x{layout[1]} (split-K off): |sharded - unsharded| sample {ds:.3e} "
                  f"pano {dp:.3e}, local K|V vs unsharded {worst:.3e}")
            assert ds == 0.0 and dp == 0.0 and worst == 0.0
    finally:
        ops.SPLIT_K = keep


def _build_cn_pair(cuda_device, config, dtype, pers):
    from oracle import mvgen as om, synth
    from panfusion_b200.mvgen import MultiViewBaseModel
    orc = synth.build_model_cn(om.MultiViewBaseModel, config, seed=0, pers=pers)
    mine = MultiViewBaseModel(orc.unet, orc.pano_unet, pers_cn=orc.pers_cn, pano_cn=orc.pano_cn, compute_dtype=dtype)
    mine.load_state_dict(orc.state_dict())
    mine.prepare(cuda_device, dtype)
    return orc, mine


def _to_dev(inp, dev):
    return {k: (v.to(dev) if torch.is_tensor(v) else {kk: vv.to(dev) for kk, vv in v.items()}) for k, v in inp.items()}


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("tag,pers", [("tiny_cn", False), ("tiny_cn2", True)])
def test_mvgen_controlnet_vs_reference_golden(cuda_device, dtype, tag, pers):
    """BASELINE config 5 (layout-conditioned): golden = the reference's MVGenModel.py executed around the ControlNet
    restatement; checks the conditioned output AND the ControlNet's own contribution (conditioned - unconditioned),
    which a wrong residual wiring / zero-conv / conditioning embedding would change."""
    from oracle import synth, unet as ou
    cfg = ou.TINY_CONFIG
    orc, mine = _build_cn_pair(cuda_device, cfg, dtype, pers)
    inp = synth.step_inputs(2, (16, 32), (16, 16), cfg["cross_attention_dim"], seed=0)
    inp.update(synth.layout_conds(1, 2, (16, 32), (16, 16), seed=5, pers=pers))
    gold = np.load(GOLD / f"mvgen_{tag}.npz")
    base = np.load(GOLD / "mvgen_tiny.npz")
    cu = _to_dev(inp, cuda_device)
    s, p = mine(**cu)
    s2, p2 = mine(**cu)  # second call: cached conditioning features
    s0, p0 = mine(**{**cu, "pano_layout_cond": None, "pers_layout_cond": None})
    torch.cuda.synchronize()
    assert torch.equal(s, s2) and torch.equal(p, p2)
    _check(f"MultiViewBaseModel {tag} sample", s, torch.from_numpy(gold["sample"]), dtype)
    _check(f"MultiViewBaseModel {tag} pano", p, torch.from_numpy(gold["pano_sample"]), dtype)
    _check(f"MultiViewBaseModel {tag} no-cond pano", p0, torch.from_numpy(base["pano_sample"]), dtype)
    # the ControlNet's contribution itself, relative to ITS magnitude
    dref = torch.from_numpy(gold["pano_sample"] - base["pano_sample"])
    dgot = (p - p0).float().cpu()
    mx = (dgot - dref).abs().max().item() / dref.abs().max().item()
    print(f"[parity] {tag} {dtype}: ControlNet contribution err {mx:.3e} of its max {dref.abs().max().item():.3e}")
    assert mx < (0.05 if dtype == torch.float16 else 0.25)
    # changing the condition image must change the output (cache is keyed on identity + version)
    cu["pano_layout_cond"].mul_(0.5)
    _, p3 = mine(**cu)
    assert (p3 - p).abs().max().item() > 1e-3


def test_controlnet_pano_only_branch(cuda_device):
    """unet=None with a panorama ControlNet (PanoOnly ablation + layout condition), timestep [b]."""
    from oracle import controlnet as ocn, mvgen as om, unet as ou
    from panfusion_b200.mvgen import MultiViewBaseModel
    cfg = ou.TINY_CONFIG
    pano_unet = ou.build_unet(cfg, seed=2)
    cn = ocn.build_controlnet(ou.build_unet(cfg, seed=3), seed=4)
    orc = om.MultiViewBaseModel(None, pano_unet, pano_cn=cn).eval()
    mine = MultiViewBaseModel(None, pano_unet, pano_cn=cn, compute_dtype=torch.float16)
    g = torch.Generator().manual_seed(0)
    pano = torch.randn(2, 1, 4, 16, 32, generator=g)
    text = torch.randn(2, 1, 77, cfg["cross_attention_dim"], generator=g)
    cond = torch.rand(2, 1, 3, 128, 256, generator=g)
    t = torch.tensor([981, 501])
    with torch.no_grad():
        _, ref = orc(None, pano, t, None, text, None, None, cond)
    s, got = mine(None, pano.to(cuda_device), t.to(cuda_device), None, text.to(cuda_device), None, None,
                  cond.to(cuda_device))
    assert s is None
    _check("pano-only + ControlNet", got, ref, torch.float16)


def test_mvgen_icosahedron_20_views(cuda_device):
    """BASELINE config 4's camera rig (utils/pano.py:34-71: 20 icosahedron face centres, phi != 0) at CPU-checkable
    size: 20 views 16x16 + pano 16x32, CFG-style batch of 2, against the oracle."""
    import sys
    sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
    from bench import icosahedron_cameras
    from oracle import mvgen as om, sampler as osamp, synth, unet as ou
    from panfusion_b200.mvgen import MultiViewBaseModel
    cfg, dtype, m = ou.TINY_CONFIG, torch.float16, 20
    orc = synth.build_model(om.MultiViewBaseModel, cfg, seed=0)
    mine = MultiViewBaseModel(orc.unet, orc.pano_unet, compute_dtype=dtype)
    mine.load_state_dict(orc.state_dict())
    theta, phi = icosahedron_cameras()
    assert len(theta) == 20 and abs(abs(phi[0]) - 52.6226) < 1e-3 and abs(abs(phi[5]) - 10.8123) < 1e-3
    cams = dict(FoV=torch.full((2, m), 90.0), theta=torch.tensor(theta, dtype=torch.float32).repeat(2, 1),
                phi=torch.tensor(phi, dtype=torch.float32).repeat(2, 1))
    g = torch.Generator().manual_seed(0)
    pano = torch.randn(2, 1, 4, 16, 32, generator=g)
    lat = osamp.init_noise(pano, 16, 16, cams)
    ts = torch.full((2, m), 501, dtype=torch.long)
    prompt = torch.randn(2, 1, 77, cfg["cross_attention_dim"], generator=g).repeat(1, m, 1, 1)
    inp = dict(latents=lat, pano_latent=pano, timestep=ts, prompt_embd=prompt, pano_prompt_embd=prompt[:, :1].clone(),
               cameras=cams)
    with torch.no_grad():
        rs, rp = orc(**inp)
    s, p = mine(**_to_dev(inp, cuda_device))
    _check("icosahedron-20 sample", s, rs, dtype)
    _check("icosahedron-20 pano", p, rp, dtype)


def test_identity_keyed_caches_survive_address_reuse(cuda_device):
    """The text K/V (and layout-condition) caches are keyed on tensor identity; a NEW prompt tensor that lands on the
    address of a freed one must not hit the stale entry."""
    from oracle import synth, unet as ou
    cfg, dtype = ou.TINY_CONFIG, torch.float16
    orc, mine = _build_cn_pair(cuda_device, cfg, dtype, False)
    inp = synth.step_inputs(2, (16, 32), (16, 16), cfg["cross_attention_dim"], seed=0)
    inp.update(synth.layout_conds(1, 2, (16, 32), (16, 16), seed=5))
    cu = _to_dev(inp, cuda_device)
    mine(**cu)
    g = torch.Generator().manual_seed(77)
    new_prompt = torch.randn(inp["pano_prompt_embd"].shape, generator=g)
    new_cond = torch.rand(inp["pano_layout_cond"].shape, generator=g)
    for _ in range(3):  # free + reallocate same-shaped tensors: the allocator hands the same blocks back
        del cu["pano_prompt_embd"], cu["pano_layout_cond"]
        cu["pano_prompt_embd"], cu["pano_layout_cond"] = new_prompt.to(cuda_device), new_cond.to(cuda_device)
        s, p = mine(**cu)
    mine.prepare(cuda_device, dtype)  # drops every cache
    s_ref, p_ref = mine(**cu)
    assert torch.equal(p, p_ref) and torch.equal(s, s_ref)
