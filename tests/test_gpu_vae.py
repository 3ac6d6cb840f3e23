"""-m gpu: image-space tail of the loop (SURVEY.md §8f rank 1) — VAE decode with circular latent padding and
tensor_to_image through the CUDA path against the oracle (oracle/vae.py: first-party decode_latent / padded panorama
decode / tensor_to_image restated from PanoGenerator.py:272-278, PanFusion.py:166-172, models/modules/utils.py:9-15;
the diffusers decoder itself is a [3P] restatement)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def test_tensor_to_image_bit_exact(cuda_device):
    from oracle import vae as ov
    from panfusion_b200.vae import tensor_to_image
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 3, 3, 20, 36, generator=g) * 0.8
    # exact ties of (x/2+0.5)*255 at k+0.5 exercise round-half-to-even, plus out-of-range values
    ties = (torch.arange(0, 255, dtype=torch.float32) + 0.5) / 255 * 2 - 1
    x.view(-1)[:255] = ties
    x.view(-1)[255:259] = torch.tensor([-1.5, 1.5, -1.0, 1.0])
    ref = ov.tensor_to_image(x)
    got = tensor_to_image(x.to(cuda_device))
    assert got.dtype == np.uint8 and got.shape == ref.shape == (2, 3, 20, 36, 3)
    assert np.array_equal(got, ref)
    u8 = torch.randint(0, 255, (2, 3, 4, 5), dtype=torch.uint8)
    assert np.array_equal(tensor_to_image(u8), ov.tensor_to_image(u8))


def _pair(cuda_device, cfg, dtype):
    from oracle import vae as ov
    from panfusion_b200.vae import VAEDecoder
    orc = ov.build_vae(cfg)
    return orc, VAEDecoder(orc, compute_dtype=dtype).prepare(cuda_device, dtype)


def _cmp(name, got, ref, dtype):
    scale = ref.abs().max().item()
    d = (got.float().cpu() - ref).abs()
    mx, mean = d.max().item() / scale, d.mean().item() / scale
    # 2x the measured worst case (fp16 3.4e-3 / 2.8e-4, bf16 3.0e-2 / 2.2e-3 of max|ref|)
    lim = (7e-3, 6e-4) if dtype == torch.float16 else (6e-2, 4.5e-3)
    print(f"[parity] {name} {dtype}: max {mx:.3e} mean {mean:.3e} (of max|ref|) limits {lim}")
    assert mx <= lim[0] and mean <= lim[1]


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_vae_decode_tiny_vs_oracle(cuda_device, dtype):
    """Narrow decoder: raw decode, decode_latent (2 views) and the circularly padded panorama decode + uint8 images."""
    from oracle import vae as ov
    from panfusion_b200 import vae as pv
    orc, mine = _pair(cuda_device, ov.TINY_VAE_CONFIG, dtype)
    g = torch.Generator().manual_seed(0)
    z = torch.randn(2, 4, 8, 8, generator=g)
    with torch.no_grad():
        ref = orc.decode(z).sample
    _cmp("vae.decode tiny", mine.decode(z.to(cuda_device)), ref, dtype)
    lat = torch.randn(1, 2, 4, 8, 8, generator=g) * 0.18215 * 4
    pano = torch.randn(1, 1, 4, 8, 16, generator=g) * 0.18215 * 4
    with torch.no_grad():
        ref_l, ref_p = ov.decode_latent(lat, orc), ov.decode_pano(pano, orc, 8)
    got_l, got_p = pv.decode_latent(lat.to(cuda_device), mine), pv.decode_pano(pano.to(cuda_device), mine, 8)
    assert got_l.shape == ref_l.shape == (1, 2, 3, 64, 64) and got_p.shape == ref_p.shape == (1, 1, 3, 64, 128)
    _cmp("decode_latent tiny", got_l, ref_l, dtype)
    _cmp("decode_pano tiny", got_p, ref_p, dtype)
    img, ref_img = pv.tensor_to_image(got_p), ov.tensor_to_image(ref_p)
    diff = np.abs(img.astype(np.int32) - ref_img.astype(np.int32))
    print(f"[parity] uint8 panorama {dtype}: max level diff {diff.max()}, mean {diff.mean():.3f}")
    assert diff.mean() < (0.5 if dtype == torch.float16 else 2.5)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_vae_decode_sd2_width_vs_oracle(cuda_device, dtype):
    """SD-2 VAE decoder widths (128/256/512/512, attention head of 512) on small latents: 2 views 8x8 + pano 8x16."""
    from oracle import vae as ov
    from panfusion_b200 import vae as pv
    orc, mine = _pair(cuda_device, ov.SD2_VAE_CONFIG, dtype)
    g = torch.Generator().manual_seed(3)
    lat = torch.randn(1, 2, 4, 8, 8, generator=g) * 0.18215 * 4
    pano = torch.randn(1, 1, 4, 8, 16, generator=g) * 0.18215 * 4
    with torch.no_grad():
        ref_l, ref_p = ov.decode_latent(lat, orc), ov.decode_pano(pano, orc, 8)
    _cmp("decode_latent SD-2 width", pv.decode_latent(lat.to(cuda_device), mine), ref_l, dtype)
    _cmp("decode_pano SD-2 width", pv.decode_pano(pano.to(cuda_device), mine, 8), ref_p, dtype)


def test_vae_rejects_cpu_and_odd_attention_size(cuda_device):
    from oracle import vae as ov
    from panfusion_b200.vae import VAEDecoder
    mine = VAEDecoder(ov.build_vae(ov.TINY_VAE_CONFIG), torch.float16)
    with pytest.raises((ValueError, RuntimeError)):
        mine.decode(torch.zeros(1, 4, 8, 8))
    with pytest.raises(NotImplementedError):
        mine.decode(torch.zeros(1, 4, 6, 6, device=cuda_device))  # 36 tokens: not a multiple of 64


def test_inference_end_to_end_vs_oracle(cuda_device):
    """PanFusion.inference after the text encoder (PanFusion.py:125-172): noise -> 6 denoising steps -> rotate back
    -> decode -> uint8, narrow UNets + narrow VAE, against the same pipeline assembled from the oracle's pieces."""
    from oracle import mvgen as om, sampler as osamp, synth, unet as ou, vae as ov
    from panfusion_b200.mvgen import MultiViewBaseModel
    from panfusion_b200.sampler import PanFusionSampler
    from panfusion_b200.vae import VAEDecoder
    cfg, dtype, m, n = ou.TINY_CONFIG, torch.float16, 4, 6
    orc = synth.build_model(om.MultiViewBaseModel, cfg, seed=0)
    mine = MultiViewBaseModel(orc.unet, orc.pano_unet, compute_dtype=dtype)
    mine.load_state_dict(orc.state_dict())
    ovae = ov.build_vae(ov.TINY_VAE_CONFIG)
    cams = osamp.horizon_cameras(m)
    g = torch.Generator().manual_seed(0)
    pano_noise = torch.randn(1, 1, 4, 16, 32, generator=g)
    text = torch.randn(1, 1, 77, cfg["cross_attention_dim"], generator=g)
    null = torch.randn(1, 1, 77, cfg["cross_attention_dim"], generator=g)
    pano_prompt = torch.cat([null, text])
    prompt = torch.cat([null.repeat(1, m, 1, 1), text.repeat(1, m, 1, 1)])
    with torch.no_grad():
        lat0 = osamp.init_noise(pano_noise, 16, 16, cams)
        rl, rp, _ = osamp.denoise_steps(orc, lat0, pano_noise, prompt, pano_prompt, cams, n)
        rp = torch.roll(rp, int(-n * 90 / 360 * 32), dims=-1)  # PanFusion.py:164
        ref_imgs = ov.tensor_to_image(ov.decode_latent(rl, ovae))
        ref_pano = ov.tensor_to_image(ov.decode_pano(rp, ovae, 8))
    s = PanFusionSampler(mine)
    imgs, pano = s.inference(cams, prompt, pano_prompt, VAEDecoder(ovae, dtype), (16, 32), (16, 16), device=cuda_device,
                             pano_noise=pano_noise, num_steps=n)
    assert imgs.shape == ref_imgs.shape == (1, m, 128, 128, 3) and pano.shape == ref_pano.shape == (1, 1, 128, 256, 3)
    for name, a, b in (("views", imgs, ref_imgs), ("pano", pano, ref_pano)):
        d = np.abs(a.astype(np.int32) - b.astype(np.int32))
        print(f"[parity] inference uint8 {name}: max level diff {d.max()}, mean {d.mean():.3f}")
        assert d.mean() < 1.0 and np.percentile(d, 99) <= 4


# ---- encoder (training step's encode_image, SURVEY.md 8f rank 4 forward half) ---------------------------------------------

def _enc_cmp(name, got, ref, dtype):
    scale = ref.abs().max().item()
    d = (got.float().cpu() - ref).abs()
    mx, mean = d.max().item() / scale, d.mean().item() / scale
    # about 2x the measured worst case over both widths (moments on an H100: fp16 1.81e-3 / 4.33e-4, bf16 2.15e-2 /
    # 3.48e-3 of max|ref|, both from the tiny-width logvar)
    lim = (4e-3, 9e-4) if dtype == torch.float16 else (4.5e-2, 7e-3)
    print(f"[parity] {name} {dtype}: max {mx:.3e} mean {mean:.3e} (of max|ref|) limits {lim}")
    assert mx <= lim[0] and mean <= lim[1]


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("cfg_name", ["TINY_VAE_CONFIG", "SD2_VAE_CONFIG"])
def test_vae_encode_vs_oracle(cuda_device, dtype, cfg_name):
    """VAEEncoder on 64x64 views and a 64x128 panorama (tiny widths and the SD-2 VAE widths): the moments (mean, logvar after
    quant_conv), the sampled + scaled latents of encode_image on the oracle's noise draw, and the circularly padded
    panorama encode (PanoGenerator.py:214-225, PanFusion.py:66-71) against oracle/vae.py."""
    from oracle import vae as ov
    from panfusion_b200 import vae as pv
    orc = ov.build_vae(getattr(ov, cfg_name))
    enc = pv.VAEEncoder(orc, compute_dtype=dtype).prepare(cuda_device, dtype)
    g = torch.Generator().manual_seed(4)
    imgs = torch.rand(1, 2, 3, 64, 64, generator=g) * 2 - 1
    pano = torch.rand(1, 1, 3, 64, 128, generator=g) * 2 - 1
    n_img = torch.randn(2, 4, 8, 8, generator=g)
    n_pano = torch.randn(1, 4, 8, 16 + 2 * 8, generator=g)
    with torch.no_grad():
        dist = orc.encode(imgs[0]).latent_dist
        ref_z = ov.encode_image(imgs, orc, noise=n_img)
        ref_p = ov.encode_pano(pano, orc, 8, noise=n_pano)
    o, N, h, w = enc.moments(imgs[0].to(cuda_device))
    mom = o[:, :8].reshape(N, h, w, 8).permute(0, 3, 1, 2)
    _enc_cmp(f"vae.encode mean {cfg_name}", mom[:, :4], dist.mean, dtype)
    _enc_cmp(f"vae.encode logvar {cfg_name}", mom[:, 4:], dist.logvar, dtype)
    got_z = pv.encode_image(imgs.to(cuda_device), enc, noise=n_img.to(cuda_device)[None])
    got_p = pv.encode_pano(pano.to(cuda_device), enc, 8, noise=n_pano.to(cuda_device)[None])
    assert got_z.shape == ref_z.shape == (1, 2, 4, 8, 8) and got_p.shape == ref_p.shape == (1, 1, 4, 8, 16)
    _enc_cmp(f"encode_image {cfg_name}", got_z, ref_z, dtype)
    _enc_cmp(f"encode_pano {cfg_name}", got_p, ref_p, dtype)
    # the reference's random draw path: runs, right shapes, different generators differ
    from panfusion_b200.training import TrainingStep
    g1 = torch.Generator(device=cuda_device).manual_seed(1)
    lat, plat = TrainingStep.encode(imgs.to(cuda_device), pano.to(cuda_device), enc, 8, generator=g1)
    assert lat.shape == (1, 2, 4, 8, 8) and plat.shape == (1, 1, 4, 8, 16) and torch.isfinite(lat).all()
