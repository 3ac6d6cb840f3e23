"""CPU (-m "not gpu"): the MVDiffusion oracle against the goldens minted from the reference's own files
(oracle/mvdiffusion.py), the CPAttn C-ABI's argument checks, and the host side of panfusion_b200.mvdiffusion
(parameter names, checkpoint loading, homographies)."""
from pathlib import Path

import numpy as np
import pytest
import torch

GOLD = Path(__file__).parent / "golden"


def test_oracle_tables_match_reference_golden():
    from oracle import mvdiffusion as omv
    g = np.load(GOLD / "mvdiff_tables.npz")
    K, R = omv.horizon_cameras(8)
    assert np.array_equal(K[0].numpy(), g["K"]) and np.array_equal(R[0].numpy(), g["R"])
    for h, img in omv.TABLE_LEVELS:
        pos, mask, rel = omv.tables(K, R, h, img)
        sel = omv._table_rows(h)
        keep = lambda t: t[0].reshape(8, h, h, *t.shape[3:])[:, sel, sel].numpy()
        assert np.array_equal(keep(pos), g[f"pos_{h}"])
        assert np.array_equal(keep(mask).astype(np.uint8), g[f"mask_{h}"])
        assert np.array_equal(keep(rel), g[f"rel_{h}"])  # bit for bit: the PE argument reaches 2^79 x this value
        assert 0 < g[f"mask_{h}"].mean() < 1  # both in-image and out-of-image keys occur


def test_oracle_cpattn_matches_reference_golden():
    from oracle import mvdiffusion as omv
    blk, x, K, R = omv.cpattn_case(omv.CPAttn)
    with torch.no_grad():
        y = blk(x, None, 512, 512, R, K, 8)
    gold = torch.from_numpy(np.load(GOLD / "mvdiff_cpattn.npz")["out"])
    torch.testing.assert_close(y, gold, rtol=1e-3, atol=1e-4)  # golden stored with 10 low significand bits cleared
    assert (gold - x).abs().max() > 1e-2  # the redrawn zero-init projections make the block non-trivial


def test_oracle_tiny_step_matches_reference_golden():
    from oracle import mvdiffusion as omv, unet as ou
    model = omv.build_model(omv.MultiViewBaseModel, ou.TINY_CONFIG)
    inp = omv.step_inputs_cfg(8, 16, ou.TINY_CONFIG["cross_attention_dim"])
    with torch.no_grad():
        s = model(**inp)
    torch.testing.assert_close(s, torch.from_numpy(np.load(GOLD / "mvdiff_tiny.npz")["sample"]), rtol=1e-4, atol=1e-4)


def test_cpattn_abi_rejects_bad_arguments():
    import ctypes as C
    from panfusion_b200 import _lib
    lib = _lib.lib()
    # non-null dummy addresses (16-byte aligned and not): every call below fails its argument check before any launch
    p, odd = C.c_void_p(16), C.c_void_p(8)
    assert lib.pf_cpattn_tables(None, None, 1, 8, 8, 8, 512, None, None, None) == -1
    assert b"null pointer" in lib.pf_last_error()
    assert lib.pf_cpattn_tables(p, p, 1, 1, 8, 8, 512, p, p, None) == -1  # one view has no neighbours
    assert lib.pf_cpattn_tables(p, p, 1, 8, 8, 4, 512, p, p, None) == -1  # non-square level
    assert lib.pf_cpattn_tables(p, p, 1, 8, 8, 8, 500, p, p, None) == -1  # image side not a multiple of the level
    assert lib.pf_cpattn_tables(p, p, 1, 8, 8, 8, 512, odd, p, None) == -1  # misaligned table
    args = lambda **kw: [kw.get(k, v) for k, v in dict(x=p, ldx=320, dt=2, B=2, m=8, h=8, w=8, C=320, G=1, pos=p, mask=p,
                                                        freq=p, keys=p, stats=p, st=None).items()]
    for bad in (dict(dt=0), dict(C=80), dict(ldx=100), dict(G=3), dict(m=1), dict(keys=odd)):
        assert lib.pf_cpattn_gather(*args(**bad)) == -1, bad
    ok = [p, 320, p, 640, p, 320, 2, C.c_longlong(64), 320, C.c_float(0.17), None]
    for i, v in ((1, 100), (3, 320), (6, 0), (8, 80), (0, odd)):
        a = list(ok)
        a[i] = v
        assert lib.pf_cpattn_attn(*a) == -1, (i, v)
    assert lib.pf_mp2e(None, 8, 64, 64, 3, p, 64, 128, p, None) == -1
    assert lib.pf_mp2e(p, 8, 64, 64, 5, p, 64, 128, p, None) == -1  # more than 4 channels
    assert lib.pf_mp2e(p, 0, 64, 64, 3, p, 64, 128, p, None) == -1


def test_oracle_sample_loop_is_mvdiffusion_inference():
    """The oracle loop's first step: CFG combine with guidance 9 and the DDIM update of timestep 981."""
    from oracle import mvdiffusion as omv
    from oracle.sampler import DDIM
    calls = []

    def model(lat, ts, prompt, meta):
        calls.append((lat.shape, ts.tolist(), meta["K"].shape[0]))
        return torch.cat([torch.ones_like(lat[:1]), 2 * torch.ones_like(lat[:1])])

    K, R = omv.horizon_cameras(3)
    lat = torch.zeros(1, 3, 4, 2, 2)
    out = omv.sample_loop(model, lat, torch.zeros(2, 3, 77, 8), K, R, num_steps=1)
    sch = DDIM()
    sch.set_timesteps(50)
    torch.testing.assert_close(out, sch.step(torch.full_like(lat, 10.0), 981, lat))
    assert calls == [((2, 3, 4, 2, 2), [[981] * 3] * 2, 2)]


def _mine_and_oracle():
    from oracle import mvdiffusion as omv, unet as ou
    from panfusion_b200.mvdiffusion import MultiViewBaseModel
    orc = omv.build_model(omv.MultiViewBaseModel, ou.TINY_CONFIG)
    return MultiViewBaseModel(orc.unet), orc


def test_parameter_names_match_reference_layout():
    mine, orc = _mine_and_oracle()
    assert sorted(mine.state_dict()) == sorted(orc.state_dict())
    mine.load_state_dict(orc.state_dict())  # strict
    assert mine.cp_blocks_encoder[0].pe.freq_bands.shape == (1, 1, 16) and mine.cp_blocks_mid.flag360
    assert len(mine.cp_blocks_encoder) == len(mine.cp_blocks_decoder) == 4
    n_cp = sum(p.numel() for b in [*mine.cp_blocks_encoder, mine.cp_blocks_mid, *mine.cp_blocks_decoder]
               for p in b.parameters())
    assert sum(p.numel() for p in mine.trainable_parameters[0][0]) == n_cp
    with pytest.raises(NotImplementedError):
        type(mine)(orc.unet, pers_cn=torch.nn.Identity())


def test_checkpoint_with_lora_loads_into_mvdiffusion():
    from panfusion_b200.checkpoint import load_reference_state_dict
    mine, orc = _mine_and_oracle()
    sd = {"mv_base_model." + k: v.clone() for k, v in orc.state_dict().items()}
    name = "unet.down_blocks.0.attentions.0.transformer_blocks.0.attn1.to_q"
    down, up = torch.randn(4, 64), torch.randn(64, 4)
    sd[f"mv_base_model.{name}.lora_layer.down.weight"] = down
    sd[f"mv_base_model.{name}.lora_layer.up.weight"] = up
    sd["vae.decoder.conv_in.weight"] = torch.zeros(1)
    want = orc.state_dict()[name + ".weight"] + up @ down  # before loading: `mine` shares the oracle's UNet
    rep = load_reference_state_dict(mine, sd)
    assert rep["folded"] == 1 and not rep["missing"] and not rep["unexpected"]
    torch.testing.assert_close(mine.state_dict()[name + ".weight"], want)
    cp = "cp_blocks_decoder.3.transformer.attn1.to_out.weight"
    assert torch.equal(mine.state_dict()[cp], orc.state_dict()[cp])


def test_homographies_match_oracle_bit_for_bit():
    from oracle import mvdiffusion as omv
    from panfusion_b200.mvdiffusion import homographies
    K, R = omv.horizon_cameras(8)
    hl, hr = homographies(K, R)
    for i in range(8):
        for n, j in enumerate(omv._neighbours(i, 8)):
            assert torch.equal(hl[:, i, n], K[:, j] @ torch.inverse(R[:, j]) @ R[:, i] @ torch.inverse(K[:, i]))
            assert torch.equal(hr[:, i, n], K[:, i] @ torch.inverse(R[:, i]) @ R[:, j] @ torch.inverse(K[:, j]))
