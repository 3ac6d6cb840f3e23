"""CPU (-m "not gpu"): the HorizonNet oracle restatement (oracle/horizonnet.py) against tests/golden/horizonnet.npz,
which was minted by executing the reference's external/HorizonNet/model.py; the circular addressing, the height
upsampling and the BN folding against torch's own layers; the state loader; the entry points' argument checks; and
that the golden is not degenerate."""
import ctypes as C
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import horizonnet as oh
from panfusion_b200 import horizonnet

GOLD = np.load(Path(__file__).parent / "golden" / "horizonnet.npz")


@pytest.fixture(scope="module")
def sd():
    return oh.synth_state(int(GOLD["seed"]))


def test_golden_inputs_regenerate(sd):
    assert str(GOLD["weights_sha256"]) == oh.state_sha256(sd)
    assert str(GOLD["images_sha256"]) == oh.images_sha256(oh.images(int(GOLD["seed"])))
    assert len(sd) == 448


def test_restatement_matches_golden(sd):
    inter = {}
    with torch.no_grad():
        bon, cor = oh.forward(sd, oh.images(int(GOLD["seed"])), inter)
    for name, got in (("bon", bon), ("cor", cor)):
        ref = GOLD[name]
        assert np.abs(got.numpy() - ref).max() <= 1e-10 * np.abs(ref).max(), name
    for name, got in (("feature_sub", inter["feature"][:, oh.FEAT_CH, oh.FEAT_T]),
                      ("lstm1_sub", inter["lstm1"][oh.LSTM_T, :, oh.LSTM_U])):
        ref = GOLD[name]
        assert np.abs(got.float().numpy() - ref).max() <= 1e-6 * np.abs(ref).max(), name
    np.testing.assert_allclose(oh.gate_stats(inter["pre"]), GOLD["gate_stats"], rtol=1e-9, atol=1e-12)


def test_circular_addressing_is_lr_pad():
    """LR_PAD(p) + Conv2d(padding=(p, 0)): columns wrapped, rows zero-padded, corners zero."""
    x = torch.randn(2, 3, 5, 9, dtype=torch.float64)
    for p in (1, 3):
        wrapped = F.pad(x, (p, p, 0, 0), mode="circular")
        assert torch.equal(oh.circular_cols(x, p), wrapped)
        w = torch.randn(4, 3, 2 * p + 1, 2 * p + 1, dtype=torch.float64)
        ref = F.conv2d(F.pad(wrapped, (0, 0, p, p)), w)
        assert torch.allclose(oh.conv(x, w, None, 2 * p + 1, 1), ref, rtol=0, atol=1e-12)


@pytest.mark.parametrize("h,w", [(8, 256), (4, 128), (2, 64), (1, 32)])
def test_height_tail_bit_equal_in_fp32(h, w):
    """GlobalHeightConv's cat / bilinear (align_corners=False) / crop in fp32, on fp16-valued inputs (the ConvCompressH
    outputs pf_hnet_height_upsample reads): the weights are exact and every product is exact in fp32."""
    g = torch.Generator().manual_seed(w)
    x = torch.randn(2, 5, h, w, generator=g).relu().half().float()
    f = 256 // w
    y = torch.cat([x[..., -1:], x, x[..., :1]], 3)
    ref = F.interpolate(y, size=(h, 256 + 2 * f), mode="bilinear", align_corners=False)[..., f:-f]
    assert torch.equal(oh.height_tail(x, 256), ref)


@pytest.mark.parametrize("name", ["stem", "l2_0_c2", "l3_0_ds", "h1_0"])
def test_bn_folding_matches_eval_layers(sd, name):
    wk, bp, bk, ci, co, k, stride = horizonnet.CONVS[name]
    conv = torch.nn.Conv2d(ci, co, k, stride=stride, padding=(k // 2, 0), bias=bk is not None).double()
    bn = torch.nn.BatchNorm2d(co, eps=horizonnet.BN_EPS).double().eval()
    conv.weight.data = sd[wk].double()
    if bk:
        conv.bias.data = sd[bk].double()
    for p in ("weight", "bias", "running_mean", "running_var"):
        getattr(bn, p).data = sd[f"{bp}.{p}"].double()
    x = torch.randn(1, ci, 12, 16, dtype=torch.float64)
    with torch.no_grad():
        ref = bn(conv(oh.circular_cols(x, k // 2)))
    w, b = horizonnet.fold_bn(sd, name)
    got = oh.conv(x, w, b, k, stride)
    assert (got - ref).abs().max() <= 1e-12 * ref.abs().max()
    w2, b2 = oh.fold_bn(sd, wk, bp, bk)
    assert torch.equal(w, w2) and torch.equal(b, b2)


def test_packing_layouts():
    w = torch.randn(8, 3, 7, 7, dtype=torch.float64)
    p = horizonnet.pack_weight(w, 16)
    assert p.shape == (49, 16, 8) and not p[:, 3:].any()
    assert p[2 * 7 + 5, 1, 6] == w[6, 1, 2, 5].half()
    whh = torch.arange(2048 * 512, dtype=torch.float32).reshape(2048, 512)
    pk = horizonnet.pack_whh(whh)
    assert torch.equal(pk[3, 2 * 32 + 7], whh[2 * 512 + 3 * 32 + 7])


def test_loader_accepts_three_forms(sd, tmp_path):
    want = horizonnet.state_shapes()
    assert set(horizonnet.load_state(sd)) >= set(want)
    ckpt = {"state_dict": {f"net.{k}": v for k, v in sd.items()}, "epoch": 3}
    assert set(horizonnet.load_state(ckpt)) >= set(want)
    torch.save(ckpt, tmp_path / "horizonnet.ckpt")
    got = horizonnet.load_state(str(tmp_path / "horizonnet.ckpt"))
    assert all(torch.equal(got[k], sd[k]) for k in want)

    class Live(torch.nn.Module):
        def state_dict(self, *a, **kw):
            return dict(sd)

    assert set(horizonnet.load_state(Live())) >= set(want)


@pytest.mark.parametrize("key", ["feature_extractor.encoder.layer3.4.conv2.1.weight",
                                 "reduce_height_module.ghc_lst.2.layer.1.layers.0.1.bias",
                                 "bi_rnn.weight_hh_l1_reverse", "linear.bias"])
def test_loader_rejects_missing_or_misshaped_key(sd, key):
    bad = dict(sd)
    del bad[key]
    with pytest.raises(ValueError, match=key.replace(".", r"\.")):
        horizonnet.HorizonNetModule(bad)
    bad[key] = sd[key][..., :1].clone()
    with pytest.raises(ValueError, match="shape"):
        horizonnet.load_state(bad)


def test_entry_points_reject_bad_arguments_without_gpu():
    from panfusion_b200 import _lib
    lib = _lib.lib()
    p = C.c_void_p(16)
    cases = [
        (lambda: lib.pf_hnet_prep(None, 1, 3, 512, 1024, p, None), b"null pointer"),
        (lambda: lib.pf_hnet_prep(p, 1, 3, 256, 512, p, None), b"512 x 1024"),
        (lambda: lib.pf_hnet_conv(p, 1, 8, 8, 64, p, p, 64, 5, 1, 1, 1, None, p, 1, None), b"kernel 5"),
        (lambda: lib.pf_hnet_conv(p, 1, 8, 8, 64, p, p, 64, 3, 1, 2, 1, None, p, 1, None), b"stride (1, 2)"),
        (lambda: lib.pf_hnet_conv(p, 1, 8, 8, 32, p, p, 64, 3, 1, 1, 1, None, p, 1, None), b"Cin=32"),
        (lambda: lib.pf_hnet_conv(p, 1, 8, 8, 64, p, p, 96, 3, 1, 1, 1, None, p, 1, None), b"Cout=96"),
        (lambda: lib.pf_hnet_conv(p, 1, 8, 8, 16, p, p, 128, 7, 2, 2, 1, None, p, 1, None), b"stem"),
        (lambda: lib.pf_hnet_conv(p, 1, 8, 2, 64, p, p, 64, 7, 2, 2, 1, None, p, 1, None), b"too small"),
        (lambda: lib.pf_hnet_conv(p, 1, 8, 8, 64, p, p, 64, 3, 1, 1, 1, None, p, 2, None), b"out_dtype"),
        (lambda: lib.pf_hnet_height_upsample(p, 1, 8, 96, 32, 256, p, 0, None), b"T a multiple of w"),
        (lambda: lib.pf_hnet_height_upsample(p, 1, 8, 256, 32, 256, p, 800, None), b"outside"),
        (lambda: lib.pf_lstm_bidir(p, p, 256, 17, p, None), b"B=17"),
        (lambda: lib.pf_lstm_bidir(p, C.c_void_p(24), 256, 1, p, None), b"16-byte aligned"),
        (lambda: lib.pf_lstm_bidir(None, p, 256, 1, p, None), b"null pointer"),
        (lambda: lib.pf_lstm_bidir_clusters(None), b"null pointer"),
        (lambda: lib.pf_hnet_head(p, 0, 1, p, p, p, p, None), b"bad shape"),
    ]
    for call, msg in cases:
        assert call() == -1 and msg in lib.pf_last_error(), (msg, lib.pf_last_error())


def test_golden_is_not_degenerate():
    cor, bon = GOLD["cor"], GOLD["bon"]
    assert (cor.std(axis=-1) > 0.02).all()  # the corner logits vary along the panorama
    s = 1 / (1 + np.exp(-cor))
    assert ((s > 0.05) & (s < 0.95)).mean() > 0.9  # sigmoid(cor) is not saturated
    assert (bon.std(axis=-1) > 0.01).all()  # both boundaries vary across columns
    std = GOLD["gate_stats"][..., 1]
    assert (std > 0.1).all() and (std < 5).all()  # gate pre-activations are O(1)
    assert GOLD["feature_sub"].std() > 0.1 and GOLD["lstm1_sub"].std() > 0.05
