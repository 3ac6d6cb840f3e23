"""CPU (-m "not gpu"): the FAED oracle restatement (oracle/faed.py) against tests/golden/faed.npz, which was minted by
executing the reference's models/faed/modules.py and FAED.py; fp64 BatchNorm folding against eval-mode layers; the
FAED entry points' argument checks."""
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import faed as of

GOLD = np.load(Path(__file__).parent / "golden" / "faed.npz")


def test_golden_inputs_regenerate():
    assert str(GOLD["weights_sha256"]) == of.state_sha256(of.synth_state(int(GOLD["seed"])))
    for tag, case in (("rd", of.RANK_DEFICIENT), ("fr", of.FULL_RANK), ("frl", of.FULL_RANK_LAT)):
        for side in ("real", "fake"):
            assert str(GOLD[f"{tag}_{side}_images_sha256"]) == of.images_sha256(of.set_images(case, side))


def test_restated_features_match_golden():
    sd = of.synth_state(int(GOLD["seed"]))
    with torch.no_grad():
        for i, (h, w) in enumerate(of.FEATURE_SIZES[:2]):
            got = of.features(sd, of.feature_images(i)).numpy()
            ref = GOLD[f"features_{h}"]
            assert np.abs(got - ref).max() <= 1e-5 * np.abs(ref).max(), h
        got = torch.cat([of.features(sd, x) for x in of.set_images(of.RANK_DEFICIENT, "fake")]).numpy()
        ref = GOLD["rd_fake_features"]
        assert np.abs(got - ref).max() <= 1e-5 * np.abs(ref).max()


@pytest.mark.parametrize("tag,case", [("rd", of.RANK_DEFICIENT), ("fr", of.FULL_RANK)])
def test_restated_statistics_and_distance_match_golden(tag, case):
    st = []
    for side in ("real", "fake"):
        f = torch.from_numpy(GOLD[f"{tag}_{side}_features"])
        s, c, n = of.stats(list(f.split(list(case["batches"]))))
        assert n == int(GOLD[f"{tag}_{side}_num_samples"])
        np.testing.assert_allclose(s.numpy(), GOLD[f"{tag}_{side}_sum"], rtol=1e-13, atol=0)
        np.testing.assert_allclose(torch.diagonal(c).numpy(), GOLD[f"{tag}_{side}_cov_sum_diag"], rtol=1e-13, atol=0)
        assert abs(float(c.norm()) - float(GOLD[f"{tag}_{side}_cov_sum_fro"])) <= 1e-13 * float(c.norm())
        st.append((s, c, n))
    tr = sum(float(of.covariances(*x)[1].trace()) for x in st)
    assert abs(of.faed(*st[0], *st[1]) - float(GOLD[f"{tag}_faed"])) <= 1e-9 * tr
    # the symmetric-eigensolver value agrees with the reference's eigvals(S1 S2) to its rounding floor
    assert abs(float(GOLD[f"{tag}_faed_eigh"]) - float(GOLD[f"{tag}_faed"])) <= 1e-7 * tr


def test_bn_folding_matches_eval_mode_layers():
    from panfusion_b200.faed import fold_conv, pack_weight
    sd = of.synth_state(1)
    x = torch.randn(2, 64, 8, 16, dtype=torch.float64)
    name, bn = "downres2_rgb.conv1", "downres2_rgb.batchnorm1"
    ref = of._conv({k: v.double() for k, v in sd.items()}, name, x, 1, 3, bn, torch.float64)
    w, b = fold_conv(sd, name, bn)
    got = torch.nn.functional.conv2d(of.circular_pad(x, 3), w, b)
    assert (got - ref).abs().max() <= 1e-12 * ref.abs().max()
    p = pack_weight(w, 64, torch.float64)
    assert p.shape == (49, 64, 64) and p[2 * 7 + 5, 11, 7] == w[7, 11, 2, 5]
    p = pack_weight(fold_conv(sd, "downconv1_rgb", None)[0], 16, torch.float64)
    assert p.shape == (81, 16, 32) and not p[:, 3:].any()


def test_circular_pad_matches_reference_definition():
    x = torch.arange(2 * 3 * 4 * 6, dtype=torch.float64).reshape(2, 3, 4, 6)
    p = 2
    ref = torch.nn.functional.pad(x, (p, p, p, p))
    ref[..., :p] = ref[..., -2 * p:-p]
    ref[..., -p:] = ref[..., p:2 * p]
    assert torch.equal(of.circular_pad(x, p), ref)


def test_faed_entry_points_reject_bad_arguments():
    from panfusion_b200 import _lib
    l = _lib.lib()
    assert l.pf_faed_prep(None, 1, 1, 3, 32, 32, None, None) == -1
    assert l.pf_conv_circ(1, 1, 8, 8, 32, 1, 1, 32, 11, 1, 5, 0, None, 1, 1, None) == -3
    assert l.pf_conv_circ(1, 1, 8, 8, 48, 1, 1, 32, 3, 1, 1, 0, None, 1, 1, None) == -3
    assert l.pf_conv_circ(1, 1, 8, 8, 32, 1, 1, 32, 3, 1, 1, 0, None, 1, 2, None) == -1  # bf16 output
    assert l.pf_conv_circ(None, 1, 8, 8, 32, 1, 1, 32, 3, 1, 1, 0, None, 1, 1, None) == -1
    assert l.pf_faed_pool(None, 1, 1, 1, 128, None, None, None) == -1
    assert l.pf_faed_stats(1, 0, 128, 1, 1, None) == -1
    import ctypes as C
    assert l.pf_frechet_fp64(1, 1, C.c_longlong(1), 1, 1, C.c_longlong(5), 128, 1, 1, None, None) == -1
    assert b"more than one sample" in l.pf_last_error()
    assert l.pf_frechet_fp64(1, 1, C.c_longlong(5), 1, 1, C.c_longlong(5), 100, 1, 1, None, None) == -1


def test_faed_refuses_cpu_tensors():
    from panfusion_b200 import faed
    with pytest.raises(Exception):
        faed.frechet_distance(*[torch.zeros(128, dtype=torch.float64)] * 2, 3, *[torch.zeros(128, dtype=torch.float64)] * 2, 3)


def test_metric_is_a_module_like_the_reference():
    """EvalPanoGen puts the metric in an nn.ModuleDict, calls requires_grad_(False) and reads _update_called; the
    states are buffers under the reference's names, built on the CPU, and a CPU image is refused."""
    from panfusion_b200 import faed
    d = torch.nn.ModuleDict({"FAED": faed.FrechetAutoEncoderDistance(64, encoder=of.synth_state(1))})
    d.requires_grad_(False)
    m = d["FAED"]
    assert not m._update_called
    bufs = dict(m.named_buffers())
    for side in ("real", "fake"):
        assert bufs[f"{side}_features_sum"].shape == (256,) and bufs[f"{side}_features_sum"].dtype == torch.float64
        assert bufs[f"{side}_features_cov_sum"].shape == (256, 256)
        assert bufs[f"{side}_features_num_samples"].dtype == torch.int64
    assert "encoder.w0" in bufs and m.encoder.w0.dtype == torch.float16
    assert not any(k.startswith(("real_", "fake_", "encoder.")) for k in d.state_dict())  # like torchmetrics' states
    with pytest.raises(Exception):
        m.update(of.images((2, 3, 64, 128), "real", 0), real=True)
    assert not m._update_called
