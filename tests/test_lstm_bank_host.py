"""CPU-only tests of LSTM model banks (nam_b200_bank_check_json and the refusals of nam_b200_create_bank_from_json, which
are decided before any CUDA call): which LSTM documents can share one handle."""
import copy

import numpy as np
import pytest

import neuralampmodelercore_b200 as nb
from oracle import nam_config
from tests import nam_fixtures as fx


def _lstm(H=3, nl=1, seed=0, in_ch=1, out_ch=1, sample_rate=48000.0) -> dict:
    config = {"input_size": in_ch, "hidden_size": H, "num_layers": nl}
    if in_ch != 1 or out_ch != 1:
        config.update(in_channels=in_ch, out_channels=out_ch)
    nam = {"version": "0.5.4", "architecture": "LSTM", "sample_rate": sample_rate, "config": config, "weights": []}
    n = nam_config.expected_weight_count(nam)
    nam["weights"] = [float(v) for v in np.random.default_rng(seed).uniform(-0.4, 0.4, n)]
    return nam


def _refused(docs, *fields):
    r = nb.bank_check(docs)
    assert r["ok"] is False, r
    for f in fields:
        assert f in r["reason"], (f, r["reason"])
    return r


@pytest.mark.parametrize("H,nl,in_ch,out_ch", [(3, 1, 1, 1), (16, 2, 1, 1), (70, 1, 1, 1), (5, 2, 2, 3)])
def test_same_shape_lstms_are_accepted_with_distinct_fingerprints(H, nl, in_ch, out_ch):
    docs = [_lstm(H, nl, seed, in_ch, out_ch) for seed in range(4)]
    r = nb.bank_check(docs)
    assert r["ok"] is True and r["reason"] == "" and r["n_models"] == 4, r
    assert len(set(r["fingerprints"])) == 4
    assert r["fingerprints"] == [nb.state_layout(d)["fingerprint"] for d in docs]


def test_the_example_lstm_pairs_with_a_reweighted_copy():
    doc = fx.load_model("lstm")
    other = copy.deepcopy(doc)
    other["weights"] = [float(w) * 1.01 for w in doc["weights"]]
    r = nb.bank_check([doc, other])
    assert r["ok"] is True, r["reason"]
    assert r["fingerprints"][0] != r["fingerprints"][1]


@pytest.mark.parametrize("part", ["h0", "c0", "head"])
def test_models_differing_only_in_initial_state_or_head_are_accepted(part):
    # lstm.nam's layout: W[12][4] (48) | b[12] | h0[3] | c0[3] | head_w[3] | head_b
    a = fx.load_model("lstm")
    b = copy.deepcopy(a)
    lo, hi = {"h0": (60, 63), "c0": (63, 66), "head": (66, 70)}[part]
    for i in range(lo, hi):
        b["weights"][i] = float(b["weights"][i]) + 0.25
    r = nb.bank_check([a, b])
    assert r["ok"] is True, r["reason"]
    assert r["fingerprints"][0] != r["fingerprints"][1]


def test_differing_hidden_size_is_refused():
    _refused([_lstm(3, 1, 0), _lstm(3, 1, 1), _lstm(4, 1, 2)], "model 2", "hidden_size")


def test_differing_num_layers_is_refused():
    _refused([_lstm(8, 2, 0), _lstm(8, 1, 1)], "model 1", "num_layers")


def test_differing_channels_are_refused():
    _refused([_lstm(5, 2, 0, 2, 3), _lstm(5, 2, 1, 2, 2)], "model 1", "out_channels")
    _refused([_lstm(5, 2, 0, 2, 3), _lstm(5, 2, 1, 1, 3)], "model 1", "in_channels")


def test_differing_sample_rate_is_refused():
    _refused([_lstm(3, 1, 0), _lstm(3, 1, 1, sample_rate=44100.0)], "model 1", "sample_rate")


def test_a_mismatch_is_a_model_error_before_touching_a_device():
    with pytest.raises(RuntimeError, match="model 1 differs from model 0 in hidden_size"):
        nb.get_dsp_bank([_lstm(3, 1, 0), _lstm(5, 1, 1)], batch=4)


def test_a_model_an_ordinary_handle_refuses_is_refused_with_its_reason():
    bad = _lstm(3, 1, 1)
    bad["config"]["input_size"] = 2  # in_channels stays 1
    bad["weights"] = [0.1] * nam_config.expected_weight_count(bad)
    r = nb.bank_check([_lstm(3, 1, 0), bad])
    assert r["ok"] is False and r["reason"] == "model 1: LSTM input_size (2) != in_channels (1)", r
    with pytest.raises(nb.UnsupportedModelError, match=r"model 1: LSTM input_size \(2\) != in_channels \(1\)"):
        nb.get_dsp_bank([_lstm(3, 1, 0), bad], batch=4)


def test_both_mixed_family_orders_are_refused():
    a1 = fx.random_wavenet(seed=0)
    with pytest.raises(nb.UnsupportedModelError, match="model 1: architecture LSTM"):
        nb.get_dsp_bank([a1, _lstm()], batch=4)
    with pytest.raises(nb.UnsupportedModelError, match="model 1: architecture WaveNet"):
        nb.get_dsp_bank([_lstm(), a1], batch=4)
    _refused([_lstm(), a1], "model 1", "model 0", "architecture")


def test_other_architectures_after_an_lstm_are_refused():
    linear = {"version": "0.5.4", "architecture": "Linear", "sample_rate": 48000.0,
              "config": {"receptive_field": 4, "bias": True}, "weights": [0.1] * 5}
    _refused([_lstm(), linear], "model 1", "architecture Linear")
    _refused([_lstm(), fx.make_container([(0.5, _lstm(seed=1)), (1.0, _lstm(seed=2))])], "model 1", "architecture")


def test_create_refuses_required_jit_with_the_reason():
    with pytest.raises(nb.UnsupportedModelError, match="jit = 1"):
        nb.get_dsp_bank([_lstm(seed=0), _lstm(seed=1)], batch=4, jit=1)


def test_create_refuses_the_general_kernel_geometry():
    with pytest.raises(nb.UnsupportedModelError, match="kernel_geometry 4"):
        nb.get_dsp_bank([_lstm(seed=0), _lstm(seed=1)], batch=4, kernel_geometry=4)
