"""CPU-only tests of model banks (include/nam_b200.h, nam_b200_bank_check_json and the refusals of
nam_b200_create_bank_from_json, which are decided before any CUDA call): which documents can share one handle."""
import copy

import numpy as np
import pytest

import neuralampmodelercore_b200 as nb
from tests import nam_fixtures as fx
from tests.test_reference_build import _convnet


def _a1(seed: int, **kw) -> dict:
    return fx.random_wavenet(seed=seed, **kw)


def _linear(seed: int) -> dict:
    w = np.random.default_rng(seed).uniform(-0.1, 0.1, 33).astype(np.float32)
    return {"version": "0.5.4", "architecture": "Linear", "sample_rate": 48000.0,
            "config": {"receptive_field": 32, "bias": True}, "weights": [float(v) for v in w]}


def _refused(docs, *fields):
    r = nb.bank_check(docs)
    assert r["ok"] is False, r
    for f in fields:
        assert f in r["reason"], (f, r["reason"])
    return r


def test_same_shape_models_are_accepted_with_distinct_fingerprints():
    docs = [_a1(seed) for seed in range(4)]
    r = nb.bank_check(docs)
    assert r["ok"] is True and r["reason"] == "" and r["n_models"] == 4
    assert len(set(r["fingerprints"])) == 4
    # the fingerprint a state record of each model carries
    assert r["fingerprints"] == [nb.state_layout(d)["fingerprint"] for d in docs]


@pytest.mark.parametrize("fixture", ["wavenet", "wavenet_a1_standard", "a2_lite", "a2_full"])
def test_fused_family_fixtures_pair_with_a_reweighted_copy(fixture):
    doc = fx.load_model(fixture)
    other = copy.deepcopy(doc)
    rng = np.random.default_rng(3)
    other["weights"] = [float(w) * float(1.0 + 0.01 * rng.standard_normal()) for w in doc["weights"]]
    r = nb.bank_check([doc, other])
    assert r["ok"] is True, r["reason"]
    assert r["fingerprints"][0] != r["fingerprints"][1]


def test_differing_head_scale_alone_is_accepted():
    a = _a1(0)
    b = copy.deepcopy(a)
    b["weights"][-1] = 0.5  # head_scale is the last weight
    b["config"]["head_scale"] = 0.5  # (the config field is not read)
    assert nb.bank_check([a, b])["ok"] is True


def test_differing_channels_are_refused():
    _refused([_a1(0), _a1(1), _a1(2, channels=(8, 8))], "model 2", "channels")


def test_differing_dilations_are_refused():
    _refused([_a1(0), _a1(1, dilations=[[1, 2, 4, 8], [1, 2, 4, 16]])], "model 1", "dilation")


def test_differing_kernel_sizes_are_refused():
    _refused([_a1(0), _a1(1, kernel_size=2)], "model 1", "kernel_size")


def test_differing_activation_is_refused():
    _refused([_a1(0), _a1(1, activation="ReLU")], "model 1", "activation")


def test_differing_sample_rate_is_refused():
    b = _a1(1)
    b["sample_rate"] = 44100.0
    _refused([_a1(0), b], "model 1", "sample_rate")


@pytest.mark.parametrize("kind", ["lstm", "linear", "convnet", "container", "slimmable_wavenet", "general_kernel"])
def test_models_outside_the_fused_family_are_refused(kind):
    other = {
        "lstm": lambda: fx.load_model("lstm"),
        "linear": lambda: _linear(1),
        "convnet": lambda: _convnet(8, [1, 2, 4], True, "Tanh", 1),
        "container": lambda: fx.make_container([(0.5, _a1(3)), (1.0, _a1(4))]),
        "slimmable_wavenet": lambda: fx.load_model("slimmable_wavenet"),
        "general_kernel": lambda: fx.load_model("wavenet_condition_dsp"),
    }[kind]()
    field = "kernel" if kind == "general_kernel" else "architecture"
    _refused([_a1(0), other], "model 1", field)
    # also as model 0
    _refused([other, _a1(0)], "model 0", field)


def test_no_models_is_refused():
    _refused([], "n_models")
    with pytest.raises(ValueError, match="n_models"):
        nb.get_dsp_bank([], batch=4)


def test_create_refuses_mismatched_documents_before_touching_a_device():
    with pytest.raises(RuntimeError, match="model 1 differs from model 0 in array 0 layer 1 dilation"):
        nb.get_dsp_bank([_a1(0), _a1(1, dilations=[[1, 4, 4, 8], [1, 2, 4, 8]])], batch=4)
    with pytest.raises(nb.UnsupportedModelError, match="model 1: architecture LSTM"):
        nb.get_dsp_bank([_a1(0), fx.load_model("lstm")], batch=4)


def test_create_refuses_required_jit_with_the_reason():
    with pytest.raises(nb.UnsupportedModelError, match="jit = 1"):
        nb.get_dsp_bank([_a1(0), _a1(1)], batch=4, jit=1)


def test_create_refuses_the_general_kernel_geometry():
    with pytest.raises(nb.UnsupportedModelError, match="kernel_geometry 4"):
        nb.get_dsp_bank([_a1(0), _a1(1)], batch=4, kernel_geometry=4)


def test_bank_entry_points_are_exported():
    from neuralampmodelercore_b200 import _capi

    lib = _capi.load()
    for name in ("nam_b200_create_bank_from_json", "nam_b200_create_bank_from_files", "nam_b200_bank_size",
                 "nam_b200_assign_streams", "nam_b200_stream_models", "nam_b200_bank_model_info",
                 "nam_b200_bank_check_json"):
        assert hasattr(lib, name)
