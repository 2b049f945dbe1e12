"""CPU-only tests of model banks of general-kernel WaveNets and of ConvNets (nam_b200_bank_check_json and the refusals of
nam_b200_create_bank_from_json, which are decided before any CUDA call): which documents can share one handle."""
import copy

import numpy as np
import pytest

import neuralampmodelercore_b200 as nb
from oracle import nam_config
from tests import nam_fixtures as fx
from tests.test_multichannel_gpu import _randomise, _wavenet_2in_3out
from tests.test_reference_build import _convnet


def _reweighted(doc: dict, seed: int) -> dict:
    """the document with every weight (head_scale, the last, too) seeded-perturbed"""
    d = copy.deepcopy(doc)
    w = np.asarray(doc["weights"], np.float32)
    rng = np.random.default_rng(seed)
    d["weights"] = [float(v) for v in w * (1.0 + 0.05 * rng.standard_normal(w.shape)).astype(np.float32)]
    return d


def _cond_dsp_reweighted(doc: dict, seed: int) -> dict:
    """a condition_dsp WaveNet whose nested document differs in its weights (its head_scale included) and metadata too"""
    d = _reweighted(doc, seed)
    inner = d["config"]["condition_dsp"]
    w = np.asarray(inner["weights"], np.float32)
    rng = np.random.default_rng(100 + seed)
    inner["weights"] = [float(v) for v in w * (1.0 + 0.05 * rng.standard_normal(w.shape)).astype(np.float32)]
    inner["weights"][-1] = 0.5 + 0.1 * seed
    inner["metadata"] = dict(inner.get("metadata") or {}, loudness=-30.0 - seed, name=f"capture {seed}")
    return d


def _edited(doc: dict, edit, seed: int = 9) -> dict:
    """the document with its config edited and fresh random weights of the count the new config expects"""
    d = copy.deepcopy(doc)
    edit(d["config"])
    cd = d["config"].get("condition_dsp")
    if cd:
        _randomise(cd, seed=seed + 1, scale=0.3)
    return _randomise(d, seed=seed, scale=0.3)


def _accepted(docs):
    r = nb.bank_check(docs)
    assert r["ok"] is True, r["reason"]
    assert r["n_models"] == len(docs)
    assert len(set(r["fingerprints"])) == len(docs)
    assert r["fingerprints"] == [nb.state_layout(d)["fingerprint"] for d in docs]
    return r


def _refused(docs, *fields):
    r = nb.bank_check(docs)
    assert r["ok"] is False, r
    for f in fields:
        assert f in r["reason"], (f, r["reason"])
    return r


@pytest.mark.parametrize("name", ["wavenet_a2_max", "wavenet_condition_dsp"])
def test_reweighted_general_fixtures_share_a_bank(name):
    base = fx.load_model(name)
    make = _cond_dsp_reweighted if "condition_dsp" in base["config"] and base["config"]["condition_dsp"] else _reweighted
    _accepted([base] + [make(base, s) for s in range(1, 4)])


def test_condition_dsp_nested_weights_metadata_and_version_are_per_model():
    base = fx.load_model("wavenet_condition_dsp")
    other = _cond_dsp_reweighted(base, 1)
    other["config"]["condition_dsp"]["version"] = "0.5.4"
    other["config"]["condition_dsp"]["config"]["head_scale"] = 0.123  # (the unused config field)
    _accepted([base, other])


def test_multichannel_general_wavenets_share_a_bank():
    base = _wavenet_2in_3out()
    docs = [base] + [_randomise(copy.deepcopy(base), seed=s, last=0.25 * s) for s in (11, 12)]
    _accepted(docs)


@pytest.mark.parametrize("batchnorm", [True, False])
def test_convnets_share_a_bank(batchnorm):
    _accepted([_convnet(8, [1, 2, 4, 8], batchnorm, "Tanh", seed) for seed in range(3)])
    _accepted([_convnet(6, [2, 4, 64], batchnorm, "ReLU", seed, in_channels=2, out_channels=3) for seed in range(3)])


A2 = "wavenet_a2_max"
# (edit of the config, the field the reason names)
A2_REFUSALS = {
    "gating": (lambda c: c["layers"][0].update(gating_mode="gated", secondary_activation="Sigmoid"), "gating mode"),
    "film_active": (lambda c: c["layers"][0]["activation_pre_film"].update(active=False), "FiLM site 4 active"),
    "film_shift": (lambda c: c["layers"][0]["conv_post_film"].update(shift=False), "FiLM site 1 shift"),
    "groups": (lambda c: c["layers"][0].update(groups_input_mixin=2), "groups_input_mixin"),
    "layer1x1_groups": (lambda c: c["layers"][0]["layer1x1"].update(groups=1), "layer1x1 groups"),
    "bottleneck": (lambda c: c["layers"][0].update(bottleneck=8), "bottleneck"),
    "head1x1": (lambda c: (c["layers"][0]["head1x1"].update(active=False),
                           c["layers"][0]["head1x1_post_film"].update(active=False)), "head1x1 active"),
    "condition_dsp_layers": (lambda c: c["condition_dsp"]["config"]["layers"][0].update(dilations=[1, 3]),
                             "condition_dsp array 0 layer 1 dilation"),
    "prelu_slopes": (lambda c: c["condition_dsp"]["config"]["layers"][1]["activation"][0].update(negative_slopes=[0.04]),
                     "PReLU slope count"),
}


@pytest.mark.parametrize("case", sorted(A2_REFUSALS))
def test_general_shape_differences_are_refused_naming_model_and_field(case):
    edit, field = A2_REFUSALS[case]
    base = fx.load_model(A2)
    other = _edited(base, edit)
    assert nb.bank_check([other])["ok"] is True, "the edited document must be valid on its own"
    r = _refused([base, _reweighted(base, 1), other], "model 2", field)
    assert r["reason"].startswith("model 2 differs from model 0")


CONVNET_REFUSALS = {
    "channels": (dict(channels=6), "channels"),
    "dilations": (dict(dilations=[1, 2, 4, 16]), "block 3 dilation"),
    "batchnorm": (dict(batchnorm=False), "batchnorm"),
    "activation": (dict(activation="ReLU"), "activation"),
}


@pytest.mark.parametrize("case", sorted(CONVNET_REFUSALS))
def test_convnet_shape_differences_are_refused_naming_model_and_field(case):
    kw, field = CONVNET_REFUSALS[case]
    base = dict(channels=8, dilations=[1, 2, 4, 8], batchnorm=True, activation="Tanh")
    docs = [_convnet(seed=0, **base), _convnet(seed=1, **dict(base, **kw))]
    _refused(docs, "model 1 differs from model 0", field)


def test_errors_are_model_errors():
    base = fx.load_model(A2)
    with pytest.raises(RuntimeError, match="model 1 differs from model 0 in array 0 bottleneck"):
        nb.get_dsp_bank([base, _edited(base, A2_REFUSALS["bottleneck"][0])], batch=4)


@pytest.mark.parametrize("first", ["fused", "general"])
def test_fused_and_general_kernel_families_do_not_mix(first):
    fused, general = fx.random_wavenet(seed=0), fx.load_model(A2)
    docs = [fused, general] if first == "fused" else [general, fused]
    other = "general" if first == "fused" else "fused"
    r = _refused(docs)
    assert r["reason"].startswith("model 1: kernel: served by the " + other + " kernel"), r["reason"]
    assert "model 0 (" + first + " family) chooses the bank's kernel family" in r["reason"]
    with pytest.raises(nb.UnsupportedModelError, match="model 1: kernel"):
        nb.get_dsp_bank(docs, batch=4)


@pytest.mark.parametrize("order", ["wavenet_first", "convnet_first"])
def test_wavenets_and_convnets_do_not_mix(order):
    wn, cn = fx.load_model(A2), _convnet(8, [1, 2, 4], True, "Tanh", 1)
    docs = [wn, cn] if order == "wavenet_first" else [cn, wn]
    arch0, arch1 = ("WaveNet", "ConvNet") if order == "wavenet_first" else ("ConvNet", "WaveNet")
    _refused(docs, f"model 1: architecture {arch1}: a bank's models share model 0's architecture ({arch0})")


def test_fused_banks_still_refuse_required_jit_and_the_general_geometry():
    docs = [fx.random_wavenet(seed=0), fx.random_wavenet(seed=1)]
    with pytest.raises(nb.UnsupportedModelError, match="jit = 1"):
        nb.get_dsp_bank(docs, batch=4, jit=1)
    with pytest.raises(nb.UnsupportedModelError, match="kernel_geometry 4"):
        nb.get_dsp_bank(docs, batch=4, kernel_geometry=4)


def test_bank_jit_prepare_shares_one_cubin_per_shape(tmp_path, monkeypatch):
    monkeypatch.setenv("NAM_B200_JIT_CACHE", str(tmp_path))
    base = fx.load_model(A2)
    first = nb.bank_jit_prepare([base, _reweighted(base, 1)], fast_tanh=False)
    assert first["ok"] and not first["from_cache"], first
    second = nb.bank_jit_prepare([_reweighted(base, 2), _reweighted(base, 3), _reweighted(base, 4)], fast_tanh=False)
    assert second["ok"] and second["from_cache"], second  # (the header holds no weight)
    assert len(list(tmp_path.glob("*.cubin"))) == 1
    with pytest.raises(nb.UnsupportedModelError, match="shape-compiled"):
        nb.bank_jit_prepare([_convnet(8, [1, 2], True, "Tanh", s) for s in range(2)])
    with pytest.raises(RuntimeError, match="model 1 differs from model 0"):
        nb.bank_jit_prepare([base, _edited(base, A2_REFUSALS["bottleneck"][0])])


def test_bank_cubin_reads_weights_from_shared_memory(tmp_path, monkeypatch):
    """The shape-compiled kernel's FFMAs take their weights from shared-memory loads; the model-specialised kernel of the
    same model has them as immediates"""
    import re
    import shutil
    import subprocess

    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    base = fx.load_model(A2)
    (tmp_path / "bank").mkdir()
    (tmp_path / "one").mkdir()
    monkeypatch.setenv("NAM_B200_JIT_CACHE", str(tmp_path / "bank"))
    assert nb.bank_jit_prepare([base, _reweighted(base, 1)], fast_tanh=False)["ok"]
    monkeypatch.setenv("NAM_B200_JIT_CACHE", str(tmp_path / "one"))
    assert nb.jit_prepare(base, fast_tanh=False)["ok"]

    def sass(d):
        (cubin,) = list(d.glob("*.cubin"))
        return subprocess.run(["cuobjdump", "-sass", str(cubin)], capture_output=True, text=True, check=True).stdout

    imm = re.compile(r"FFMA R\d+, R\d+(?:\.reuse)?, -?[0-9]")
    bank, one = sass(tmp_path / "bank"), sass(tmp_path / "one")
    n_bank, n_one = len(imm.findall(bank)), len(imm.findall(one))
    assert n_one > 500 and n_bank * 10 < n_one, (n_bank, n_one)
    assert len(re.findall(r"\bLDS(\.\w+)*\b", bank)) > 100
    assert len(re.findall(r"\bFFMA\b", bank)) > 500


def test_record_fingerprints_keep_the_nested_document():
    """The bank rule ignores the nested document's weights; a stream's record still names the whole model"""
    base = fx.load_model("wavenet_condition_dsp")
    other = copy.deepcopy(base)
    other["config"]["condition_dsp"]["weights"][0] += 0.25
    assert nb.state_layout(base)["fingerprint"] != nb.state_layout(other)["fingerprint"]
    assert nb.bank_check([base, other])["ok"] is True
    assert nam_config.expected_weight_count(other) == len(other["weights"])
