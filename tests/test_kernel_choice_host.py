"""CPU-only tests of the kernel choice: nam_b200_inspect_json, nam_b200_jit_prepare_json and a handle (create) make one
decision per model, so inspect reports the kernel, variant, work and state size a handle with the default options gets.
tests/test_kernel_choice_gpu.py checks the same numbers against real handles."""
import pytest

import neuralampmodelercore_b200 as nb
from tests import nam_fixtures as fx

# (kernel, kernel_variant, flops_per_frame, reason) of every fixture under tests/golden/models
FIXTURE_KERNELS = {
    "a2_full": ("fused", 800, 23552, ""),
    "a2_lite": ("fused", 400, 3462, ""),
    "lstm": ("lstm", 2003, 102, ""),
    "slimmable_wavenet": ("fused", 400, 792, ""),
    "wavenet": ("fused", 404, 226, ""),
    "wavenet_a1_standard": ("fused", 1608, 26640, ""),
    "wavenet_a2_max": ("generic", 9000, 3166, "fused kernel: condition_dsp sub-model"),
    "wavenet_condition_dsp": ("generic", 9000, 492, "fused kernel: condition_dsp sub-model"),
}


@pytest.mark.parametrize("name", sorted(FIXTURE_KERNELS))
def test_inspect_of_every_fixture_is_pinned(name):
    rep = nb.inspect(fx.load_model(name))
    assert (rep["kernel"], rep["kernel_variant"], rep["flops_per_frame"], rep["reason"]) == FIXTURE_KERNELS[name]


def _large_wavenet():
    # 52,002 weights: a 208 KB packed blob, which with the 36 KB tile of the default geometry exceeds the 227 KB of shared
    # memory of the fused kernel
    return fx.random_wavenet(channels=(16, 16), dilations=[[1, 2, 4, 8, 16, 32] * 4] * 2)


def test_inspect_of_a_wavenet_too_large_for_the_fused_kernel_reports_the_general_one():
    nam = _large_wavenet()
    rep = nb.inspect(nam)
    assert rep["n_weights"] == 52002
    assert rep["kernel"] == "generic" and rep["kernel_variant"] == 9000, rep
    assert rep["reason"] == "fused kernel: packed weights + tile exceed the 227 KB of shared memory of the fused kernel"
    assert (rep["flops_per_frame"], rep["state_bytes_per_stream"]) == (100928, 786432)  # the general kernel's rings


def test_jit_prepare_of_a_wavenet_too_large_for_the_fused_kernel_builds_the_general_one(tmp_path, monkeypatch):
    monkeypatch.setenv("NAM_B200_JIT_CACHE", str(tmp_path))
    rep = nb.jit_prepare(_large_wavenet(), fast_tanh=False)
    # the general kernel's builder declines to unroll that many weights (its 128-thread tile), and no low-latency kernel
    # (a fused-family kernel) is built
    assert not rep["ok"] and rep["why_not"].startswith("too many weights to unroll"), rep
    assert rep["threads"] == 128 and not rep["lat_ok"]


def _lstm(out_channels, hidden=2):
    H, O = hidden, out_channels
    return {"version": "0.5.4", "architecture": "LSTM", "sample_rate": 48000,
            "config": {"input_size": 1, "hidden_size": H, "num_layers": 1, "out_channels": O},
            "weights": [0.01] * (4 * H * (1 + H) + 4 * H + 2 * H + O * H + O)}


def test_inspect_of_an_lstm_create_refuses_is_unsupported():
    rep = nb.inspect(_lstm(out_channels=65))
    assert rep["kernel"] == "unsupported" and rep["reason"] == "LSTM head with 65 rows for 65 output channels", rep
    assert (rep["kernel_variant"], rep["flops_per_frame"], rep["state_bytes_per_stream"]) == (0, 0, 0)
    assert nb.inspect(_lstm(out_channels=64))["kernel"] == "lstm"


def test_inspect_state_bytes_are_the_handles():
    # LSTM rows (per layer h | c) and Linear histories are rounded up to 4 floats; Linear keeps at least one float
    assert nb.inspect(fx.load_model("lstm"))["state_bytes_per_stream"] == 32  # 1 layer x 2 x 3 floats -> 8
    assert nb.inspect(_lstm(out_channels=2, hidden=3))["state_bytes_per_stream"] == 32
    for rf, floats in ((6, 8), (9, 8), (1, 4)):
        lin = {"version": "0.5.4", "architecture": "Linear", "sample_rate": 48000,
               "config": {"receptive_field": rf, "bias": True}, "weights": [0.01] * (rf + 1)}
        assert nb.inspect(lin)["state_bytes_per_stream"] == 4 * floats, rf
