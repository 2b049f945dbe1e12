"""inspect() describes what a handle with the default options runs: its kernel variant, work per frame and state size per
stream are the handle's own (nam_b200_get_info), for every fixture and for the models where the two once disagreed."""
import pytest

import neuralampmodelercore_b200 as nb
from tests import nam_fixtures as fx
from tests.test_kernel_choice_host import FIXTURE_KERNELS, _large_wavenet, _lstm

pytestmark = pytest.mark.gpu


def _linear(rf):
    return {"version": "0.5.4", "architecture": "Linear", "sample_rate": 48000,
            "config": {"receptive_field": rf, "bias": True}, "weights": [0.01] * (rf + 1)}


MODELS = {**{name: (lambda name=name: fx.load_model(name)) for name in FIXTURE_KERNELS},
          "wavenet_too_large_for_fused": _large_wavenet, "lstm_2ch_h3": lambda: _lstm(out_channels=2, hidden=3),
          "linear_rf6": lambda: _linear(6), "linear_rf1": lambda: _linear(1)}


@pytest.mark.parametrize("name", sorted(MODELS))
def test_inspect_matches_the_handle(name):
    nam = MODELS[name]()
    rep = nb.inspect(nam)
    d = nb.get_dsp(nam, batch=2)
    try:
        info = d.info
        assert rep["state_bytes_per_stream"] == info.state_bytes_per_stream
        assert rep["kernel_variant"] == info.kernel_variant
        assert rep["flops_per_frame"] == info.flops_per_frame
    finally:
        d.close()
    if name == "wavenet_too_large_for_fused":
        assert info.kernel_variant == 9000  # the general kernel
