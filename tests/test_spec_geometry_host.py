"""CPU-only tests of the model-specialised throughput kernel's tile (csrc/jit_spec.h, spec_tile_geometry): one 1024-thread
CTA per SM for models with at least 512 FFMAs per thread and frame per layer whose history window and 1024-column tile fit
in shared memory, two 512-thread CTAs per SM otherwise.  Shared memory is the widest array's planes of 4 channels x
(history window + tile columns) x 16 bytes per CTA, 226 KB for the CTAs of one SM.  Two 512-thread CTAs took twice the
planes x (history window + 512 columns), never less than one 1024-thread CTA, so every model that had the specialised
kernel keeps it."""
import pytest

import neuralampmodelercore_b200 as nb
from tests import nam_fixtures as fx

SMEM_PER_SM = 226 * 1024


def _window_fits(planes: int, lookback: int, nt: int, ctas: int) -> bool:
    return ctas * planes * (lookback + nt) * 16 <= SMEM_PER_SM


@pytest.mark.parametrize("batch", [1, 256, 4096])
def test_a1_standard_gets_1024_threads(batch):
    rep = nb.jit_prepare(fx.load_model("wavenet_a1_standard"), fast_tanh=True, batch=batch)
    assert rep["ok"], rep["why_not"]
    assert rep["threads"] == 1024
    assert rep["smem_bytes"] == 4 * (1024 + 1024) * 16  # 16 channels, look-back 2 x 512


@pytest.mark.parametrize("name", ["wavenet", "a2_full", "a2_lite"])
def test_fixtures_with_less_work_per_layer_keep_two_512_thread_ctas(name):
    # a2_full: 8 channels, 483 FFMAs per frame per layer; a2_lite and wavenet.nam far fewer
    rep = nb.jit_prepare(fx.load_model(name), fast_tanh=True)
    assert rep["ok"], rep["why_not"]
    assert rep["threads"] == 512


# (channels, kernel size, dilation, threads): the longest single-layer look-back that two 512-thread CTAs per SM could
# hold for 16, 8 and 4 channels (4, 2 and 1 planes); (kernel size + 1) x channels^2 FFMAs per frame and layer: 1024, 192, 48
EDGE_OF_512x2 = [(16, 3, 648, 1024), (8, 2, 3104, 512), (4, 2, 6720, 512)]


@pytest.mark.parametrize("channels,kernel,dilation,threads", EDGE_OF_512x2, ids=["16ch", "8ch", "4ch"])
def test_models_eligible_for_two_512_thread_ctas_stay_eligible(channels, kernel, dilation, threads):
    planes, lookback = channels // 4, (kernel - 1) * dilation
    assert _window_fits(planes, lookback, 512, 2) and not _window_fits(planes, lookback + 1, 512, 2)
    nam = fx.random_wavenet(channels=(channels,), kernel_size=kernel, dilations=[[1, dilation]], seed=4)
    rep = nb.jit_prepare(nam, fast_tanh=False)
    assert rep["ok"], rep["why_not"]
    assert rep["threads"] == threads
    assert rep["smem_bytes"] == planes * (lookback + threads) * 16


def test_a_window_that_does_not_fit_with_1024_columns_gets_512_and_is_refused():
    # 16 channels, look-back 2 x 1300 = 2600: 4 x (2600 + 1024) x 16 = 231,936 B > 226 KB, and two 512-thread CTAs need more
    nam = fx.random_wavenet(channels=(16,), kernel_size=3, dilations=[[1, 1300]], seed=4)
    assert not _window_fits(4, 2600, 1024, 1) and not _window_fits(4, 2600, 512, 2)
    rep = nb.jit_prepare(nam, fast_tanh=False)
    assert rep["threads"] == 512
    assert not rep["ok"]
    assert "do not fit in shared memory" in rep["why_not"]
