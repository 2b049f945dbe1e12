"""Host-only checks of the sample-rate conversion (nam_b200_options.resample): the published filter design against its
documented formula and its frequency-response requirements, the refusals, and the ABI fields.  No GPU needed."""
import ctypes
import inspect
import math

import numpy as np
import pytest
from scipy import signal

import neuralampmodelercore_b200 as nb
from neuralampmodelercore_b200 import _capi


def _formula(host, model):
    """The design include/nam_b200.h documents, restated in numpy (float64)."""
    g = math.gcd(int(host), int(model))
    L, M = int(model) // g, int(host) // g
    fs = host * L
    fmin = min(host, model)
    A = 84.0
    beta = 0.1102 * (A - 8.7)
    fc, df = 0.45 * fmin / fs, 0.1 * fmin / fs
    N = int(math.ceil((A - 7.95) / (2.285 * 2 * math.pi * df))) + 1
    n = np.arange(N)
    c = (N - 1) / 2
    w = np.i0(beta * np.sqrt(np.maximum(0.0, 1 - ((n - c) / c) ** 2))) / np.i0(beta)
    return L, M, 2 * fc * np.sinc(2 * fc * (n - c)) * w


def test_44k1_to_48k_is_the_documented_design():
    d = nb.resampler(44100, 48000)
    assert (d["L"], d["M"]) == (160, 147)
    assert d["taps_per_output_up"] <= 64 and d["taps_per_output_down"] <= 64
    L, M, g = _formula(44100.0, 48000.0)
    assert d["n_taps"] == len(g) == len(d["g_up"]) == len(d["g_dn"])
    assert d["taps_per_output_up"] == -(-len(g) // L) and d["taps_per_output_down"] == -(-len(g) // M)
    np.testing.assert_allclose(d["g_up"], L * g, rtol=0, atol=1e-7)
    np.testing.assert_allclose(d["g_dn"], M * g, rtol=0, atol=1e-7)
    assert d["latency_frames"] == pytest.approx((len(g) - 1) / L, rel=1e-8)


@pytest.mark.parametrize("host,model", [(44100, 48000), (48000, 44100), (96000, 48000), (32000, 48000)])
def test_published_taps_meet_ripple_and_stopband(host, model):
    d = nb.resampler(host, model)
    L = d["L"]
    fs = host * L
    fmin = min(host, model)
    for taps, gain in ((d["g_up"], L), (d["g_dn"], d["M"])):
        g = taps.astype(np.float64) / gain
        f_pass = np.linspace(0.0, 0.4 * fmin, 4000)
        f_stop = np.linspace(0.5 * fmin, fs / 2, 200000)
        _, hp = signal.freqz(g, worN=f_pass, fs=fs)
        _, hs = signal.freqz(g, worN=f_stop, fs=fs)
        db_pass = 20 * np.log10(np.abs(hp))
        assert db_pass.max() - db_pass.min() <= 0.1
        assert 20 * np.log10(np.abs(hs).max()) - db_pass.max() <= -80.0
    assert max(d["taps_per_output_up"], d["taps_per_output_down"]) <= 128


@pytest.mark.parametrize("host,model,words", [
    (48000, 44101, ("48000", "44101", "1024")),  # L, M > 1024
    (44100.5, 48000, ("44100.5", "48000", "integer")),
    (44100, -1, ("44100", "unknown")),
])
def test_refusals_name_both_rates(host, model, words):
    with pytest.raises(ValueError) as e:
        nb.resampler(host, model)
    for w in words:
        assert w in str(e.value)


def test_abi_fields():
    o = _capi.Options
    assert ctypes.sizeof(o) == 56 and o.resample.offset == o.bank_capacity.offset + 4 == 40
    opts = o()
    ctypes.memset(ctypes.byref(opts), 0x5A, ctypes.sizeof(opts))
    lib = _capi.load()
    lib.nam_b200_default_options(ctypes.byref(opts))
    assert opts.resample == 0 and list(opts.reserved_tail) == [0, 0, 0]
    i = _capi.Info
    assert i.resample_up.offset == i.jit_lat_state.offset + 4
    assert i.resample_down.offset == i.resample_up.offset + 4
    assert i.resample_latency_frames.offset == i.resample_down.offset + 4
    assert i.reserved.offset + i.reserved.size == ctypes.sizeof(i)
    header = (_capi.lib_path().parents[2] / "include" / "nam_b200.h").read_text()
    assert "int nam_b200_resampler_json(" in header and "int32_t resample;" in header
    assert "nam_b200_resampler_json" in _capi.EXPORTED_SYMBOLS and hasattr(lib, "nam_b200_resampler_json")


def test_python_signatures():
    assert inspect.signature(nb.get_dsp).parameters["resample"].default is False
    assert inspect.signature(nb.get_dsp_bank).parameters["resample"].default is False
    assert isinstance(inspect.getattr_static(nb.DSP, "resample_ratio"), property)
    assert isinstance(inspect.getattr_static(nb.DSP, "resample_latency"), property)


def test_small_buffer_is_refused():
    lib = _capi.load()
    buf = ctypes.create_string_buffer(64)
    assert lib.nam_b200_resampler_json(44100.0, 48000.0, buf, len(buf)) == -1
