"""GPU tests of the sample-rate conversion (get_dsp(resample=True), nam_b200_options.resample): equal rates change
nothing, each converted stream matches scipy's upfirdn around the C oracle, the result does not depend on how the audio
is split into calls, a tone comes back at its level after the documented latency, and banks, records, slimmable
containers and the device entries carry the conversion like every other per-stream state."""
import copy

import numpy as np
import pytest
from scipy import signal

import neuralampmodelercore_b200 as nb
from oracle import oracle
from tests import nam_fixtures as fx
from tests.test_process_streams_gpu import _linear
from tests.test_reference_build import CONVNETS, _convnet

pytestmark = pytest.mark.gpu
TOL = 2e-5
MODELS = ["wavenet", "wavenet_a1_standard", "lstm", "wavenet_a2_max", "linear", "convnet"]


def _with_rate(doc, rate):
    """The document with every (sub-)model's sample_rate set, a condition_dsp's included (they must agree)."""
    if isinstance(doc, dict):
        out = {k: _with_rate(v, rate) for k, v in doc.items()}
        if "architecture" in doc:
            out["sample_rate"] = rate
        return out
    if isinstance(doc, list) and doc and isinstance(doc[0], (dict, list)):
        return [_with_rate(v, rate) for v in doc]
    return doc


def _model(name, rate=None):
    nam = _convnet(**CONVNETS[0]) if name == "convnet" else _linear() if name == "linear" else fx.load_model(name)
    return copy.deepcopy(nam) if rate is None else _with_rate(nam, rate)


def _dsp(nam, host, block, batch=1, resample=True, **kw):
    d = nb.get_dsp(nam, batch=batch, resample=resample, **kw)
    d.Reset(host, block)
    return d


def _signal(n, seed=0, batch=1):
    """Audio-like test input: the golden sine section plus a little noise."""
    x = fx.input_wav()[48000:48000 + n]
    rng = np.random.default_rng(seed)
    return np.ascontiguousarray((x[None, :] + 0.05 * rng.standard_normal((batch, n))).astype(np.float32))


def _in_calls(d, x, block):
    return np.concatenate([d.process_batch(np.ascontiguousarray(x[:, i:i + block])) for i in range(0, x.shape[1], block)], axis=1)


@pytest.mark.parametrize("name", MODELS)
def test_equal_rates_change_nothing(name):
    nam = _model(name)
    rate = nb.get_dsp(nam).GetExpectedSampleRate()
    x = _signal(1000, batch=3)
    d0 = _dsp(nam, rate, 256, batch=3, resample=False)
    d1 = _dsp(nam, rate, 256, batch=3, resample=True)
    assert d1.resample_ratio == (1, 1) and d1.resample_latency == 0
    y0, y1 = _in_calls(d0, x, 256), _in_calls(d1, x, 256)
    assert y0.tobytes() == y1.tobytes()
    assert d0.launch_count() == d1.launch_count()
    assert d0.state_record_bytes == d1.state_record_bytes


def _oracle_route(nam, x, host, model_rate, block, fast_tanh):
    """upfirdn (float64, published taps) -> the C oracle at the model's rate on the float32 signal -> upfirdn back."""
    r = nb.resampler(host, model_rate)
    L, M = r["L"], r["M"]
    n = len(x)
    k = -(-n * L // M)
    y = signal.upfirdn(r["g_up"].astype(np.float64), x.astype(np.float64), L, M)[:k].astype(np.float32)
    om = oracle.OracleModel.from_dict(nam, fast_tanh=fast_tanh)
    mb = -(-block * L // M)
    om.reset(model_rate, mb)
    z = np.concatenate([np.asarray(om.process(y[i:i + mb]), np.float32).reshape(-1) for i in range(0, k, mb)])
    om.close()
    return signal.upfirdn(r["g_dn"].astype(np.float64), z.astype(np.float64), M, L)[:n]


@pytest.mark.parametrize("fast_tanh", [False, True])
@pytest.mark.parametrize("pair", [(44100.0, 48000.0), (48000.0, 44100.0), (96000.0, 48000.0)])
@pytest.mark.parametrize("name", MODELS)
def test_matches_upfirdn_around_the_oracle(name, pair, fast_tanh):
    host, model_rate = pair
    nam = _model(name, model_rate)
    block = 512
    x = _signal(6000, seed=1)
    d = _dsp(nam, host, block, fast_tanh=fast_tanh)
    r = nb.resampler(host, model_rate)
    assert d.resample_ratio == (r["L"], r["M"]) and d.resample_latency == round(r["latency_frames"])
    y = _in_calls(d, x, block)[0]
    ref = _oracle_route(nam, x[0], host, model_rate, block, fast_tanh)
    err = float(np.max(np.abs(y - ref)))
    assert err <= TOL, f"{err:.3e} from upfirdn around the oracle"


def test_call_split_invariance():
    nam = _model("wavenet_a1_standard", 48000.0)
    x = fx.input_wav()[None, :].astype(np.float32)  # 2 s, taken as 44.1 kHz audio
    n = x.shape[1]
    ref = _in_calls(_dsp(nam, 44100.0, 64), x, 64)
    assert ref.tobytes() == _in_calls(_dsp(nam, 44100.0, 4096), x, 4096).tobytes()
    assert ref.tobytes() == _dsp(nam, 44100.0, n).process_batch(x).tobytes()
    # ragged calls: three streams of the same audio, each cut at its own random lengths
    rng = np.random.default_rng(7)
    d = _dsp(nam, 44100.0, 1000, batch=3)
    pos = [0, 0, 0]
    outs = [[], [], []]
    while min(pos) < n:
        counts = [int(min(rng.integers(0, 1001), n - p)) for p in pos]
        xr = np.zeros((3, max(max(counts), 1)), np.float32)
        for i in range(3):
            xr[i, :counts[i]] = x[0, pos[i]:pos[i] + counts[i]]
        if max(counts) == 0:
            continue
        y = d.process_streams([0, 1, 2], np.ascontiguousarray(xr[:, :max(counts)]), n_frames=counts)
        for i in range(3):
            outs[i].append(y[i, :counts[i]])
            pos[i] += counts[i]
    for i in range(3):
        assert np.concatenate(outs[i]).tobytes() == ref[0].tobytes(), f"ragged stream {i}"
    # streams left out of process_streams calls resume where they were
    d = _dsp(nam, 44100.0, 512, batch=3)
    outs = [[], [], []]
    pos = [0, 0, 0]
    for c in range(0, 60):
        streams = [s for s in range(3) if (c + s) % 3 != 0]
        xs = np.stack([x[0, pos[s]:pos[s] + 512] for s in streams])
        y = d.process_streams(streams, np.ascontiguousarray(xs))
        for i, s in enumerate(streams):
            outs[s].append(y[i])
            pos[s] += 512
    for s in range(3):
        got = np.concatenate(outs[s])
        assert got.tobytes() == ref[0, :len(got)].tobytes(), f"stream {s} after sitting out calls"


def test_identity_tone_level_and_latency():
    nam = {"version": "0.5.4", "architecture": "Linear", "config": {"receptive_field": 1, "bias": False}, "weights": [1.0],
           "sample_rate": 48000}
    host = 44100.0
    d = _dsp(nam, host, 441)
    n = 44100
    t = np.arange(n) / host
    x = (0.5 * np.sin(2 * np.pi * 1000.0 * t)).astype(np.float32)[None, :]
    y = _in_calls(d, x, 441)[0]
    lat = nb.resampler(host, 48000.0)["latency_frames"]
    assert d.resample_latency == round(lat)
    steady = slice(2000, n - 2000)
    level = 20 * np.log10(np.sqrt(np.mean(y[steady] ** 2)) / np.sqrt(np.mean(x[0, steady] ** 2)))
    assert abs(level) <= 0.1, f"{level:.3f} dB"
    # the delay: cross-correlation with a Hann-windowed burst of the same tone (its envelope makes the true lag the
    # highest peak, where the steady tone repeats every 44.1 frames), fed after the steady part
    burst = np.zeros((1, 4410), np.float32)
    burst[0, 441:441 + 882] = (0.5 * np.hanning(882) * np.sin(2 * np.pi * 1000.0 * np.arange(882) / host)).astype(np.float32)
    d2 = _dsp(nam, host, 441)
    yb = _in_calls(d2, burst, 441)[0]
    xc = [float(np.dot(yb[k:], burst[0, :len(yb) - k])) for k in range(200)]
    best = int(np.argmax(xc))
    assert abs(best - lat) <= 1.0, (best, lat)


def _a1_variants(k):
    base = _model("wavenet_a1_standard", 48000.0)
    out = []
    for i in range(k):
        m = copy.deepcopy(base)
        m["weights"] = [float(w) * (1.0 + 0.03 * i) for w in base["weights"]]
        out.append(m)
    return out


def test_bank_streams_equal_ordinary_converting_handles():
    models = _a1_variants(3)
    bank = nb.get_dsp_bank(models, batch=3, resample=True)
    bank.Reset(44100.0, 256)
    bank.assign_streams([0, 1, 2], [0, 1, 2])
    singles = [_dsp(m, 44100.0, 256, jit=2) for m in models]
    x = _signal(2000, seed=3, batch=3)
    y = _in_calls(bank, x, 256)
    for k in range(3):
        assert y[k].tobytes() == _in_calls(singles[k], x[k:k + 1], 256)[0].tobytes(), f"model {k}"
    # a reassigned / reset stream is a freshly reset handle of its model
    bank.assign_streams([0], [2])
    bank.reset_streams([1])
    x2 = _signal(1500, seed=4, batch=3)
    y2 = _in_calls(bank, x2, 256)
    for s, k in ((0, 2), (1, 1)):
        fresh = _dsp(models[k], 44100.0, 256, jit=2)
        assert y2[s].tobytes() == _in_calls(fresh, x2[s:s + 1], 256)[0].tobytes(), f"stream {s}"


def test_records_carry_the_conversion():
    nam = _model("wavenet_a1_standard", 48000.0)
    x = _signal(3000, seed=5, batch=2)
    a = _dsp(nam, 44100.0, 300, batch=2)
    _in_calls(a, x[:, :1337], 300)
    rec = a.export_streams([0, 1])
    assert rec.shape[1] == a.state_record_bytes > _dsp(nam, 44100.0, 300, resample=False).state_record_bytes
    assert int.from_bytes(rec[0, 12:16].tobytes(), "little") == (160 << 16 | 147)
    b = _dsp(nam, 44100.0, 300, batch=2)
    b.import_streams([1, 0], rec)
    ya = _in_calls(a, x[:, 1337:], 300)
    yb = _in_calls(b, x[::-1, 1337:], 300)
    assert ya.tobytes() == yb[::-1].tobytes()
    # a handle at another ratio, or one that converts nothing, refuses the record naming the field
    for other in (_dsp(nam, 44100.0, 300, resample=False), _dsp(nam, 96000.0, 300)):
        with pytest.raises(ValueError, match="resample ratio"):
            other.import_streams([0], rec[:1])
    with pytest.raises(ValueError, match="resample ratio"):
        a.import_streams([0], _dsp(nam, 44100.0, 300, resample=False).export_streams([0]))
    # a copy_streams swap carries the conversion state along
    c = _dsp(nam, 44100.0, 300, batch=2)
    _in_calls(c, x[:, :1337], 300)
    c.copy_streams([0, 1], [1, 0])
    yc = _in_calls(c, x[::-1, 1337:], 300)
    assert yc[::-1].tobytes() == ya.tobytes()


def test_slimmable_container_converts_like_its_sub_model():
    lite, full = fx.load_model("a2_lite"), fx.load_model("a2_full")
    cont = nb.get_dsp(fx.make_container([(0.5, lite), (1.0, full)]), resample=True)
    cont.Reset(44100.0, 256)
    cont.SetSlimmableSize(0.3)
    ref = _dsp(lite, 44100.0, 256)
    assert cont.resample_ratio == (160, 147)
    x = _signal(1500, seed=6)
    assert _in_calls(cont, x, 256).tobytes() == _in_calls(ref, x, 256).tobytes()


def test_device_entries_equal_host_entries():
    torch = pytest.importorskip("torch")
    nam = _model("wavenet_a1_standard", 48000.0)
    x = _signal(2048, seed=8, batch=4)
    host = _dsp(nam, 44100.0, 512, batch=4)
    dev = _dsp(nam, 44100.0, 512, batch=4)
    st = torch.cuda.Stream()
    xin = torch.from_numpy(x).cuda()
    out = torch.empty_like(xin)
    yh = []
    for i in range(0, 2048, 512):
        yh.append(host.process_batch(np.ascontiguousarray(x[:, i:i + 512])))
        xi = xin[:, i:i + 512].contiguous()
        oi = torch.empty_like(xi)
        with torch.cuda.stream(st):
            dev.process_batch_device(xi.data_ptr(), oi.data_ptr(), 4, 512, cuda_stream=st.cuda_stream)
        st.synchronize()
        out[:, i:i + 512] = oi
    assert out.cpu().numpy().tobytes() == np.concatenate(yh, axis=1).tobytes()
    # the stream-list and ragged device entries against their host twins
    counts = [100, 0, 512, 37]
    xr = np.zeros((4, 512), np.float32)
    for i, k in enumerate(counts):
        xr[i, :k] = x[i, :k]
    yr = host.process_streams([3, 1, 0, 2], xr, n_frames=counts)
    xi = torch.from_numpy(xr).cuda()
    oi = torch.zeros_like(xi)
    with torch.cuda.stream(st):
        dev.process_streams_device([3, 1, 0, 2], xi.data_ptr(), oi.data_ptr(), counts, cuda_stream=st.cuda_stream)
    st.synchronize()
    assert oi.cpu().numpy().tobytes() == yr.tobytes()
    assert np.array_equal(host.export_streams([0, 1, 2, 3]), dev.export_streams([0, 1, 2, 3]))


def test_planar_process_equals_batched():
    nam = _model("wavenet")
    x = _signal(1024, seed=9)
    a = _dsp(nam, 44100.0, 128)
    b = _dsp(nam, 44100.0, 128)
    y = []
    for i in range(0, 1024, 128):
        out = np.zeros(128, np.float64)
        a.process([x[0, i:i + 128].astype(np.float64)], [out], 128)
        y.append(out.astype(np.float32))
    assert np.concatenate(y).tobytes() == _in_calls(b, x, 128)[0].tobytes()


def test_refusals():
    nam = _model("wavenet")
    d = nb.get_dsp(nam, resample=True)
    with pytest.raises(ValueError, match="44101"):
        d.Reset(44101.0, 64)
    unknown = copy.deepcopy(nam)
    unknown.pop("sample_rate", None)
    du = nb.get_dsp(unknown, resample=True)
    if du.GetExpectedSampleRate() == -1:
        with pytest.raises(ValueError, match="unknown"):
            du.Reset(44100.0, 64)
    d.Reset(44100.0, 64)
    with pytest.raises(ValueError, match="max_frames"):
        d.process_batch(np.zeros((1, 65), np.float32))
