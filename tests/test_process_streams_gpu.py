"""GPU tests of nam_b200_process_streams_f32 (DSP.process_streams): any set of stream slots in one call, each stream
continuing from its own clock.  The yardstick is the route the library offered before: import the listed streams' records
into slots [0, n) of a second handle with the same options, run a contiguous call there, export them back.  Outputs and
records must match that route byte for byte, and each stream's output must match the oracle run on its own input."""
import ctypes as C

import numpy as np
import pytest

import neuralampmodelercore_b200 as nb
from oracle import nam_config, oracle
from tests import nam_fixtures as fx
from tests.test_multichannel_gpu import _wavenet_2in_3out
from tests.test_reference_build import CONVNETS, _convnet
from tests.test_spec_kernel_gpu import _random_lstm

pytestmark = pytest.mark.gpu
TOL = 1e-5
BLOCK = 256


def _linear():
    rng = np.random.default_rng(3)
    rf = 200
    return {"version": "0.5.4", "architecture": "Linear", "config": {"receptive_field": rf, "bias": True},
            "weights": [float(v) for v in rng.uniform(-0.1, 0.1, rf + 1)], "sample_rate": 48000}


def _model(name):
    if name == "convnet":
        return _convnet(**CONVNETS[0])
    if name == "linear":
        return _linear()
    if name == "multichannel":
        return _wavenet_2in_3out()
    if name == "lstm_h5":
        return _random_lstm(5, 2)
    if name == "lstm_2in_3out":  # multi-channel: the thread-per-stream kernel (lstm_kernel)
        nam = {"version": "0.5.4", "architecture": "LSTM", "sample_rate": 48000.0,
               "config": {"in_channels": 2, "out_channels": 3, "input_size": 2, "hidden_size": 5, "num_layers": 2},
               "weights": []}
        w = np.random.default_rng(23).uniform(-0.35, 0.35, nam_config.expected_weight_count(nam)).astype(np.float32)
        nam["weights"] = [float(v) for v in w]
        return nam
    return fx.load_model(name)


def _dsp(nam, batch, block=BLOCK, slim=None, **kw):
    d = nb.get_dsp(nam, batch=batch, **kw)
    if slim is not None:
        d.SetSlimmableSize(slim)
    d.Reset(48000.0, block)
    return d


class Emulation:
    """The documented route on a second handle: records in, contiguous call on slots [0, n), records out."""

    def __init__(self, d):
        self.d = d
        self.fresh = d.export_streams([0])[0]
        self.rec = {}

    def record(self, s):
        return self.rec.get(s, self.fresh)

    def call(self, streams, x):
        n = len(streams)
        self.d.import_streams(list(range(n)), np.stack([self.record(s) for s in streams]))
        y = self.d.process_batch(x)
        out = self.d.export_streams(list(range(n)))
        for i, s in enumerate(streams):
            self.rec[s] = out[i]
        return y


def _signal(n, frames, ci, seed):
    x = fx.synthetic_batch(n * ci, frames, seed=seed)
    return np.ascontiguousarray(x.reshape(n, ci, frames) if ci > 1 else x)


def _oracle_stream(nam, chunks, block):
    """One oracle instance fed this stream's calls in order.  A chunk None is a standalone DSP::prewarm: zeros in
    `block`-frame calls until at least prewarm_samples were fed (dsp.cpp:67-101), outputs dropped."""
    m = oracle.OracleModel.from_dict(nam)
    m.reset(48000.0, block)
    ys = []
    for c in chunks:
        if c is None:
            for _ in range(0, m.prewarm_samples, block):
                m.process(np.zeros((m.in_channels, block), np.float32))
            continue
        y = m.process(np.ascontiguousarray(c))
        ys.append(np.atleast_2d(y) if c.ndim == 2 else np.asarray(y).reshape(-1))
    m.close()
    return np.concatenate(ys, axis=-1)


def _check_schedule(nam, schedule, frames, batch, block=BLOCK, oracle_streams=None, slim=None, min_launches=1, **kw):
    """schedule: list of stream lists; frames: frames per call (an int or one per call); every call must launch at least
    `min_launches` kernels.  Returns the tested handle."""
    a = _dsp(nam, batch, block, slim=slim, **kw)
    e = Emulation(_dsp(nam, batch, block, slim=slim, **kw))
    ci = a.in_channels
    frames = [frames] * len(schedule) if isinstance(frames, int) else frames
    ins, outs = {}, {}
    for c, (streams, n) in enumerate(zip(schedule, frames)):
        x = _signal(len(streams), n, ci, seed=100 + c)
        n0 = a.launch_count()
        y = a.process_streams(streams, x)
        assert a.launch_count() - n0 >= min_launches, f"call {c}: {a.launch_count() - n0} launches"
        ye = e.call(streams, x)
        assert np.array_equal(y, ye), f"call {c}: outputs differ from the import / contiguous / export route"
        for i, s in enumerate(streams):
            ins.setdefault(s, []).append(x[i])
            outs.setdefault(s, []).append(y[i])
    touched = sorted(ins)
    got = a.export_streams(touched)
    for i, s in enumerate(touched):
        assert np.array_equal(got[i], e.record(s)), f"stream {s}: record differs"
    untouched = [s for s in range(batch) if s not in ins][:8]
    if untouched:
        rec = a.export_streams(untouched)
        assert all(np.array_equal(r, e.fresh) for r in rec), "an unlisted stream changed"
    # (a slimmable handle at size `slim` serves its first sub-model whose max_value is above it)
    ref_nam = nam if slim is None else next(m for mv, m in nb.submodels(nam) if slim < mv)
    for s in (touched if oracle_streams is None else oracle_streams):
        ref = _oracle_stream(ref_nam, ins[s], block)
        err = float(np.max(np.abs(np.concatenate(outs[s], axis=-1) - ref)))
        assert err <= TOL, f"stream {s}: {err:.3e} from the oracle"
    e.d.close()
    return a


def _random_schedule(batch, calls, seed):
    """Random, unordered, non-contiguous subsets; stream 0 sits out the middle calls, stream 1 every call but the last."""
    rng = np.random.default_rng(seed)
    out = []
    for c in range(calls):
        k = int(rng.integers(2, batch))
        s = [int(v) for v in rng.permutation(batch)[:k] if not (v == 0 and 2 <= c < 6) and not (v == 1 and c < calls - 1)]
        if c == calls - 1:
            s = [v for v in s if v != 1] + [1]
        out.append(s or [2])
    return out


# (model, handle options): WaveNet fused, model-specialised and general kernels, A2, condition_dsp, multi-channel, ConvNet,
# Linear, LSTM in its three kernel forms, a slimmable container
CASES = [("wavenet", {}), ("wavenet_a1_standard", {"jit": 1}), ("wavenet_a1_standard", {"jit": 2}),
         ("wavenet_a1_standard", {"kernel_geometry": 4}), ("a2_full", {}), ("wavenet_a2_max", {}), ("multichannel", {}),
         ("convnet", {}), ("linear", {}), ("lstm_h5", {"jit": 1, "kernel_geometry": 1}),
         ("lstm_h5", {"jit": 1, "kernel_geometry": 2}), ("lstm", {"jit": 2}), ("lstm_2in_3out", {"jit": 2}),
         ("slimmable_wavenet", {"slim": 0.0})]
IDS = [f"{n}-{'-'.join(f'{k}{v}' for k, v in kw.items()) or 'default'}" for n, kw in CASES]


@pytest.mark.parametrize("name,kw", CASES, ids=IDS)
def test_subsets_match_the_record_route_and_the_oracle(name, kw):
    nam = _model(name)
    B = 9
    a = _check_schedule(nam, _random_schedule(B, 8, seed=sum(map(ord, name))), BLOCK, B, **kw)
    a.close()


@pytest.mark.parametrize("name,kw", [("wavenet_a1_standard", {"jit": 1}), ("wavenet_a1_standard", {"jit": 2}), ("linear", {}),
                                     ("lstm", {})], ids=["a1-jit1", "a1-jit2", "linear", "lstm"])
def test_identity_list_is_the_contiguous_call(name, kw):
    nam = _model(name)
    B = 6
    a, b = _dsp(nam, B, **kw), _dsp(nam, B, **kw)
    for c in range(3):
        x = fx.synthetic_batch(B, BLOCK, seed=30 + c)
        na, nb_ = a.launch_count(), b.launch_count()
        ya = a.process_streams(list(range(B)), x)
        yb = b.process_batch(x)
        assert np.array_equal(ya, yb)
        assert a.launch_count() - na == b.launch_count() - nb_
    assert np.array_equal(a.export_streams(list(range(B))), b.export_streams(list(range(B))))
    a.close()
    b.close()


def test_low_latency_kernels_take_the_table(monkeypatch):
    """Single-stream 64-frame calls on slot 3 (and a few others) of a jit=3 handle: the model-specialised low-latency
    kernel, then the precompiled one."""
    nam = _model("wavenet_a1_standard")
    sched = [[3], [0, 3], [3], [5], [3], [3, 5], [1], [3]]
    a = _check_schedule(nam, sched, 64, 8, 64, jit=3)
    assert a.jit_lat_state == 1, a.jit_note()
    a.close()
    monkeypatch.setenv("NAM_B200_LAT_KERNEL", "precompiled")
    _check_schedule(nam, sched, 64, 8, 64, jit=3).close()


@pytest.mark.parametrize("jit", [1, 2], ids=["spec_short", "fused_short"])
def test_short_call_kernels_take_the_table(jit):
    """64 / 128 / 256-frame calls on at least 2q streams: the specialised short-call entry points (jit=1), the fused
    short geometries (jit=2)."""
    nam = _model("wavenet_a1_standard")
    B = 48
    rng = np.random.default_rng(7)
    sched = [[int(v) for v in rng.permutation(B)[:int(k)]] for k in (40, 30, 44, 36, 24, 40)]
    a = _check_schedule(nam, sched, [64, 128, 256, 64, 192, 96], B, 256, oracle_streams=sched[0][:3], jit=jit)
    a.close()


def test_single_frame_geometry_and_tile_parallel_modes_take_the_table(monkeypatch):
    nam = _model("wavenet_a1_standard")
    # 128 x 1: few streams, <= 128 frames, the low-latency kernels switched off
    monkeypatch.setenv("NAM_B200_LAT_KERNEL", "off")
    _check_schedule(nam, [[4], [1, 4], [4], [2, 0], [4, 1]], 128, 6, 128, jit=2).close()
    monkeypatch.delenv("NAM_B200_LAT_KERNEL")
    # lock-step tile-parallel (few streams x 4096 frames) and the wavefront (tile_mode 1)
    for tm in (0, 1):
        _check_schedule(nam, [[2], [0, 2], [2], [1, 0]], 4096, 3, 4096, oracle_streams=[2], jit=2, tile_mode=tm).close()


def test_pipelined_host_path_takes_table_chunks():
    """A host-buffer call this large is split into chunks of whole kernel waves, one launch each: at least two launches
    per call show that the chunked path ran (3,400 streams is two chunks or more at up to 3 CTAs per SM on 132 SMs)."""
    nam = _model("wavenet_a1_standard")
    B, n = 4096, 3400
    rng = np.random.default_rng(11)
    sched = [[int(v) for v in rng.permutation(B)[:n]] for _ in range(2)]
    a = _check_schedule(nam, sched, 4096, B, 4096, oracle_streams=[sched[0][0], sched[1][-1]], min_launches=2)
    a.close()


@pytest.mark.parametrize("name", ["wavenet_a1_standard", "linear"])
def test_prewarm_keeps_paused_streams_at_their_own_clock(name):
    """A standalone DSP.prewarm while streams sit out prewarms every stream from its own history, and a paused stream
    stays paused where it stopped: resumed through process_streams or process_batch it matches the oracle."""
    nam = _model(name)
    B = 4
    d = _dsp(nam, B)
    ins = {s: [] for s in range(B)}
    outs = {s: [] for s in range(B)}

    def run(streams, seed, contiguous=False):
        x = fx.synthetic_batch(len(streams), BLOCK, seed=seed)
        y = d.process_batch(x) if contiguous else d.process_streams(streams, x)
        for i, s in enumerate(streams):
            ins[s].append(x[i])
            outs[s].append(y[i])

    run(list(range(B)), 80, contiguous=True)
    run([2, 0], 81)  # streams 1 and 3 sit out
    run([0], 82)
    d.prewarm()
    for s in range(B):
        ins[s].append(None)
    run([3, 1, 0], 83)  # 3 and 1 resume through a table call
    run([2], 84)
    run(list(range(B)), 85, contiguous=True)  # every stream, each behind by its own amount
    run([1, 3], 86)
    for s in range(B):
        ref = _oracle_stream(nam, ins[s], BLOCK)
        err = float(np.max(np.abs(np.concatenate(outs[s]) - ref)))
        assert err <= TOL, f"stream {s}: {err:.3e} from the oracle"
    d.close()


def test_streams_that_sat_out_rejoin_contiguous_calls():
    """process_batch over a prefix that includes streams left out of earlier calls, and DSP::process on stream 0 through
    the low-latency kernel: each continues from its own clock."""
    nam = _model("wavenet_a1_standard")
    B = 6
    d = _dsp(nam, B)
    x = [fx.synthetic_batch(B, BLOCK, seed=40 + c) for c in range(5)]
    widths = [B, 2, 3, 1, B]  # streams >= width sit out a call
    ys = [d.process_batch(np.ascontiguousarray(x[c][:w])) for c, w in enumerate(widths)]
    for s in range(B):
        mine = [c for c, w in enumerate(widths) if s < w]
        ref = _oracle_stream(nam, [x[c][s] for c in mine], BLOCK)
        got = np.concatenate([ys[c][s] for c in mine])
        assert np.max(np.abs(got - ref)) <= TOL, f"stream {s}"
    d.close()

    p = _dsp(nam, 2, 64, jit=3)
    sig = fx.synthetic_batch(2, 64 * 6, seed=50)
    o0 = []
    for c in range(6):
        if c in (1, 2, 3):  # stream 0 sits out: only stream 1 runs
            p.process_streams([1], np.ascontiguousarray(sig[1:2, 64 * c:64 * (c + 1)]))
            continue
        o = np.zeros(64, np.float32)
        p.process([np.ascontiguousarray(sig[0, 64 * c:64 * (c + 1)])], [o], 64)
        o0.append(o)
    ref = _oracle_stream(nam, [sig[0, 64 * c:64 * (c + 1)] for c in (0, 4, 5)], 64)
    assert np.max(np.abs(np.concatenate(o0) - ref)) <= TOL
    p.close()


def test_device_variant_matches_host_variant():
    torch = pytest.importorskip("torch")
    nam = _model("wavenet_a1_standard")
    B = 12
    a, b = _dsp(nam, B), _dsp(nam, B)
    side = torch.cuda.Stream()
    for c, streams in enumerate([[3, 7, 1], [11, 0, 3, 5], [7, 2]]):
        x = fx.synthetic_batch(len(streams), BLOCK, seed=60 + c)
        ya = a.process_streams(streams, x)
        xin = torch.from_numpy(x).cuda()
        out = torch.zeros_like(xin)
        torch.cuda.synchronize()
        b.process_streams_device(streams, xin.data_ptr(), out.data_ptr(), BLOCK, cuda_stream=side.cuda_stream)
        side.synchronize()
        assert np.array_equal(out.cpu().numpy(), ya)
    assert np.array_equal(a.export_streams(list(range(B))), b.export_streams(list(range(B))))
    a.close()
    b.close()


def test_refusals_are_caught_on_the_host():
    nam = _model("wavenet")
    d = nb.get_dsp(nam, batch=4)
    x = fx.synthetic_batch(2, BLOCK, seed=70)
    with pytest.raises(RuntimeError, match="before reset"):
        d.process_streams([0, 1], x)
    d.Reset(48000.0, BLOCK)
    d.process_batch(fx.synthetic_batch(4, BLOCK, seed=71))
    before = d.export_streams([0, 1, 2, 3])
    n0 = d.launch_count()
    with pytest.raises(ValueError, match=r"streams\[1\] = 4: stream index outside"):
        d.process_streams([0, 4], x)
    with pytest.raises(ValueError, match=r"streams\[1\] = 2: duplicate"):
        d.process_streams([2, 2], x)
    with pytest.raises(ValueError, match="outside"):
        d.process_streams([0, 1, 2, 3, 0], fx.synthetic_batch(5, BLOCK, seed=72))
    with pytest.raises(ValueError, match="max_frames"):
        d.process_streams([0, 1], fx.synthetic_batch(2, BLOCK + 1, seed=73))
    s = np.array([0, 1], np.int32)
    sp = s.ctypes.data_as(C.POINTER(C.c_int32))
    buf = np.zeros((2, BLOCK), np.float32)
    vp = buf.ctypes.data_as(C.c_void_p)
    lib, h = d._lib, d._h
    assert lib.nam_b200_process_streams_f32(h, sp, 2, vp, vp, BLOCK, BLOCK - 1, BLOCK) == nb.dsp.ERR_INVALID_ARGUMENT
    assert b"in_stride" in lib.nam_b200_last_error()
    assert lib.nam_b200_process_streams_f32(h, sp, 2, vp, vp, BLOCK, BLOCK, BLOCK - 1) == nb.dsp.ERR_INVALID_ARGUMENT
    assert b"out_stride" in lib.nam_b200_last_error()
    assert lib.nam_b200_process_streams_f32(h, sp, 2, None, vp, BLOCK, BLOCK, BLOCK) == nb.dsp.ERR_INVALID_ARGUMENT
    assert lib.nam_b200_process_streams_f32(h, None, 2, vp, vp, BLOCK, BLOCK, BLOCK) == nb.dsp.ERR_INVALID_ARGUMENT
    assert lib.nam_b200_process_streams_f32_device(h, sp, -1, vp, vp, BLOCK, BLOCK, BLOCK, None) == nb.dsp.ERR_INVALID_ARGUMENT
    assert lib.nam_b200_process_streams_f32(h, sp, 0, None, None, BLOCK, BLOCK, BLOCK) == 0  # no-ops
    assert lib.nam_b200_process_streams_f32(h, sp, 2, vp, vp, 0, 0, 0) == 0
    assert d.launch_count() == n0
    assert np.array_equal(d.export_streams([0, 1, 2, 3]), before)
    d.close()
