"""GPU tests of per-stream state control (include/nam_b200.h: nam_b200_reset_streams, copy, export / import of state
records, per-stream clocks): round trips, exact continuation across handles and kernels, single-stream resets, copies,
streams that sat out calls, and the refusals -- which feed bad arguments only and are all caught on the host."""
import json

import numpy as np
import pytest

import neuralampmodelercore_b200 as nb
from oracle import oracle
from tests import nam_fixtures as fx
from tests.test_reference_build import CONVNETS, _convnet

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
    return fx.load_model(name)


# WaveNet fused (+ model-specialised), A2 (kernel-16 head convolution), general kernel with condition_dsp, ConvNet, Linear, LSTM
CASES = [("wavenet", {}), ("wavenet_a1_standard", {"jit": 1}), ("wavenet_a1_standard", {"jit": 2}), ("a2_full", {}),
         ("wavenet_a2_max", {}), ("convnet", {}), ("linear", {}), ("lstm", {})]
IDS = [f"{n}-{'-'.join(f'{k}{v}' for k, v in kw.items()) or 'default'}" for n, kw in CASES]


def _dsp(nam, batch, block=BLOCK, **kw):
    d = nb.get_dsp(nam, batch=batch, **kw)
    d.Reset(48000.0, block)
    return d


def _run(d, x, block=BLOCK):
    """x (batch, n) through `block`-frame calls of x.shape[0] streams."""
    return np.concatenate([d.process_batch(np.ascontiguousarray(x[:, p:p + block])) for p in range(0, x.shape[1], block)], axis=1)


def _oracle(nam, x, block=BLOCK, fast=False):
    x = np.ascontiguousarray(x, np.float32)
    if nam["architecture"] == "ConvNet":  # (no batched oracle runs: one instance per stream)
        ys = []
        for row in x:
            m = oracle.OracleModel.from_dict(nam, fast_tanh=fast)
            m.reset(48000.0, block)
            ys.append(m.run(row, block))
            m.close()
        return np.stack(ys)
    proto = oracle.OracleModel.from_dict(nam, fast_tanh=fast)
    proto.reset(48000.0, block)
    y = proto.run_batch(x, block)
    proto.close()
    return y


@pytest.mark.parametrize("name,kw", CASES, ids=IDS)
def test_round_trip_is_byte_identical(name, kw):
    nam = _model(name)
    d = _dsp(nam, 5, **kw)
    _run(d, fx.synthetic_batch(5, 700, seed=1))
    streams = [0, 1, 2, 3, 4]
    rec = d.export_streams(streams)
    assert rec.shape == (5, d.state_record_bytes) == (5, nb.state_layout(nam)["record_bytes"])
    assert bytes(rec[0, :4]) == b"NAMS"
    d.import_streams(streams, rec)
    assert np.array_equal(d.export_streams(streams), rec)
    d.import_streams([4, 3, 2, 1, 0], rec)  # (the clock moves nothing: records are phase-free)
    assert np.array_equal(d.export_streams([4, 3, 2, 1, 0]), rec)
    d.close()


@pytest.mark.parametrize("name,kw", CASES, ids=IDS)
def test_exact_continuation_across_handles(name, kw):
    """Handle A processes x[:, :T1] and exports; handle B (other max_batch, other clock, other state in the target slots)
    imports into permuted slots; both continue bit for bit, and within 1e-5 of the oracle run on the whole signal."""
    nam = _model(name)
    T1, T = 3 * BLOCK, 5 * BLOCK
    x = fx.synthetic_batch(4, T, seed=21)
    a = _dsp(nam, 4, **kw)
    ya = _run(a, x[:, :T1])
    rec = a.export_streams([0, 1, 2, 3])
    b = _dsp(nam, 7, **kw)
    _run(b, fx.synthetic_batch(7, 300, seed=5), 150)  # other audio, other clock
    perm = [2, 0, 3, 1]
    b.import_streams(perm, rec)
    ya2 = _run(a, x[:, T1:])
    xb = np.zeros((4, T - T1), np.float32)
    xb[perm] = x[:, T1:]
    yb = _run(b, xb)
    assert np.array_equal(yb[perm], ya2)
    ref = _oracle(nam, x)
    assert np.max(np.abs(np.concatenate([ya, ya2], axis=1) - ref)) <= TOL
    a.close()
    b.close()


@pytest.mark.parametrize("name", ["wavenet_a1_standard", "a2_full"])
def test_records_move_between_kernels(name):
    """The general kernel's row rings and the fused / model-specialised kernels' plane rings exchange records both ways."""
    nam = _model(name)
    T1, T = 2 * BLOCK, 4 * BLOCK
    x = fx.synthetic_batch(3, T, seed=8)
    ref = _oracle(nam, x)
    for src_kw, dst_kw in (({"kernel_geometry": 4}, {"jit": 1}), ({"jit": 1}, {"kernel_geometry": 4}),
                           ({"kernel_geometry": 4}, {"jit": 2})):
        src = _dsp(nam, 3, **src_kw)
        y1 = _run(src, x[:, :T1])
        dst = _dsp(nam, 3, **dst_kw)
        _run(dst, fx.synthetic_batch(3, 100, seed=2), 100)
        dst.import_streams([0, 1, 2], src.export_streams([0, 1, 2]))
        y2 = _run(dst, x[:, T1:])
        err = np.max(np.abs(np.concatenate([y1, y2], axis=1) - ref))
        assert err <= TOL, f"{src_kw} -> {dst_kw}: {err:.3e}"
        src.close()
        dst.close()


@pytest.mark.parametrize("name", ["wavenet", "wavenet_a2_max", "convnet", "linear"])
def test_reset_streams_touches_only_the_listed_streams(name):
    nam = _model(name)
    B = 20
    x, y = fx.synthetic_batch(B, 600, seed=3), fx.synthetic_batch(B, 400, seed=4)
    d, ctrl, fresh = _dsp(nam, B), _dsp(nam, B), _dsp(nam, B)
    _run(d, x)
    _run(ctrl, x)
    d.reset_streams([3, 17])
    got, want, new = _run(d, y), _run(ctrl, y), _run(fresh, y)
    others = [s for s in range(B) if s not in (3, 17)]
    assert np.array_equal(got[others], want[others])
    assert np.array_equal(got[[3, 17]], new[[3, 17]])
    for h in (d, ctrl, fresh):
        h.close()


def test_reset_streams_lstm_keeps_or_restarts_the_running_state():
    """LSTM Reset keeps h, c and prewarms on top (fresh=False: the oracle's reset() after the same history);
    fresh=True is a new instance."""
    nam = _model("lstm")
    B = 20
    x, y = fx.synthetic_batch(B, 600, seed=3), fx.synthetic_batch(B, 400, seed=4)
    for fresh in (False, True):
        d, ctrl = _dsp(nam, B), _dsp(nam, B)
        _run(d, x)
        _run(ctrl, x)
        d.reset_streams([3, 17], fresh=fresh)
        got, want = _run(d, y), _run(ctrl, y)
        others = [s for s in range(B) if s not in (3, 17)]
        assert np.array_equal(got[others], want[others])
        for s in (3, 17):
            m = oracle.OracleModel.from_dict(nam)
            m.reset(48000.0, BLOCK)
            if not fresh:
                m.run(x[s], BLOCK)
                m.reset(48000.0, BLOCK)  # keeps h, c; prewarms on top
            ref = m.run(y[s], BLOCK)
            m.close()
            assert np.max(np.abs(got[s] - ref)) <= TOL, (fresh, s)
        d.close()
        ctrl.close()


@pytest.mark.parametrize("name", ["wavenet", "wavenet_a2_max", "linear", "lstm"])
def test_copy_streams_and_swap(name):
    nam = _model(name)
    B = 6
    x, y = fx.synthetic_batch(B, 500, seed=6), fx.synthetic_batch(B, 300, seed=7)
    d, ctrl = _dsp(nam, B), _dsp(nam, B)
    _run(d, x)
    _run(ctrl, x)
    d.copy_streams([1], [4])
    d.copy_streams([2, 3], [3, 2])  # swap
    y2 = y.copy()
    y2[4], y2[2], y2[3] = y[1], y[3], y[2]
    got, want = _run(d, y2), _run(ctrl, y)
    for s_got, s_want in ((0, 0), (1, 1), (4, 1), (2, 3), (3, 2), (5, 5)):
        assert np.array_equal(got[s_got], want[s_want]), (s_got, s_want)
    d.close()
    ctrl.close()


@pytest.mark.parametrize("name,paused_calls", [("wavenet", 3), ("wavenet_a1_standard", 2), ("wavenet_a2_max", 3),
                                               ("linear", 3), ("linear", 2)])
def test_stream_that_sat_out_calls_exports_at_its_own_clock(name, paused_calls):
    nam = _model(name)
    B, k = 6, 2
    x0 = fx.synthetic_batch(B, 500, seed=9)
    d = _dsp(nam, B)
    _run(d, x0)
    for c in range(paused_calls):
        _run(d, fx.synthetic_batch(k, 200, seed=10 + c))  # streams >= k sit out
    rec = d.export_streams([4])
    h = _dsp(nam, 1)
    h.import_streams([0], rec)
    y = fx.synthetic_batch(1, 400, seed=11)
    got = _run(h, y)
    ref = _oracle(nam, np.concatenate([x0[4:5], y], axis=1))[:, 500:]
    assert np.max(np.abs(got - ref)) <= TOL
    d.close()
    h.close()


def test_prewarm_after_import_prewarms_every_stream():
    """A standalone prewarm after an import must prewarm each stream from its own state (no broadcast of stream 0)."""
    nam = _model("wavenet")
    x, y = fx.synthetic_batch(3, 500, seed=12), fx.synthetic_batch(3, 300, seed=13)
    a = _dsp(nam, 3, prewarm=False)
    _run(a, x)
    b = _dsp(nam, 3, prewarm=False)
    b.import_streams([0, 1, 2], a.export_streams([0, 1, 2]))
    a.prewarm()
    b.prewarm()
    ya, yb = _run(a, y), _run(b, y)
    assert np.array_equal(ya, yb)
    assert not np.array_equal(yb[0], yb[1])
    a.close()
    b.close()


def test_low_latency_single_stream_continues_after_import():
    """One stream, the plugin protocol (Reset(48000, 64), 64-frame DSP::process calls: the low-latency kernel)."""
    nam = _model("wavenet_a1_standard")
    x = fx.synthetic_batch(1, 64 * 24, seed=14)[0]
    T1 = 64 * 10

    def run(d, sig):
        out = []
        for p in range(0, len(sig), 64):
            o = np.zeros(64, np.float32)
            d.process([np.ascontiguousarray(sig[p:p + 64])], [o], 64)
            out.append(o)
        return np.concatenate(out)

    a = _dsp(nam, 1, 64, jit=3)
    y1 = run(a, x[:T1])
    b = _dsp(nam, 1, 64, jit=3)
    run(b, fx.synthetic_batch(1, 64 * 3, seed=15)[0])
    b.import_streams([0], a.export_streams([0]))
    ya, yb = run(a, x[T1:]), run(b, x[T1:])
    assert np.array_equal(ya, yb)
    ref = _oracle(nam, x[None, :], 64)[0]
    assert np.max(np.abs(np.concatenate([y1, ya]) - ref)) <= TOL
    a.close()
    b.close()


def test_record_of_another_slimmable_size_is_refused():
    nam = fx.load_model("slimmable_wavenet")
    d = nb.get_dsp(nam, batch=2)
    d.SetSlimmableSize(0.0)
    d.Reset(48000.0, BLOCK)
    _run(d, fx.synthetic_batch(2, 300, seed=16))
    small = d.export_streams([0, 1])
    d.import_streams([1, 0], small)  # same size: accepted
    d.SetSlimmableSize(1.0)
    assert d.state_record_bytes == nb.state_layout(nam)["record_bytes"] > small.shape[1]
    n0 = d.launch_count()
    with pytest.raises(ValueError, match="smaller than the record"):
        d.import_streams([0, 1], small)
    padded = np.zeros((2, d.state_record_bytes), np.uint8)  # the small records in slots of the full size's stride
    padded[:, :small.shape[1]] = small
    with pytest.raises(ValueError, match=r"record 0 \(stream 0\): payload float count"):
        d.import_streams([0, 1], padded)
    assert d.launch_count() == n0
    d.close()


def test_fast_tanh_and_handle_options_are_not_part_of_the_record():
    nam = _model("wavenet")
    a = _dsp(nam, 2, fast_tanh=True, jit=2)
    _run(a, fx.synthetic_batch(2, 300, seed=17))
    rec = a.export_streams([0, 1])
    fp = int(np.frombuffer(rec[0, 24:32].tobytes(), "<u8")[0])
    assert fp == nb.state_layout(nam)["fingerprint"]
    b = _dsp(nam, 9, fast_tanh=False, kernel_geometry=4)
    b.import_streams([8, 0], rec)
    assert np.array_equal(b.export_streams([8, 0]), rec)
    a.close()
    b.close()


def test_device_records_match_host_records():
    torch = pytest.importorskip("torch")
    nam = _model("wavenet_a1_standard")
    d = _dsp(nam, 8)
    _run(d, fx.synthetic_batch(8, 600, seed=18))
    host = d.export_streams([7, 1, 5])
    rb = d.state_record_bytes
    stride = rb + 64
    buf = torch.zeros(3 * stride, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    side = torch.cuda.Stream()  # the device variants run asynchronously on a caller's stream
    s = side.cuda_stream
    d.export_streams_device([7, 1, 5], buf.data_ptr(), stride, s)
    torch.cuda.synchronize()
    dev = buf.view(3, stride)[:, :rb].cpu().numpy()
    assert np.array_equal(dev, host)
    d.import_streams_device([0, 2, 3], buf.data_ptr(), stride, s)
    torch.cuda.synchronize()
    assert np.array_equal(d.export_streams([0, 2, 3]), host)
    bad = buf.clone()
    bad[1 * stride + 24] ^= 1  # record 1's fingerprint
    n0 = d.launch_count()
    with pytest.raises(ValueError, match=r"record 1 \(stream 2\).*fingerprint"):
        d.import_streams_device([0, 2, 3], bad.data_ptr(), stride, s)
    assert d.launch_count() == n0
    d.close()


def test_refusals_are_checked_before_any_launch():
    nam = _model("wavenet")
    d = nb.get_dsp(nam, batch=4)
    with pytest.raises(RuntimeError, match="before reset"):
        d.export_streams([0])
    with pytest.raises(RuntimeError, match="before reset"):
        d.reset_streams([0])
    d.Reset(48000.0, BLOCK)
    _run(d, fx.synthetic_batch(4, 300, seed=19))
    rec = d.export_streams([0, 1])
    n0 = d.launch_count()
    with pytest.raises(ValueError, match=r"streams\[1\] = 4: stream index outside"):
        d.export_streams([0, 4])
    with pytest.raises(ValueError, match=r"streams\[0\] = -1"):
        d.reset_streams([-1])
    with pytest.raises(ValueError, match=r"streams\[1\] = 2: duplicate destination"):
        d.import_streams([2, 2], rec)
    with pytest.raises(ValueError, match=r"dst\[1\] = 0: duplicate destination"):
        d.copy_streams([1, 2], [0, 0])
    with pytest.raises(ValueError, match="duplicate destination"):
        d.reset_streams([3, 3])
    # a short stride, through the C ABI directly
    import ctypes as C

    s = np.array([0], np.int32)
    buf = np.zeros(d.state_record_bytes, np.uint8)
    rc = d._lib.nam_b200_import_streams(d._h, s.ctypes.data_as(C.POINTER(C.c_int32)), 1, buf.ctypes.data_as(C.c_void_p),
                                        d.state_record_bytes - 4)
    assert rc == nb.dsp.ERR_INVALID_ARGUMENT and b"record_stride" in d._lib.nam_b200_last_error()
    # corrupted headers
    for offset, field in ((0, "magic"), (4, "version"), (8, "architecture"), (16, "payload"), (24, "fingerprint")):
        bad = rec.copy()
        bad[1, offset] ^= 0x5A
        with pytest.raises(ValueError, match=rf"record 1 \(stream 3\): .*{field}"):
            d.import_streams([2, 3], bad)
    # a record of another model with the same shape (other weights)
    other = fx.random_wavenet(channels=(2, 2), dilations=[[1, 2], [4]], seed=1)
    again = fx.random_wavenet(channels=(2, 2), dilations=[[1, 2], [4]], seed=2)
    o = _dsp(other, 1)
    g = _dsp(again, 1)
    with pytest.raises(ValueError, match="fingerprint"):
        g.import_streams([0], o.export_streams([0]))
    with pytest.raises(ValueError, match="payload"):
        d.import_streams([0], _dsp(_model("wavenet_a1_standard"), 1).export_streams([0]))
    assert d.launch_count() == n0
    for h in (d, o, g):
        h.close()
