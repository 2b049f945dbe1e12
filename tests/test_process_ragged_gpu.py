"""GPU tests of nam_b200_process_streams_ragged_f32 (DSP.process_streams(..., n_frames=[...])): every listed stream runs
its own number of frames in one launch.  The yardstick is a second handle with the same options running one
process_streams call per distinct length; outputs and records must match it byte for byte, and each stream must match
the oracle fed that stream's own chunks."""
import ctypes as C

import numpy as np
import pytest

import neuralampmodelercore_b200 as nb
from tests import nam_fixtures as fx
from tests.test_process_streams_gpu import CASES, IDS, TOL, _dsp, _model, _oracle_stream

pytestmark = pytest.mark.gpu
MAX = 1024  # max_frames of the handles below
# 0, 1, an odd count, tile boundaries +-1 of the 64 / 128 / 512-frame tiles, max_frames
COUNTS = [0, 1, 37, 63, 64, 65, 127, 128, 129, 511, 512, 513, MAX]


def _ragged_signal(counts, ci, seed, pad=0.0):
    """[n, F] (ci == 1) or [n, ci, F] with F = max(counts); frames past a row's count hold `pad`."""
    n, f = len(counts), max(counts) if len(counts) else 0
    x = fx.synthetic_batch(n * ci, max(f, 1), seed=seed)[:, :f].reshape(n, ci, f).copy()
    for i, k in enumerate(counts):
        x[i, :, k:] = pad
    return np.ascontiguousarray(x if ci > 1 else x[:, 0])


def _per_length(d, streams, counts, x):
    """The yardstick: one process_streams call per distinct non-zero length, the outputs assembled zero-padded."""
    y = np.zeros((x.shape[0], d.out_channels, x.shape[-1]) if x.ndim == 3 else x.shape, np.float32)
    for k in sorted(set(counts) - {0}):
        rows = [i for i, c in enumerate(counts) if c == k]
        y[rows, ..., :k] = d.process_streams([streams[i] for i in rows], np.ascontiguousarray(x[rows, ..., :k]))
    return y


def _chunk(x, i, k):
    return np.ascontiguousarray(x[i, ..., :k])


def _run_ragged_schedule(nam, schedule, batch, block=MAX, slim=None, oracle_streams=None, **kw):
    """schedule: list of (streams, counts) on handles of `batch` streams.  Returns the tested handle."""
    a = _dsp(nam, batch, block, slim=slim, **kw)
    b = _dsp(nam, batch, block, slim=slim, **kw)
    ci = a.in_channels
    ins, outs = {}, {}
    for c, (streams, counts) in enumerate(schedule):
        x = _ragged_signal(counts, ci, seed=200 + c)
        y = a.process_streams(streams, x, n_frames=counts)
        ye = _per_length(b, streams, counts, x)
        assert np.array_equal(y, ye), f"call {c}: outputs differ from one process_streams call per length"
        for i, (s, k) in enumerate(zip(streams, counts)):
            assert not np.any(y[i, ..., k:]), f"call {c} row {i}: output padding not zero"
            if k:
                ins.setdefault(s, []).append(_chunk(x, i, k))
                outs.setdefault(s, []).append(_chunk(y, i, k))
    touched = sorted(set(s for st, _ in schedule for s in st))
    assert np.array_equal(a.export_streams(touched), b.export_streams(touched)), "records differ from the yardstick"
    ref_nam = nam if slim is None else next(m for mv, m in nb.submodels(nam) if slim < mv)
    for s in (sorted(ins) if oracle_streams is None else [s for s in oracle_streams if s in ins]):
        ref = _oracle_stream(ref_nam, ins[s], block)
        err = float(np.max(np.abs(np.concatenate(outs[s], axis=-1) - ref)))
        assert err <= TOL, f"stream {s}: {err:.3e} from the oracle"
    b.close()
    return a


def _random_ragged(batch, calls, seed, counts=COUNTS):
    rng = np.random.default_rng(seed)
    out = []
    for c in range(calls):
        k = int(rng.integers(2, batch + 1))
        streams = [int(v) for v in rng.permutation(batch)[:k]]
        n = [int(v) for v in rng.choice(counts, size=k)]
        if max(n) == 0:
            n[0] = counts[-1]
        out.append((streams, n))
    return out


@pytest.mark.parametrize("name,kw", CASES, ids=IDS)
def test_ragged_schedule_matches_per_length_calls_and_the_oracle(name, kw):
    nam = _model(name)
    _run_ragged_schedule(nam, _random_ragged(9, 4, seed=sum(map(ord, name)) + 1), batch=9, **kw).close()


@pytest.mark.parametrize("name,kw", [("wavenet_a1_standard", {"jit": 1}), ("wavenet_a1_standard", {"jit": 2}), ("linear", {}),
                                     ("lstm", {}), ("convnet", {})], ids=["a1-jit1", "a1-jit2", "linear", "lstm", "convnet"])
def test_equal_counts_are_process_streams(name, kw):
    nam = _model(name)
    B = 6
    a, b = _dsp(nam, B, **kw), _dsp(nam, B, **kw)
    for c, streams in enumerate([[4, 1, 0], [0, 1, 2, 3, 4, 5], [5, 2]]):
        x = fx.synthetic_batch(len(streams), 256, seed=30 + c)
        na, nb_ = a.launch_count(), b.launch_count()
        ya = a.process_streams(streams, x, n_frames=[256] * len(streams))
        yb = b.process_streams(streams, x)
        assert np.array_equal(ya, yb)
        assert a.launch_count() - na == b.launch_count() - nb_
    assert np.array_equal(a.export_streams(list(range(B))), b.export_streams(list(range(B))))
    a.close()
    b.close()


def test_fused_and_specialised_short_geometries():
    """n_max of 64 / 128 on many streams: the fused short geometries (jit=2) and the specialised short-call entry points
    (jit=1), sub-tiles of ended streams masked with Tv = 0."""
    nam = _model("wavenet_a1_standard")
    B = 48
    rng = np.random.default_rng(5)
    for jit in (1, 2):
        for n_max in (64, 128):
            pool = [v for v in (0, 1, 31, 33, 63, 64, 65, 127, 128) if v <= n_max]
            sched = []
            for _ in range(3):
                s = [int(v) for v in rng.permutation(B)[:40]]
                n = [int(v) for v in rng.choice(pool, size=40)]
                n[0] = n_max
                sched.append((s, n))
            _run_ragged_schedule(nam, sched, block=n_max, batch=B, oracle_streams=sched[0][0][:4] + sched[1][0][:2],
                                 jit=jit).close()


def test_single_frame_geometry_and_long_persistent(monkeypatch):
    nam = _model("wavenet_a1_standard")
    monkeypatch.setenv("NAM_B200_LAT_KERNEL", "off")  # 128 x 1: few streams, <= 128 frames
    _run_ragged_schedule(nam, [([4, 1], [128, 37]), ([1, 4, 2], [0, 128, 65]), ([2, 0], [1, 127])], block=128, batch=6,
                         jit=2).close()
    monkeypatch.delenv("NAM_B200_LAT_KERNEL")
    # one CTA walking each stream's own tiles (tile_mode 2), both fused geometries
    for kg in (1, 2):
        _run_ragged_schedule(nam, [([0, 1, 2], [4096, 1000, 0]), ([2, 0, 1], [513, 0, 4096]), ([1, 2], [4096, 4096])],
                             block=4096, batch=3, jit=2, tile_mode=2, kernel_geometry=kg).close()


@pytest.mark.parametrize("tile_mode", [0, 1], ids=["lockstep", "wavefront"])
def test_tile_parallel_modes_stop_at_each_streams_tiles(tile_mode):
    """Lock-step and wavefront: a tile past its stream's count has no work and nobody waits on it; a contiguous call
    afterwards (every stream then at its own clock) matches the oracle."""
    nam = _model("wavenet_a1_standard")
    d = _dsp(nam, 3, 4096, jit=2, tile_mode=tile_mode)
    ins = {s: [] for s in range(3)}
    outs = {s: [] for s in range(3)}
    for c, (streams, counts) in enumerate([([0, 1, 2], [4096, 1000, 0]), ([0, 1, 2], [0, 4096, 513])]):
        x = _ragged_signal(counts, 1, seed=300 + c, pad=np.nan)
        y = d.process_streams(streams, x, n_frames=counts)
        for i, (s, k) in enumerate(zip(streams, counts)):
            if k:
                ins[s].append(x[i, :k])
                outs[s].append(y[i, :k])
    x = fx.synthetic_batch(3, 4096, seed=310)
    y = d.process_batch(x)
    for s in range(3):
        ins[s].append(x[s])
        outs[s].append(y[s])
        ref = _oracle_stream(nam, ins[s], 4096)
        err = float(np.max(np.abs(np.concatenate(outs[s]) - ref)))
        assert err <= TOL, f"stream {s}: {err:.3e} from the oracle"
    d.close()


@pytest.mark.parametrize("name,kw", [("wavenet_a2_max", {}), ("wavenet_a1_standard", {"kernel_geometry": 4}),
                                     ("convnet", {}), ("linear", {})], ids=["generic-jit", "generic-precompiled", "convnet",
                                                                           "linear"])
def test_generic_convnet_and_linear_paths(name, kw):
    nam = _model(name)
    sched = [([3, 0, 1], [513, 0, 129]), ([1, 2, 0, 3], [1, 1024, 200, 0]), ([3, 1], [1024, 64])]
    _run_ragged_schedule(nam, sched, batch=4, **kw).close()


@pytest.mark.parametrize("name,kw", [("lstm_h5", {"jit": 1, "kernel_geometry": 1}), ("lstm_h5", {"jit": 1, "kernel_geometry": 2}),
                                     ("lstm", {"jit": 2}), ("lstm_2in_3out", {"jit": 2})],
                         ids=["spec-thread", "spec-4lane", "group", "thread-per-stream"])
def test_lstm_streams_sharing_a_cta_at_different_counts(name, kw):
    """Neighbouring positions share one warp / group CTA / thread-per-stream CTA: counts 0, 1 and 37 next to each other
    and next to longer ones; a stream's h and c freeze at its own count."""
    nam = _model(name)
    B = 40
    counts = [0, 1, 37, 256, 37, 0, 1, 255, 64, 0] * 4
    sched = [(list(range(B)), counts), (list(range(B))[::-1], counts[::-1]), (list(range(0, B, 3)), [37] * len(range(0, B, 3)))]
    _run_ragged_schedule(nam, sched, block=256, batch=B, oracle_streams=list(range(12)), **kw).close()


def test_pipelined_host_path_with_mixed_counts():
    """3,400 streams with mixed counts on a 4,096-stream handle: the chunked host path (at least 2 launches), the
    output staging of each chunk zeroed for the padding."""
    nam = _model("wavenet_a1_standard")
    B, n = 4096, 3400
    rng = np.random.default_rng(12)
    streams = [int(v) for v in rng.permutation(B)[:n]]
    counts = [int(v) for v in rng.choice([0, 1, 513, 2048, 4095, 4096], size=n)]
    d = _dsp(nam, B, 4096)
    x = _ragged_signal(counts, 1, seed=400, pad=np.nan)
    zero = [streams[i] for i, k in enumerate(counts) if k == 0][:4]
    before = d.export_streams(zero)
    n0 = d.launch_count()
    y = d.process_streams(streams, x, n_frames=counts)
    assert d.launch_count() - n0 >= 2
    for i, k in enumerate(counts):
        assert not np.any(y[i, k:]), f"row {i}: padding"
    for i in [0, 1, 2, n // 2, n - 1] + [counts.index(v) for v in (0, 1, 513)]:
        if counts[i]:
            ref = _oracle_stream(nam, [x[i, :counts[i]]], 4096)
            err = float(np.max(np.abs(y[i, :counts[i]] - ref)))
            assert err <= TOL, f"row {i}: {err:.3e} from the oracle"
    assert np.array_equal(d.export_streams(zero), before), "a zero-frame stream changed"
    d.close()


@pytest.mark.parametrize("name,kw", [("wavenet_a1_standard", {"jit": 1}), ("wavenet_a1_standard", {"jit": 2}),
                                     ("lstm", {}), ("linear", {}), ("multichannel", {})],
                         ids=["a1-jit1", "a1-jit2", "lstm", "linear", "multichannel"])
def test_nan_input_padding_changes_nothing(name, kw):
    nam = _model(name)
    B = 5
    a, b = _dsp(nam, B, **kw), _dsp(nam, B, **kw)
    ci = a.in_channels
    for c, (streams, counts) in enumerate([([0, 1, 2, 3, 4], [256, 0, 37, 129, 1]), ([4, 2, 0], [64, 256, 255])]):
        x0 = _ragged_signal(counts, ci, seed=500 + c, pad=0.0)
        xn = _ragged_signal(counts, ci, seed=500 + c, pad=np.nan)
        ya = a.process_streams(streams, x0, n_frames=counts)
        yb = b.process_streams(streams, xn, n_frames=counts)
        assert np.array_equal(ya, yb)
    assert np.array_equal(a.export_streams(list(range(B))), b.export_streams(list(range(B))))
    a.close()
    b.close()


def test_device_entry_leaves_output_padding_untouched():
    torch = pytest.importorskip("torch")
    nam = _model("wavenet_a1_standard")
    B = 8
    a, b = _dsp(nam, B), _dsp(nam, B)
    side = torch.cuda.Stream()
    for c, (streams, counts) in enumerate([([3, 7, 1], [256, 0, 100]), ([7, 0, 3, 5], [1, 256, 129, 0])]):
        x = _ragged_signal(counts, 1, seed=600 + c, pad=np.nan)
        ya = a.process_streams(streams, x, n_frames=counts)
        xin = torch.from_numpy(x).cuda()
        out = torch.full_like(xin, 7.0)
        torch.cuda.synchronize()
        b.process_streams_device(streams, xin.data_ptr(), out.data_ptr(), counts, cuda_stream=side.cuda_stream)
        side.synchronize()
        got = out.cpu().numpy()
        for i, k in enumerate(counts):
            assert np.array_equal(got[i, :k], ya[i, :k])
            assert np.all(got[i, k:] == 7.0), f"call {c} row {i}: output padding written"
            assert not np.any(ya[i, k:])
    assert np.array_equal(a.export_streams(list(range(B))), b.export_streams(list(range(B))))
    a.close()
    b.close()


@pytest.mark.parametrize("name", ["wavenet_a1_standard", "lstm", "linear", "convnet"])
def test_zero_frame_entries_leave_the_stream_exactly_as_it_was(name):
    nam = _model(name)
    B = 3
    d = _dsp(nam, B, 256)
    x0 = fx.synthetic_batch(B, 256, seed=700)
    y0 = d.process_batch(x0)
    before = d.export_streams([1])
    x1 = _ragged_signal([256, 0, 100], 1, seed=701)
    y1 = d.process_streams([0, 1, 2], x1, n_frames=[256, 0, 100])
    assert np.array_equal(d.export_streams([1]), before)
    assert not np.any(y1[1])
    x2 = fx.synthetic_batch(1, 200, seed=702)
    y2 = d.process_streams([1], x2)
    ref = _oracle_stream(nam, [x0[1], x2[0]], 256)
    assert float(np.max(np.abs(np.concatenate([y0[1], y2[0]]) - ref))) <= TOL
    d.close()


def test_refusals_are_caught_on_the_host():
    nam = _model("wavenet")
    d = nb.get_dsp(nam, batch=4)
    lib, h = d._lib, d._h
    s = np.array([0, 1], np.int32)
    sp = s.ctypes.data_as(C.POINTER(C.c_int32))
    buf = np.zeros((2, 256), np.float32)
    vp = buf.ctypes.data_as(C.c_void_p)
    cnt = np.array([256, 100], np.int32)
    cp = cnt.ctypes.data_as(C.POINTER(C.c_int32))
    assert lib.nam_b200_process_streams_ragged_f32(h, sp, 2, cp, vp, vp, 256, 256) == nb.dsp.ERR_STATE
    d.Reset(48000.0, 256)
    d.process_batch(fx.synthetic_batch(4, 256, seed=71))
    before = d.export_streams([0, 1, 2, 3])
    n0 = d.launch_count()

    def refused(counts, streams=(0, 1), in_stride=256, out_stride=256, device=False):
        st = np.array(streams, np.int32)
        stp = st.ctypes.data_as(C.POINTER(C.c_int32))
        c = None if counts is None else np.array(counts, np.int32)
        ptr = None if c is None else c.ctypes.data_as(C.POINTER(C.c_int32))
        if device:
            rc = lib.nam_b200_process_streams_ragged_f32_device(h, stp, len(st), ptr, vp, vp, in_stride, out_stride, None)
        else:
            rc = lib.nam_b200_process_streams_ragged_f32(h, stp, len(st), ptr, vp, vp, in_stride, out_stride)
        assert rc == nb.dsp.ERR_INVALID_ARGUMENT, rc
        return lib.nam_b200_last_error()

    assert b"null n_frames" in refused(None)
    assert b"n_frames[1] = -1" in refused([256, -1])
    assert b"n_frames[0] = 257" in refused([257, 3])
    assert b"in_stride" in refused([256, 3], in_stride=255)
    assert b"out_stride" in refused([3, 256], out_stride=255, device=True)
    assert b"duplicate" in refused([256, 3], streams=(1, 1))
    with pytest.raises(ValueError):
        d.process_streams([0, 1], fx.synthetic_batch(2, 256, seed=72), n_frames=[256, -1])
    with pytest.raises(ValueError):
        d.process_streams([0, 1], fx.synthetic_batch(2, 256, seed=72), n_frames=[200, 100])  # F != max(n_frames)
    assert lib.nam_b200_process_streams_ragged_f32(h, sp, 0, None, None, None, 0, 0) == 0  # no-ops
    z = np.zeros(2, np.int32)
    assert lib.nam_b200_process_streams_ragged_f32(h, sp, 2, z.ctypes.data_as(C.POINTER(C.c_int32)), vp, vp, 0, 0) == 0
    assert d.launch_count() == n0
    assert np.array_equal(d.export_streams([0, 1, 2, 3]), before)
    d.close()


def test_slimmable_container_and_multichannel_forms():
    """A slimmable container at a non-default size forwards the call to its active sub-model; a multi-channel WaveNet
    takes [n, C, F]."""
    _run_ragged_schedule(_model("slimmable_wavenet"), _random_ragged(5, 3, seed=9), batch=5, slim=0.0).close()
    _run_ragged_schedule(_model("multichannel"), _random_ragged(5, 3, seed=10), batch=5).close()
