"""GPU parity of the model-specialised kernel (csrc/wavenet_spec.cuh: the model compiled by NVRTC at load time, weights
as FFMA immediates, history staged by cp.async.bulk): against the CPU oracle (<= 1e-5 max-abs, BASELINE.json) and, bit
for bit, against the precompiled fused kernel that serves the same rings.

`jit=1` makes the specialised kernel mandatory (creation fails otherwise); `tile_mode=2` keeps small test batches off
the lock-step mode so that every long call really takes the specialised kernel.
"""
import numpy as np
import pytest

import neuralampmodelercore_b200 as nb
from oracle import oracle
from tests import nam_fixtures as fx

pytestmark = pytest.mark.gpu

TOL = 1e-5


def _spec(nam, batch, fast, **kw):
    d = nb.get_dsp(nam, batch=batch, fast_tanh=fast, jit=1, tile_mode=2, **kw)
    assert d.jit_state == 1, d.jit_note()
    return d


def _oracle_batch(nam, x, fast, block=64):
    proto = oracle.OracleModel.from_dict(nam, fast_tanh=fast)
    proto.reset(48000.0, block)
    return proto.run_batch(x, block)


@pytest.mark.parametrize("fast", [False, True], ids=["exact_tanh", "fast_tanh"])
def test_a1_standard_vs_oracle_and_vs_fused_kernel(fast):
    nam = fx.load_model("wavenet_a1_standard")
    B, N = 16, 3000  # 5 full 512-frame tiles + a partial one
    x = fx.synthetic_batch(B, N, seed=11)
    ref = _oracle_batch(nam, x, fast)
    d = _spec(nam, B, fast)
    d.Reset(48000.0, N)
    n0 = d.launch_count()
    got = d.process_batch(x)
    assert d.launch_count() == n0 + 1
    d.close()
    err = float(np.max(np.abs(got - ref)))
    assert err <= TOL, f"max-abs vs oracle {err:.3e}"
    g = nb.get_dsp(nam, batch=B, fast_tanh=fast, jit=2, tile_mode=2)
    assert g.jit_state == 0
    g.Reset(48000.0, N)
    fused = g.process_batch(x)
    g.close()
    # same summation order, same operations: with the library tanh the two kernels agree to the last bit; the packed
    # rational fast-tanh comes out of the two compilers (nvcc for the library, NVRTC for the model) one ulp apart in places
    d_fused = float(np.max(np.abs(got - fused)))
    assert (d_fused <= 2.5e-7) if fast else np.array_equal(got, fused), f"max-abs vs fused kernel {d_fused:.3e}"


def test_call_splitting_and_mixed_kernels_on_one_handle():
    """Long calls (specialised kernel), 64-frame calls (multi-stream geometry of the precompiled kernel), odd lengths
    (the absolute frame counter becomes odd, ring pieces wrap): all on the same rings, equal to one oracle run."""
    nam = fx.load_model("wavenet_a1_standard")
    B, N = 32, 6001
    x = fx.synthetic_batch(B, N, seed=5)
    ref = _oracle_batch(nam, x, True)
    d = _spec(nam, B, True)
    d.Reset(48000.0, 2048)
    chunks = [700, 64, 1, 2048, 63, 513, 64, 999, 1500, 49]
    assert sum(chunks) == N
    out, pos = [], 0
    for n in chunks:
        out.append(d.process_batch(np.ascontiguousarray(x[:, pos:pos + n])))
        pos += n
    d.close()
    got = np.concatenate(out, axis=1)
    err = float(np.max(np.abs(got - ref)))
    assert err <= TOL, f"max-abs {err:.3e}"


@pytest.mark.parametrize("case", [
    dict(channels=(16, 8), kernel_size=3, dilations=[[1, 2, 4, 8, 16, 32], [1, 3, 9, 27, 81]], activation="Tanh", head_scale=1.5),
    dict(channels=(8, 4), kernel_sizes=[[2, 3, 4, 5], [5, 2, 3]], dilations=[[1, 7, 13, 64], [2, 5, 128]], activation="ReLU",
         head_scale=5.0),
    dict(channels=(12, 6), kernel_size=3, dilations=[[1, 2, 4, 300], [1, 2, 512]], activation="Sigmoid",
         head_scale=40.0),  # padded channels
    dict(channels=(3,), kernel_size=3, dilations=[[1, 2, 8]], activation="Hardtanh", head_scale=12.5),  # one array, like wavenet.nam's first
    dict(channels=(16,), kernel_sizes=[[1, 3, 1, 2]], dilations=[[1, 1, 5, 1024]], activation="SiLU",
         head_scale=2.0),  # kernel-size-1 layers: no history
    dict(channels=(4, 16), kernel_size=4, dilations=[[1, 2], [3, 100, 341]], activation="LeakyReLU", head_scale=2.5),  # look-back 1023
], ids=["a1_like_odd_dilations", "kernels_2_to_5", "padded_12_6", "single_array", "kernel_1_layers", "narrow_then_wide"])
def test_shape_family(case):
    B, N = 8, 1400
    x = 4.0 * fx.synthetic_batch(B, N, seed=2)  # with each case's head_scale: the output's std over time is above 0.1
    nam, offset = fx.centred(fx.random_wavenet(seed=3, **case), x)
    ref = _oracle_batch(nam, x, False)
    assert np.min(np.std(ref, axis=1)) >= 0.1 and np.max(np.abs(ref)) <= 4.0
    d = _spec(nam, B, False)
    d.Reset(48000.0, 1024)
    got = np.concatenate([d.process_batch(np.ascontiguousarray(x[:, p:p + 1024])) for p in range(0, N, 1024)], axis=1)
    d.close()
    tol = TOL * max(1.0, float(np.max(np.abs(ref)))) + fx.CENTRED_ROUNDING * abs(offset)
    err = float(np.max(np.abs(got - ref)))
    assert err <= tol, f"max-abs {err:.3e} (tolerance {tol:.2e})"


# the head_scale that puts each model's output std over time above 0.1 (the last head's bias cancels the constant part)
ACTIVATION_SET_HEAD_SCALE = {"Tanh": 14.0, "Hardtanh": 13.0, "Fasttanh": 14.0, "ReLU": 11.0, "LeakyReLU": 12.0, "PReLU": 12.0,
                             "Sigmoid": 58.0, "SiLU": 19.0, "Hardswish": 20.0, "LeakyHardtanh": 13.0, "Softsign": 15.0}


@pytest.mark.parametrize("act", ["Tanh", "Hardtanh", "Fasttanh", "ReLU", "LeakyReLU", "PReLU", "Sigmoid", "SiLU", "Hardswish",
                                 "LeakyHardtanh", "Softsign"])
def test_activation_set(act):
    """All eleven activations of NAM/activations.h:26-39 compiled into the specialised kernel."""
    activation = act
    if act == "PReLU":
        activation = {"type": "PReLU", "negative_slopes": [0.05 * (i + 1) for i in range(8)]}
    elif act == "LeakyHardtanh":
        activation = {"type": "LeakyHardtanh", "min_val": -0.5, "max_val": 0.7, "min_slope": 0.1, "max_slope": 0.2}
    elif act == "LeakyReLU":
        activation = {"type": "LeakyReLU", "negative_slope": 0.2}
    B, N = 4, 700
    x = fx.synthetic_batch(B, N, seed=8) * 4.0  # drive the saturating activations into both branches
    nam, offset = fx.centred(fx.random_wavenet(channels=(8,), kernel_size=3, dilations=[[1, 2, 4]], activation=activation,
                                               seed=9, head_scale=ACTIVATION_SET_HEAD_SCALE[act]), x)
    ref = _oracle_batch(nam, x, False)
    assert np.min(np.std(ref, axis=1)) >= 0.1 and np.max(np.abs(ref)) <= 4.0  # the output follows the input
    d = _spec(nam, B, False)
    d.Reset(48000.0, N)
    got = d.process_batch(x)
    d.close()
    tol = TOL * max(1.0, float(np.max(np.abs(ref)))) + fx.CENTRED_ROUNDING * abs(offset)
    assert float(np.max(np.abs(got - ref))) <= tol


def test_prewarmed_state_and_second_reset():
    """Reset prewarms through the precompiled kernels (short blocks); the specialised kernel continues from that state,
    and a second Reset returns to it."""
    nam = fx.load_model("wavenet_a1_standard")
    x = fx.synthetic_batch(4, 2000, seed=1)
    ref = _oracle_batch(nam, x, True)
    d = _spec(nam, 4, True)
    for _ in range(2):
        d.Reset(48000.0, 2000)
        got = d.process_batch(x)
        assert float(np.max(np.abs(got - ref))) <= TOL
    d.close()


@pytest.mark.parametrize("name", ["wavenet_a2_max", "wavenet_condition_dsp"])
@pytest.mark.parametrize("fast", [False, True], ids=["exact_tanh", "fast_tanh"])
def test_general_kernel_compiled_per_model(name, fast):
    """WaveNets outside the fused family (gated / blended activations, FiLM, groups, head1x1, condition_dsp, post-stack head)
    run on the general kernel; with jit it is compiled for the model (wavenet_generic_spec.cuh: the descriptors and weights as
    constant data, the whole network unrolled)."""
    nam = fx.load_model(name)
    B, N = 70, 1500
    x = fx.synthetic_batch(B, N, seed=19)
    ref = _oracle_batch(nam, x, fast)
    d = nb.get_dsp(nam, batch=B, fast_tanh=fast, jit=1)
    assert d.jit_state == 1 and "general kernel" in d.jit_note(), d.jit_note()
    d.Reset(48000.0, 600)
    got = np.concatenate([d.process_batch(np.ascontiguousarray(x[:, p:p + c])) for p, c in ((0, 600), (600, 1), (601, 299), (900, 600))], axis=1)
    d.close()
    scale = max(1.0, float(np.max(np.abs(ref))))
    err = float(np.max(np.abs(got - ref)))
    assert err <= TOL * scale, f"max-abs {err:.3e} (|y| up to {scale:.1f})"


@pytest.mark.parametrize("name", ["a2_full", "a2_lite"])
@pytest.mark.parametrize("fast", [False, True], ids=["exact_tanh", "fast_tanh"])
def test_a2_family_convolutional_head(name, fast):
    """The A2 family (23 layers of 8 / 3 channels, kernel sizes 6 and 15, odd dilations up to 239, head rechannel = a causal
    convolution of kernel size 16 over the head accumulator, model.cpp:397-400,548) compiled into the specialised kernel:
    the head accumulator has its own ring and history window."""
    nam = fx.load_model(name)
    B, N = 6, 2600
    x = fx.synthetic_batch(B, N, seed=13)
    ref = _oracle_batch(nam, x, fast)
    d = _spec(nam, B, fast)
    d.Reset(48000.0, 1024)
    got = np.concatenate([d.process_batch(np.ascontiguousarray(x[:, p:p + c])) for p, c in ((0, 1024), (1024, 513), (1537, 1), (1538, 1024), (2562, 38))], axis=1)
    d.close()
    err = float(np.max(np.abs(got - ref)))
    assert err <= TOL, f"max-abs {err:.3e}"


def test_default_policy_uses_it_for_throughput_handles():
    nam = fx.load_model("wavenet_a1_standard")
    d = nb.get_dsp(nam, batch=256, fast_tanh=True)
    assert d.jit_state == 1, d.jit_note()
    d.close()
    d = nb.get_dsp(nam, batch=1, fast_tanh=True)
    assert d.jit_state == 0
    d.close()


# ---- the model-specialised LSTM kernel (csrc/lstm_spec.cuh) ---------------------------------------------------------------
def _random_lstm(H, nl, seed=4):
    rng = np.random.default_rng(seed)
    n = sum(4 * H * ((1 if l == 0 else H) + H) + 4 * H + 2 * H for l in range(nl)) + H + 1
    return {"version": "0.5.4", "architecture": "LSTM", "config": {"input_size": 1, "hidden_size": H, "num_layers": nl},
            "weights": [float(v) for v in rng.uniform(-0.4, 0.4, n)], "sample_rate": 48000}


def test_lstm_spec_example_model_both_regimes_and_runtime_switch():
    """lstm.nam on one thread per stream: 70 streams (two full warps + a partial one), 64-frame calls; the fast-tanh
    switch is read at run time like the reference (lstm.cpp:48): one handle, both kernels of the cubin."""
    nam = fx.load_model("lstm")
    x = fx.synthetic_batch(70, 1999, seed=9)
    for geometry in (1, 2):
        _lstm_example_both_regimes(nam, x, geometry)


def _lstm_example_both_regimes(nam, x, geometry):
    d = nb.get_dsp(nam, batch=70, fast_tanh=False, jit=1, kernel_geometry=geometry)
    assert d.jit_state == 1, d.jit_note()
    for fast in (False, True):
        proto = oracle.OracleModel.from_dict(nam, fast_tanh=fast)
        proto.reset(48000.0, 64)
        ref = proto.run_batch(x, 64)
        d.set_fast_tanh(fast)
        d.Reset(48000.0, 64)
        got = np.concatenate([d.process_batch(np.ascontiguousarray(x[:, p:p + 64])) for p in range(0, 1999, 64)], axis=1)
        err = float(np.max(np.abs(got - ref)))
        assert err <= TOL, f"fast={fast}: {err:.3e}"
    d.close()


@pytest.mark.parametrize("geometry", [1, 2], ids=["gate_split", "thread_per_stream"])
@pytest.mark.parametrize("H,nl", [(1, 1), (3, 1), (3, 3), (5, 2), (8, 1)])
def test_lstm_spec_random_cells(H, nl, geometry):
    """Both mappings of lstm_spec.cuh: four lanes per stream (lane = gate, kernel_geometry 1) and one thread per stream (2)."""
    nam = _random_lstm(H, nl)
    x = fx.synthetic_batch(37, 1000, seed=1)
    proto = oracle.OracleModel.from_dict(nam)
    proto.reset(48000.0, 256)
    ref = proto.run_batch(x, 256)
    d = nb.get_dsp(nam, batch=37, jit=1, kernel_geometry=geometry)
    assert d.jit_state == 1, d.jit_note()
    d.Reset(48000.0, 256)
    got = np.concatenate([d.process_batch(np.ascontiguousarray(x[:, p:p + c])) for p, c in ((0, 1), (1, 31), (32, 256), (288, 33), (321, 256), (577, 256), (833, 167))], axis=1)
    d.close()
    assert float(np.max(np.abs(got - ref))) <= TOL


def test_lstm_spec_refuses_large_cells_loudly():
    with pytest.raises(Exception, match="too large"):
        nb.get_dsp(_random_lstm(16, 1), batch=4, jit=1)
    d = nb.get_dsp(_random_lstm(16, 1), batch=256)  # default policy: falls back to the lane-group kernel
    assert d.jit_state == -1 and "too large" in d.jit_note()
    d.close()


# ---- the low-latency kernel (csrc/wavenet_lat.cuh): few streams, short calls --------------------------------------------
@pytest.mark.parametrize("fast", [False, True], ids=["exact_tanh", "fast_tanh"])
def test_lat_kernel_plugin_protocol(fast, monkeypatch):
    """One stream, Reset(sr, 64), 64-frame process() calls (tools/benchmodel.cpp:116-133) on the model-specialised
    low-latency kernel (NAM_B200_LAT_KERNEL=jit: by default the precompiled wavenet_lat2.cuh takes these calls)."""
    monkeypatch.setenv("NAM_B200_LAT_KERNEL", "jit")
    nam = fx.load_model("wavenet_a1_standard")
    x = fx.synthetic_batch(1, 64 * 40, seed=21)
    ref = _oracle_batch(nam, x, fast)
    d = nb.get_dsp(nam, batch=1, fast_tanh=fast, jit=3)
    d.Reset(48000.0, 64)
    assert d.jit_lat_state == 1, d.jit_note()
    n0 = d.launch_count()
    got = np.concatenate([d.process_batch(np.ascontiguousarray(x[:, p:p + 64])) for p in range(0, x.shape[1], 64)], axis=1)
    assert d.launch_count() == n0 + 40
    d.close()
    err = float(np.max(np.abs(got - ref)))
    assert err <= TOL, f"max-abs {err:.3e}"


@pytest.mark.parametrize("which", ["jit", "precompiled"])
def test_lat_kernel_irregular_short_calls_several_streams_and_mixing(which, monkeypatch):
    """Both low-latency kernels (wavenet_lat.cuh compiled per model / wavenet_lat2.cuh precompiled).  5 streams; call lengths 1..128 (a 128-frame handle: 4 frame warps), odd lengths, and a long call in between that the
    precompiled kernels serve on the same rings."""
    monkeypatch.setenv("NAM_B200_LAT_KERNEL", which)
    nam = fx.load_model("wavenet_a1_standard")
    chunks = [64, 1, 17, 128, 63, 100, 2, 127, 64, 33]
    N = sum(chunks)
    x = fx.synthetic_batch(5, N, seed=4)
    ref = _oracle_batch(nam, x, True)
    d = nb.get_dsp(nam, batch=5, fast_tanh=True, jit=3)
    d.Reset(48000.0, 128)
    assert d.jit_lat_state == 1, d.jit_note()
    out, pos = [], 0
    for n in chunks:
        out.append(d.process_batch(np.ascontiguousarray(x[:, pos:pos + n])))
        pos += n
    d.close()
    err = float(np.max(np.abs(np.concatenate(out, axis=1) - ref)))
    assert err <= TOL, f"max-abs {err:.3e}"
    # the same handle type with a larger maxBufferSize has no low-latency kernel and still matches
    d = nb.get_dsp(nam, batch=5, fast_tanh=True, jit=3)
    d.Reset(48000.0, 512)
    assert d.jit_lat_state == 0
    got = np.concatenate([d.process_batch(np.ascontiguousarray(x[:, p:p + 512])) for p in range(0, N, 512)], axis=1)
    d.close()
    assert float(np.max(np.abs(got - ref))) <= TOL


@pytest.mark.parametrize("case", [
    dict(channels=(16, 8), kernel_size=3, dilations=[[1, 2, 4, 8, 16, 32, 64], [1, 3, 9, 27, 81, 200]], activation="Tanh",
         head_scale=1.5),
    dict(channels=(8, 4), kernel_sizes=[[2, 3, 4, 5], [5, 1, 3]], dilations=[[1, 7, 13, 64], [2, 5, 128]], activation="ReLU",
         head_scale=8.0),
    dict(channels=(4, 16), kernel_size=3, dilations=[[1, 2], [3, 100, 341]], activation={"type": "PReLU", "negative_slopes": [0.02 * (i + 1) for i in range(16)]},
         head_scale=1.5),
    dict(channels=(12,), kernel_size=3, dilations=[[1, 2, 40]], activation="Sigmoid", head_scale=21.0),
], ids=["a1_like", "kernels_1_to_5", "prelu_slices", "single_padded_array"])
@pytest.mark.parametrize("which", ["jit", "precompiled"])
def test_lat_kernel_shape_family(case, which, monkeypatch):
    monkeypatch.setenv("NAM_B200_LAT_KERNEL", which)
    case = dict(case)
    act = case.pop("activation")
    if isinstance(act, dict) and act["type"] == "PReLU":
        # per-array slope counts differ: use a shared slope list sized for the widest array only where it applies
        act = {"type": "PReLU", "negative_slopes": [0.05]}
    x = 4.0 * fx.synthetic_batch(3, 64 * 12, seed=2)  # with each case's head_scale: the output's std over time is above 0.1
    nam, offset = fx.centred(fx.random_wavenet(seed=6, activation=act, **case), x)
    ref = _oracle_batch(nam, x, False)
    assert np.min(np.std(ref, axis=1)) >= 0.1 and np.max(np.abs(ref)) <= 4.0
    d = nb.get_dsp(nam, batch=3, jit=3)
    d.Reset(48000.0, 64)
    assert d.jit_lat_state == 1, d.jit_note()
    got = np.concatenate([d.process_batch(np.ascontiguousarray(x[:, p:p + 64])) for p in range(0, x.shape[1], 64)], axis=1)
    d.close()
    tol = TOL * max(1.0, float(np.max(np.abs(ref)))) + fx.CENTRED_ROUNDING * abs(offset)
    err = float(np.max(np.abs(got - ref)))
    assert err <= tol, f"max-abs {err:.3e} (tolerance {tol:.2e})"


def test_short_call_variant_many_streams():
    """64-frame process() calls on many streams (the reference's calling convention at scale): 8 streams x 64 frames per
    CTA of the specialised kernel, ring columns read directly.  37 streams (the last CTA is partly empty), call lengths
    64 / 17 / 1 / 33, a long call in between (throughput kernel, same rings)."""
    nam = fx.load_model("wavenet_a1_standard")
    chunks = [64] * 6 + [17, 64, 1, 64, 33, 700, 64, 64, 5]
    N = sum(chunks)
    x = fx.synthetic_batch(37, N, seed=31)
    ref = _oracle_batch(nam, x, True)
    d = _spec(nam, 37, True)
    d.Reset(48000.0, 1024)
    out, pos = [], 0
    for n in chunks:
        out.append(d.process_batch(np.ascontiguousarray(x[:, pos:pos + n])))
        pos += n
    d.close()
    err = float(np.max(np.abs(np.concatenate(out, axis=1) - ref)))
    assert err <= TOL, f"max-abs {err:.3e}"


@pytest.mark.parametrize("name", ["wavenet_a1_standard", "wavenet"])
def test_short_call_variants_for_128_and_256_frame_calls(name):
    """Calls of 65..128 and 129..256 frames take the 128- / 256-frame entry points (3-4 / 2 streams per CTA); mixed with 64-frame
    and long calls on the same rings, odd lengths, a stream count that leaves the last CTA partly empty; one launch per call."""
    nam = fx.load_model(name)
    chunks = [128, 128, 100, 65, 256, 256, 129, 200, 64, 128, 1000, 256, 77, 128, 3]
    N = sum(chunks)
    B = 23
    x = fx.synthetic_batch(B, N, seed=41)
    ref = _oracle_batch(nam, x, True)
    d = _spec(nam, B, True)
    d.Reset(48000.0, 1024)
    out, pos = [], 0
    n0 = d.launch_count()
    for n in chunks:
        out.append(d.process_batch(np.ascontiguousarray(x[:, pos:pos + n])))
        pos += n
    assert d.launch_count() == n0 + len(chunks)
    d.close()
    scale = max(1.0, float(np.max(np.abs(ref))))
    err = float(np.max(np.abs(np.concatenate(out, axis=1) - ref)))
    assert err <= TOL * scale, f"max-abs {err:.3e}"


def test_reserved_sms_change_the_grid_not_the_result():
    """nam_b200_set_reserved_sms: the persistent kernels walk the streams with fewer CTAs; same outputs bit for bit, and the
    setting can change between calls on live rings."""
    nam = fx.load_model("wavenet_a1_standard")
    B, N = 700, 1024  # more streams than CTAs, so the stride of the persistent loop really changes
    x = fx.synthetic_batch(B, 2 * N, seed=23)
    d = _spec(nam, B, True)
    d.Reset(48000.0, N)
    a = np.concatenate([d.process_batch(x[:, :N]), d.process_batch(x[:, N:])], axis=1)
    d.Reset(48000.0, N)
    d.set_reserved_sms(8)
    b0 = d.process_batch(x[:, :N])
    d.set_reserved_sms(147)
    b1 = d.process_batch(x[:, N:])
    assert np.array_equal(a, np.concatenate([b0, b1], axis=1))
    with pytest.raises(Exception):
        d.set_reserved_sms(-1)
    d.close()


def test_tensor_core_kernel_is_refused_loudly():
    """The sm_90a library has no tensor-core WaveNet kernel: kernel_geometry=3 is refused with a reason."""
    nam = fx.load_model("wavenet_a1_standard")
    assert not nb.has_tensor_core_kernel()
    with pytest.raises(Exception, match="has none"):
        nb.get_dsp(nam, batch=2, kernel_geometry=3)
