"""The general WaveNet kernel's and the ConvNet kernel's option cases (tests/general_kernel_cases.py) on the host: the
oracle against the reference build for every case, the kernel each case is served by, the per-model compiled kernel's
compilation, and a refusal one step past each limit of csrc/generic_desc.h, naming the field.

The oracle and the kernels are two readings of NAM/wavenet/model.cpp, film.h, gating_activations.h and convnet.cpp;
the reference build is the only check of a reading they share.  The reference's outputs come from
tests/golden/reference_outputs.npz under general_options/ (nam_fixtures.reference)."""
import copy

import numpy as np
import pytest

import neuralampmodelercore_b200 as nb
from oracle import oracle, ref
from tests import general_kernel_cases as gk
from tests import nam_fixtures as fx

TOL = 1e-5
N, BLOCK, SEED = 4096, 256, 7  # one stream; the long look-back case needs more than 3072 frames to reach its far taps


def _reference_run(case, fast):
    x = gk.signal(case, 1, N, SEED)[0]
    r = ref.ReferenceModel.from_dict(case.nam, fast_tanh=fast)
    r.reset(48000.0, BLOCK)
    y = np.concatenate([r.process_planar(x[:, p:p + BLOCK]) for p in range(0, N, BLOCK)], axis=1)
    r.close()
    return y


def _reference_prewarm(case, fast):
    r = ref.ReferenceModel.from_dict(case.nam, fast_tanh=fast)
    n = r.prewarm_samples
    r.close()
    return np.array([n], np.float32)


def _oracle_run(case, fast):
    x = gk.signal(case, 1, N, SEED)[0]
    m = oracle.OracleModel.from_dict(case.nam, fast_tanh=fast)
    m.reset(48000.0, BLOCK)
    y = np.concatenate([np.atleast_2d(m.process(np.ascontiguousarray(x[:, p:p + BLOCK]))) for p in range(0, N, BLOCK)], axis=1)
    prewarm = m.prewarm_samples
    m.close()
    return y, prewarm


REGIMES = [(c, False) for c in gk.CASES] + [(c, True) for c in gk.CASES if c.has_tanh]


@pytest.mark.parametrize("case,fast", REGIMES, ids=[f"{c.name}-{'fast' if f else 'exact'}_tanh" for c, f in REGIMES])
def test_oracle_matches_the_reference_build(case, fast):
    regime = "fast" if fast else "exact"
    yr = fx.reference(f"general_options/{case.name}/{regime}", lambda: _reference_run(case, fast))
    yo, prewarm = _oracle_run(case, fast)
    assert fx.reference(f"general_options/prewarm_samples/{case.name}/{regime}", lambda: _reference_prewarm(case, fast))[0] == prewarm
    peak = float(np.max(np.abs(yr)))
    assert 1e-3 < peak < 1e2, f"{case.name}: the reference's output peaks at {peak:.3e}"
    err = float(np.max(np.abs(fx.sample(yo) - yr)))
    assert err <= TOL * max(1.0, peak), f"{case.name}: max|reference - oracle| = {err:.3e} (max|y| {peak:.3f})"


@pytest.mark.parametrize("case", gk.CASES, ids=[c.name for c in gk.CASES])
def test_each_case_takes_its_kernel(case):
    info = nb.inspect(case.nam)
    assert info["kernel"] == case.kernel, info
    assert (info["in_channels"], info["out_channels"]) == (oracle.OracleModel.from_dict(case.nam).in_channels,
                                                           oracle.OracleModel.from_dict(case.nam).out_channels)
    # the read-only cases really are past what the kernels stage in shared memory (the packed blob is no smaller than the
    # document's weights), the others within it
    if "read_only" in case.name:
        assert 4 * info["n_weights"] > gk.SMEM_BLOB_BYTES
    else:
        assert 4 * info["n_weights"] < gk.SMEM_BLOB_BYTES


COMPILED = [c for c in gk.CASES if c.compiled]


@pytest.mark.parametrize("case", COMPILED, ids=[c.name for c in COMPILED])
def test_the_compiled_kernel_builds_for_every_compiled_case(case):
    rep = nb.jit_prepare(case.nam, fast_tanh=False)
    assert rep["ok"], rep["why_not"][:2000]
    print(f"{case.name}: compile_seconds {rep['compile_seconds']:.2f} (from cache: {rep['from_cache']})")


def test_the_wavenets_that_are_not_compiled_cases_are_past_the_unroll_cap():
    for case in gk.CASES:
        if case.kernel == "generic" and not case.compiled:
            rep = nb.jit_prepare(case.nam, fast_tanh=False)
            assert not rep["ok"] and "too many weights to unroll" in rep["why_not"], (case.name, rep)


# ---- one past each limit ------------------------------------------------------------------------------------------------
def _gated(**kw):
    return gk._layer(dilations=(1, 2), **kw)


def _refusal(nam) -> str:
    info = nb.inspect(nam)
    assert info["kernel"] == "unsupported", info
    return info["reason"]


@pytest.mark.parametrize("role,layer_kw,config_kw,field", [
    ("channels", dict(channels=65, bottleneck=8), {}, "channels 65"),
    ("bottleneck", dict(channels=16, bottleneck=33), {}, "2 x bottleneck (gated / blended layer) 66"),
    ("head1x1", dict(channels=8, bottleneck=4, head1x1={"active": True, "out_channels": 65, "groups": 1}), {},
     "head1x1 out_channels 65"),
    ("condition", dict(input_size=65, condition_size=65, channels=8, bottleneck=4), {"in_channels": 65}, "input channels 65"),
], ids=["channels", "gated_bottleneck", "head1x1_out", "condition"])
def test_a_width_of_65_is_refused_with_the_field_named(role, layer_kw, config_kw, field):
    nam = gk._wavenet([_gated(**layer_kw)], seed=1, scale=0.1, **config_kw)
    reason = _refusal(nam)
    assert "general kernel: " + field in reason and "handles 1..64" in reason, reason
    rep = nb.jit_prepare(nam, fast_tanh=False)
    assert not rep["ok"] and field in rep["why_not"], rep
    # one less is served
    ok_kw = {k: (v - 1 if isinstance(v, int) and v in (65, 33) else v) for k, v in layer_kw.items()}
    if role == "head1x1":
        ok_kw["head1x1"] = {"active": True, "out_channels": 64, "groups": 1}
    ok_config = {"in_channels": 64} if config_kw else {}
    assert nb.inspect(gk._wavenet([_gated(**ok_kw)], seed=1, scale=0.1, **ok_config))["kernel"] == "generic"


def test_a_condition_dsp_output_of_65_is_refused_as_the_condition_size():
    cond = gk._wavenet([gk._layer(channels=4, bottleneck=4, gating="none", dilations=(1,), head_size=65)], seed=2, scale=0.1)
    nam = gk._wavenet([_gated(condition_size=65, channels=6, bottleneck=3)], seed=3, scale=0.1, condition_dsp=cond)
    assert "condition size 65" in _refusal(nam)


def test_five_arrays_are_refused():
    case = gk.BY_NAME["four_arrays_head_dilation"]
    assert nb.inspect(case.nam)["kernel"] == "generic"
    layers = copy.deepcopy(case.nam["config"]["layers"])
    width = layers[-1]["head"]["out_channels"]  # an array's channels and head accumulator are the previous head's width
    extra = gk._layer(input_size=layers[-1]["channels"], channels=width, bottleneck=width,
                      head1x1={"active": True, "out_channels": width, "groups": 1})
    nam = gk._wavenet(layers + [extra], seed=4, scale=0.3)
    assert "5 layer arrays (general kernel handles 1..4)" in _refusal(nam)


def test_nine_head_convolutions_are_refused():
    case = gk.BY_NAME["post_stack_head_8_convs"]
    assert len(case.nam["config"]["head"]["kernel_sizes"]) == 8 and nb.inspect(case.nam)["kernel"] == "generic"
    head = dict(case.nam["config"]["head"], kernel_sizes=case.nam["config"]["head"]["kernel_sizes"] + [2])
    nam = gk._wavenet(copy.deepcopy(case.nam["config"]["layers"]), seed=5, scale=0.3, head=head)
    assert "post-stack head with 9 convolutions (general kernel handles up to 8)" in _refusal(nam)


def test_49_convnet_blocks_are_refused():
    case = gk.BY_NAME["convnet_48_blocks"]
    assert len(case.nam["config"]["dilations"]) == 48 and nb.inspect(case.nam)["kernel"] == "convnet"
    nam = gk._convnet(4, case.nam["config"]["dilations"] + [1], True, "Tanh", seed=6)
    assert "49 ConvNet blocks (kernel handles up to 48)" in _refusal(nam)


def _at_the_unroll_cap(head_kernel: int) -> dict:
    """a general WaveNet that packs 39,908 + 4 * head_kernel floats: 40,000 with a head kernel of 23, 40,004 (the first
    size past the cap: the blob is a whole number of float4s) with 24.  Five gated layers of 48 channels, bottleneck 24,
    with three FiLMs, and a one-convolution post-stack head whose kernel size sets the last few floats."""
    film = {"active": True, "shift": True, "groups": 1}
    layer = gk._layer(channels=48, bottleneck=24, dilations=(1, 2, 4, 8, 16), kernel_size=[3, 3, 3, 3, 2], gating="gated",
                      head1x1={"active": True, "out_channels": 4, "groups": 1}, head_size=1,
                      activation_post_film=film, head1x1_post_film=film, input_mixin_pre_film=film)
    head = {"in_channels": 1, "channels": 1, "out_channels": 1, "kernel_sizes": [head_kernel], "activation": "Tanh"}
    return gk._wavenet([layer], seed=9, scale=0.05, head=head)


def test_the_unroll_cap():
    """40,000 packed floats compile; 40,004 are refused by jit_prepare before compiling, and the precompiled kernel still
    serves the model"""
    rep = nb.jit_prepare(_at_the_unroll_cap(23), fast_tanh=False)
    assert rep["ok"], rep["why_not"][:2000]
    past = _at_the_unroll_cap(24)
    assert nb.inspect(past)["kernel"] == "generic"
    rep = nb.jit_prepare(past, fast_tanh=False)
    assert not rep["ok"] and rep["why_not"] == "too many weights to unroll (40004)", rep
