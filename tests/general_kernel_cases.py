"""Model builders for the tests of the general WaveNet kernel and the ConvNet kernel (csrc/wavenet_generic.cuh, its per-model
NVRTC form csrc/wavenet_generic_spec.cuh, and convnet_kernel): one seeded .nam per option of the reference's WaveNet and
ConvNet, and one at each limit of csrc/generic_desc.h.  Not a test module: test_general_options_host.py holds the oracle
to the reference build on these cases, test_general_options_gpu.py holds both kernels to the oracle.

Each case's weight scale is chosen so that the model's output is neither near zero nor huge (1e-3 < max|y| < 1e2 on
`signal()`): a comparison of near-zeros proves nothing."""
from __future__ import annotations

import json
from dataclasses import dataclass

import numpy as np

from oracle import nam_config
from tests import nam_fixtures as fx
from tests.test_reference_build import _convnet

# the per-model compiled kernel unrolls every packed weight into an immediate and refuses more than this many
# (csrc/jit_spec.cpp); a "compiled" case is one the compiled kernel takes
UNROLL_CAP = 40000
# the kernels stage a blob of at most this many bytes in shared memory; larger ones are read through the read-only path
SMEM_BLOB_BYTES = 200 * 1024


@dataclass
class Case:
    name: str
    nam: dict
    kernel: str  # what inspect() reports: "generic" or "convnet"
    compiled: bool  # the per-model compiled kernel (jit=1) takes it
    lookback: int = 0  # the longest look-back of any convolution, in frames

    @property
    def has_tanh(self) -> bool:
        """the model has a Tanh activation somewhere, so fast_tanh changes what it computes"""
        return '"Tanh"' in json.dumps(self.nam)

    @property
    def in_channels(self) -> int:
        return int(self.nam["config"].get("in_channels", 1))


def signal(case: Case, streams: int, n: int, seed: int) -> np.ndarray:
    """[streams, in_channels, n]: the synthetic benchmark signal, one row per (stream, channel), at four times its level
    (peaks near 1.5): the saturating activations are driven into both of their branches"""
    ci = case.in_channels
    return np.ascontiguousarray(4.0 * fx.synthetic_batch(streams * ci, n, seed=seed).reshape(streams, ci, n))


def _randomise(nam: dict, seed: int, scale: float, head_scale: float = 0.5) -> dict:
    n = nam_config.expected_weight_count(nam)
    w = np.random.default_rng(seed).uniform(-scale, scale, size=n).astype(np.float32)
    w[-1] = head_scale
    nam["weights"] = [float(v) for v in w]
    return nam


def _film(shift=True, groups=1):
    return {"active": True, "shift": shift, "groups": groups}


def _layer(*, input_size=1, condition_size=1, channels=6, bottleneck=4, dilations=(1, 3, 7), kernel_size=3,
           activation="Tanh", gating="gated", secondary="Sigmoid", head_size=1, head_bias=True, **extra) -> dict:
    n = len(dilations)
    lc = {"input_size": input_size, "condition_size": condition_size, "channels": channels, "bottleneck": bottleneck,
          "head_size": head_size, "head_bias": head_bias, "dilations": list(dilations),
          "activation": activation, "gating_mode": gating}
    if isinstance(kernel_size, (list, tuple)):
        lc["kernel_sizes"] = list(kernel_size)
    else:
        lc["kernel_size"] = kernel_size
    gl = gating if isinstance(gating, list) else [gating] * n
    if any(g != "none" for g in gl):
        lc["secondary_activation"] = secondary
    lc.update(extra)
    return lc


def _wavenet(layers, seed, scale, head_scale=0.5, head=None, **config_extra) -> dict:
    nam = fx.make_wavenet_nam(layers, [], version="0.7.0", **config_extra)
    if head is not None:
        nam["config"]["head"] = head
    return _randomise(nam, seed, scale, head_scale)


def _lookback(nam: dict) -> int:
    lb = 0
    for lc in nam["config"]["layers"]:
        ks = lc.get("kernel_sizes") or [lc["kernel_size"]] * len(lc["dilations"])
        lb = max([lb] + [(k - 1) * d for k, d in zip(ks, lc["dilations"])])
    return lb


def _prelu(n, base=0.05):
    return {"type": "PReLU", "negative_slopes": [round(base * (1 + 2 * i), 4) for i in range(n)]}


LEAKY_HARDTANH = {"type": "LeakyHardtanh", "min_val": -0.6, "max_val": 0.5, "min_slope": 0.08, "max_slope": 0.15}
LEAKY_RELU = {"type": "LeakyReLU", "negative_slope": 0.07}

FILM_SITES = ["conv_pre_film", "conv_post_film", "input_mixin_pre_film", "input_mixin_post_film", "activation_pre_film",
              "activation_post_film", "layer1x1_post_film", "head1x1_post_film"]


def _gating_cases():
    secs = ["Hardswish", "Softsign", "Fasttanh", "SiLU"]
    for mode, order in (("gated", secs), ("blended", secs[::-1])):
        layer = _layer(channels=6, bottleneck=4, dilations=(1, 2, 5, 11, 3), kernel_size=3,
                       gating=[mode] * 4 + ["none"], secondary=order + ["Sigmoid"])
        yield f"{mode}_secondaries", _wavenet([layer], seed=11 if mode == "gated" else 12, scale=0.45)
    # primary activations with parameters, in gated and blended layers: PReLU with one slope per activated channel
    # (the bottleneck rows), LeakyHardtanh, LeakyReLU
    layer = _layer(channels=6, bottleneck=4, dilations=(1, 3, 2, 7, 4, 9), kernel_size=3,
                   activation=[_prelu(4), _prelu(4, 0.08), LEAKY_HARDTANH, LEAKY_HARDTANH, LEAKY_RELU, LEAKY_RELU],
                   gating=["gated", "blended"] * 3, secondary=["Sigmoid", "Softsign", "Hardswish", "Sigmoid", "SiLU", "Sigmoid"])
    yield "parametric_primaries", _wavenet([layer], seed=13, scale=0.5)


def _film_cases():
    # a two-channel input is the condition, so a FiLM can have groups = 2 (its condition -> scale / shift matrix is grouped)
    for i, site in enumerate(FILM_SITES):
        gating = ["blended", "blended", "none"] if site == "layer1x1_post_film" else ["gated", "blended", "none"]
        layer = _layer(input_size=2, condition_size=2, channels=6, bottleneck=4, dilations=(1, 3, 7),
                       gating=gating, secondary="Sigmoid", head1x1={"active": True, "out_channels": 6, "groups": 1},
                       **{site: _film(shift=True, groups=2)})
        yield f"film_{site}", _wavenet([layer], seed=30 + i, scale=0.45, in_channels=2)
    # layer1x1_post_film in a gated (and a plain) layer: the reference applies it in blended layers only
    layer = _layer(input_size=2, condition_size=2, channels=6, bottleneck=4, dilations=(1, 3, 7),
                   gating=["gated", "none", "gated"], layer1x1_post_film=_film(shift=True, groups=2))
    yield "film_layer1x1_post_in_gated_layers", _wavenet([layer], seed=40, scale=0.45, in_channels=2)


def _grouping_cases():
    layer = _layer(channels=8, bottleneck=4, dilations=(1, 4, 2), gating=["gated", "blended", "none"],
                   groups_input=2, secondary="Softsign")
    yield "groups_input_2", _wavenet([layer], seed=50, scale=0.45)
    layer = _layer(input_size=2, condition_size=2, channels=8, bottleneck=4, dilations=(1, 4, 2, 6),
                   gating=["gated", "blended", "none", "gated"], groups_input=4, groups_input_mixin=2,
                   layer1x1={"active": True, "groups": 2}, head1x1={"active": True, "out_channels": 6, "groups": 2})
    yield "groups_input_4_mixin_layer1x1_head1x1", _wavenet([layer], seed=51, scale=0.45, in_channels=2)
    layer = _layer(channels=5, bottleneck=5, dilations=(1, 2, 4, 8), gating=["gated", "none", "blended", "none"],
                   layer1x1={"active": False, "groups": 1}, head_size=3)
    a1 = _layer(input_size=5, channels=3, bottleneck=3, dilations=(1, 3), gating="none", activation="Tanh")
    yield "layer1x1_inactive", _wavenet([layer, a1], seed=52, scale=0.45)
    layer = _layer(channels=6, bottleneck=4, dilations=(1, 1, 3, 1, 5), kernel_size=[1, 3, 1, 4, 2],
                   gating=["gated", "none", "blended", "gated", "none"])
    yield "kernel_size_1_layers", _wavenet([layer], seed=53, scale=0.45)


def _limit_cases():
    # four arrays of different widths, A2-style head convolutions (kernel size > 1, head_dilation) between them
    widths, heads = [3, 8, 5, 2], [(8, 3, 2), (5, 2, 3), (2, 3, 1), (1, 4, 2)]  # (out_channels, kernel_size, head_dilation)
    arrays = []
    for a, (c, (ho, hk, hd)) in enumerate(zip(widths, heads)):
        lc = _layer(input_size=1 if a == 0 else widths[a - 1], channels=c, bottleneck=c,
                    dilations=(1, 2 + a, 5), gating=["gated", "none", "blended"], secondary="Softsign")
        del lc["head_size"], lc["head_bias"]
        lc["head"] = {"out_channels": ho, "kernel_size": hk, "bias": a % 2 == 1, "head_dilation": hd}
        if a:  # the head accumulator an array adds into is the previous array's head output
            lc["head1x1"] = {"active": True, "out_channels": heads[a - 1][0], "groups": 1}
        arrays.append(lc)
    yield "four_arrays_head_dilation", _wavenet(arrays, seed=60, scale=0.4)
    layer = _layer(channels=6, bottleneck=3, dilations=(1, 3), head_size=4, gating=["gated", "blended"])
    head = {"in_channels": 4, "channels": 5, "out_channels": 1, "kernel_sizes": [3, 2, 1, 4, 2, 3, 1, 2], "activation": "LeakyReLU"}
    yield "post_stack_head_8_convs", _wavenet([layer], seed=61, scale=0.9, head=head)
    layer = _layer(channels=64, bottleneck=32, dilations=(1,), kernel_size=2, gating="gated",
                   head1x1={"active": True, "out_channels": 64, "groups": 1}, head_size=1)
    yield "width_64", _wavenet([layer], seed=62, scale=0.3)


def _read_only_wavenet():
    layer = _layer(channels=64, bottleneck=32, dilations=(1, 2, 4, 8), kernel_size=3, gating="blended",
                   secondary="Sigmoid", head1x1={"active": True, "out_channels": 16, "groups": 1}, head_size=1)
    return _wavenet([layer], seed=70, scale=0.25)


def _long_and_conditioned_cases():
    layer = _layer(channels=4, bottleneck=2, dilations=(1, 1024, 7), kernel_size=[3, 4, 2], gating=["gated", "blended", "none"])
    yield "lookback_3072", _wavenet([layer], seed=80, scale=0.5)
    cond_layer = _layer(channels=4, bottleneck=4, dilations=(1, 2), gating="none", head_size=2)
    cond = _wavenet([cond_layer], seed=81, scale=0.5, head_scale=0.8)
    layer = _layer(condition_size=2, channels=6, bottleneck=3, dilations=(1, 4, 2), gating=["gated", "blended", "gated"],
                   secondary=["Softsign", "Hardswish", "SiLU"], head_size=3, activation_pre_film=_film(groups=2))
    head = {"in_channels": 3, "channels": 4, "out_channels": 1, "kernel_sizes": [2, 3], "activation": "Tanh"}
    yield "condition_dsp_gated_head", _wavenet([layer], seed=82, scale=0.45, head=head, condition_dsp=cond)
    a0 = _layer(input_size=2, condition_size=2, channels=5, bottleneck=3, dilations=(1, 2, 9), head_size=4,
                gating=["blended", "gated", "none"], head1x1={"active": True, "out_channels": 3, "groups": 1})
    a1 = _layer(input_size=5, condition_size=2, channels=4, bottleneck=4, dilations=(1, 6), head_size=3, gating="gated",
                head1x1={"active": True, "out_channels": 4, "groups": 1})
    yield "two_in_three_out", _wavenet([a0, a1], seed=83, scale=0.45, in_channels=2)


def convnet(channels, dilations, activation, seed, scale, batchnorm=True) -> dict:
    """a ConvNet (convnet.cpp) with convolution and head weights U(-scale, scale) and BatchNorm statistics near the identity
    (running mean, running variance, weight, bias, eps per block), so that a deep stack still passes the signal on"""
    nam = _convnet(channels, dilations, batchnorm, activation, seed)
    rng = np.random.default_rng(seed + 1000)
    w = rng.uniform(-scale, scale, size=len(nam["weights"])).astype(np.float32)
    if batchnorm:
        pos, cin = 0, 1
        for _d in dilations:
            pos += cin * channels * 2
            c = channels
            w[pos:pos + c] = rng.uniform(-0.1, 0.1, c)  # running mean
            w[pos + c:pos + 2 * c] = rng.uniform(0.5, 1.5, c)  # running variance
            w[pos + 2 * c:pos + 3 * c] = rng.uniform(0.8, 1.4, c) * rng.choice([-1.0, 1.0], c)  # weight
            w[pos + 3 * c:pos + 4 * c] = rng.uniform(-0.1, 0.1, c)  # bias
            w[pos + 4 * c] = 1e-5
            pos += 4 * c + 1
            cin = channels
    nam["weights"] = [float(v) for v in w]
    return nam


def _convnet_cases():
    dil = [2 ** (i % 8) for i in range(48)]
    # (at scale 1.0 the 48 blocks amplify rounding: two fp32 implementations drift apart by 7e-5 however right both are;
    # at 0.9 they agree to 1e-6 and the output still follows the input)
    yield "convnet_48_blocks", convnet(4, dil, "Tanh", seed=90, scale=0.9)
    yield "convnet_read_only", convnet(64, [1, 2, 4, 8, 16, 32, 64, 128], {"type": "LeakyReLU", "negative_slope": 0.1},
                                       seed=91, scale=0.2)


def _all():
    for gen in (_gating_cases, _film_cases, _grouping_cases, _limit_cases):
        for name, nam in gen():
            yield Case(name, nam, "generic", _compiled(nam), _lookback(nam))
    yield Case("read_only_wavenet", _read_only_wavenet(), "generic", False, _lookback(_read_only_wavenet()))
    for name, nam in _long_and_conditioned_cases():
        yield Case(name, nam, "generic", _compiled(nam), _lookback(nam))
    for name, nam in _convnet_cases():
        yield Case(name, nam, "convnet", False, max(nam["config"]["dilations"]))


def _compiled(nam) -> bool:
    return nam_config.expected_weight_count(nam) <= UNROLL_CAP


CASES = list(_all())
BY_NAME = {c.name: c for c in CASES}
