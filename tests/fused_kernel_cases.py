"""Model builders for the tests of the fused WaveNet family: the precompiled wavenet_fused_kernel (every geometry, with and
without a slot table), the precompiled wavenet_lat2_kernel, and the per-model NVRTC kernels wavenet_spec*_kernel and
wavenet_lat_kernel.  Not a test module: test_fused_cases_host.py holds the oracle to the reference build on these cases
and checks that each case can tell a wrong kernel from a right one; test_fused_paths_gpu.py runs each case on every
launch path of the family against the oracle.

Together the cases reach every channel pair the fused kernels are compiled for (kChannelPairs in csrc/nam_b200.cu), each
pair also in a case without a convolutional head (the low-latency kernels and the compiled short-call kernels serve only
those), with
exact (4, 8, 16) and padded (3, 6, 12, 13) channel counts in both array positions, kernel sizes 1-5 (and A2's 6 and 15),
look-backs inside the 64-column halo, past a 512-frame tile and past 1024 frames (so a 2048-column ring wraps inside one
call), A2-style convolutional heads, and all eleven activations.

Each case's weight scale and head_scale are fixed so that on `signal()` the output follows the input (its standard
deviation over time is between 0.1 and 1) and stays below 4 in magnitude: an off-by-one ring tap or a wrong weight then
moves the output by far more than the 1e-5 tolerance (test_fused_cases_host.py measures by how much)."""
from __future__ import annotations

import json
from dataclasses import dataclass

import numpy as np

from oracle import nam_config
from tests import nam_fixtures as fx


@dataclass
class Case:
    name: str
    nam: dict
    pair: tuple  # (C0, C1): the padded channels of array 0 and array 1 (0: one array), the fused kernel's template pair
    spec_threads: int  # threads per CTA of the compiled throughput kernel (spec_tile_geometry in csrc/jit_spec.cpp)
    seed: int  # of the weights; reseeded() derives a bank's second model from it

    @property
    def layers(self) -> list:
        return self.nam["config"]["layers"]

    @property
    def has_tanh(self) -> bool:
        """the model has a Tanh or Fasttanh activation, so fast_tanh is worth running too"""
        text = json.dumps(self.nam["config"])
        return '"Tanh"' in text or '"Fasttanh"' in text

    @property
    def conv_head(self) -> bool:
        return any(lc.get("head", {}).get("kernel_size", 1) > 1 for lc in self.layers)

    @property
    def lookback(self) -> int:
        """the longest look-back of any convolution (layers and heads), in frames"""
        lb = 0
        for lc in self.layers:
            ks = lc.get("kernel_sizes") or [lc["kernel_size"]] * len(lc["dilations"])
            lb = max([lb] + [(k - 1) * d for k, d in zip(ks, lc["dilations"])])
            if "head" in lc:
                lb = max(lb, (lc["head"]["kernel_size"] - 1) * lc["head"].get("head_dilation", 1))
        return lb

    @property
    def ring(self) -> int:
        """the frames of the largest ring: the longest look-back rounded up to a power of two (csrc/wavenet_pack.cpp)"""
        r = 1
        while r < self.lookback:
            r <<= 1
        return r


def signal(streams: int, n: int, seed: int) -> np.ndarray:
    """[streams, n]: the synthetic benchmark signal at four times its level (peaks near 1.5), which drives the saturating
    activations into both of their branches"""
    return np.ascontiguousarray(4.0 * fx.synthetic_batch(streams, n, seed=seed))


def _prelu(n: int) -> dict:
    return {"type": "PReLU", "negative_slopes": [round(0.03 + 0.04 * i, 4) for i in range(n)]}


LEAKY_RELU = {"type": "LeakyReLU", "negative_slope": 0.06}
LEAKY_HARDTANH = {"type": "LeakyHardtanh", "min_val": -0.6, "max_val": 0.5, "min_slope": 0.08, "max_slope": 0.15}


def _case(name, pair, spec_threads, channels, dilations, activations, scale, head_scale, seed, **kw) -> Case:
    nam = fx.random_wavenet(channels=channels, dilations=dilations, seed=seed, scale=scale, head_scale=head_scale, **kw)
    for lc, act in zip(nam["config"]["layers"], activations):
        lc["activation"] = act
    return Case(name, nam, pair, spec_threads, seed)


def _a2_full_like() -> Case:
    # A2-Full's shape (one array of 8 channels, kernel sizes 6 and 15, a 16-tap head), fewer layers: look-back 5 x 239
    dil = [1, 3, 7, 17, 41, 101, 239, 1, 13, 1, 3, 7, 17, 41, 101, 239]
    ks = [6] * 7 + [15, 15] + [6] * 7
    return _case("a2_full_like", (8, 0), 512, (8,), [dil], [LEAKY_RELU], scale=0.3, head_scale=0.13, seed=102,
                 kernel_sizes=[ks], head_kernel=16)


CASES = [
    # (4, 0): 3 channels padded to 4, kernel sizes 1-5, every look-back inside the halo
    _case("c3_halo", (4, 0), 512, (3,), [[1, 3, 7, 11, 15]], ["Hardtanh"], scale=0.6, head_scale=0.23, seed=113,
          kernel_sizes=[[2, 1, 3, 4, 5]]),
    _a2_full_like(),
    # (8, 0) without a convolutional head, so the low-latency kernel serves it; kernel sizes 2-5, look-back 239
    _case("c8_plain", (8, 0), 512, (8,), [[1, 5, 13, 40, 101, 239]], ["Hardswish"], scale=0.45, head_scale=2.06, seed=114,
          kernel_sizes=[[3, 2, 5, 4, 3, 2]]),
    # (16, 0): 13 channels padded to 16, look-back 1400 (rings of 2048 columns); the compiled kernel's 1024 x 1 tile
    _case("c13_ring_2048", (16, 0), 1024, (13,), [[1, 4, 1, 150, 300, 700]], ["SiLU"], scale=0.45, head_scale=0.44,
          seed=103, kernel_sizes=[[2, 3, 1, 4, 5, 3]]),
    # (4, 4): a convolutional head on each array (array 0's into array 1's head accumulator), look-back 64 = the halo
    _case("c4_c3_conv_heads", (4, 4), 512, (4, 3), [[1, 2, 4, 8, 16, 32], [1, 5, 25]], ["Tanh", "Fasttanh"], scale=0.6,
          head_scale=0.2, seed=104, kernel_size=3, head_kernel=3, head_dilation=4),
    # (4, 4) without a convolutional head, both arrays exact; look-back 256
    _case("c4_c4", (4, 4), 512, (4, 4), [[1, 2, 4, 8, 16, 32, 64, 128], [1, 3, 9, 27, 81]], ["Tanh", LEAKY_HARDTANH],
          scale=0.6, head_scale=1.02, seed=114, kernel_size=3),
    # (4, 8): per-channel PReLU slopes on 6 channels padded to 8; look-back 600 (past a 512-frame tile)
    _case("c3_c6_prelu", (4, 8), 512, (3, 6), [[1, 9], [2, 200, 1, 300]], ["Softsign", _prelu(6)], scale=0.6,
          head_scale=0.65, seed=105, kernel_sizes=[[3, 5], [2, 4, 1, 3]]),
    # (4, 16): 13 channels padded to 16 behind 4; look-back 1050
    _case("c4_c13", (4, 16), 1024, (4, 13), [[1, 2], [3, 100, 350]], ["Sigmoid", "Hardswish"], scale=0.45, head_scale=0.85,
          seed=106, kernel_size=4),
    # (8, 4): convolutional heads (4 taps 8 apart) on a two-array pair, 6 channels padded to 8
    _case("c6_c4_conv_heads", (8, 4), 512, (6, 4), [[1, 2, 30, 1, 10], [1, 64, 130]], [LEAKY_HARDTANH, "Tanh"],
          scale=0.45, head_scale=0.6, seed=107, kernel_sizes=[[5, 3, 2, 1, 4], [3, 3, 3]], head_kernel=4, head_dilation=8),
    # (8, 4) without a convolutional head, 3 channels padded to 4 in the second array; look-back 300
    _case("c8_c3", (8, 4), 512, (8, 3), [[1, 11, 100], [3, 50]], ["Softsign", "Sigmoid"], scale=0.6, head_scale=1.61,
          seed=115, kernel_sizes=[[2, 4, 3], [5, 3]]),
    # (8, 8): a1's dilations on 8 channels (look-back 1024), then 6 padded to 8
    _case("c8_c6", (8, 8), 512, (8, 6), [[1, 2, 4, 8, 16, 32, 64, 128, 256, 512], [1, 300]], ["ReLU", "Tanh"],
          scale=0.45, head_scale=0.063, seed=108, kernel_size=3),
    # (8, 16): kernel size 5 throughout
    _case("c8_c16", (8, 16), 1024, (8, 16), [[1, 7, 33], [2, 13, 150]], ["Hardswish", LEAKY_RELU], scale=0.45,
          head_scale=0.57, seed=109, kernel_size=5),
    # (16, 4): 12 and 3 channels padded to 16 and 4, PReLU slopes on the padded 3; look-back 520
    _case("c12_c3_prelu", (16, 4), 1024, (12, 3), [[1, 2, 4, 8, 16, 32, 64, 128, 260], [1, 2, 4]], ["Fasttanh", _prelu(3)],
          scale=0.45, head_scale=0.32, seed=110, kernel_size=3),
    # (16, 8): a1_standard's pair with odd dilations
    _case("c16_c8", (16, 8), 1024, (16, 8), [[1, 3, 9, 27, 81, 243, 500], [1, 2, 5, 11, 23]], ["SiLU", "Softsign"],
          scale=0.45, head_scale=0.19, seed=111, kernel_size=3),
    # (16, 16): 12 channels padded to 16 in the second position, kernel size 2
    _case("c16_c12", (16, 16), 1024, (16, 12), [[1, 3, 7, 17, 41, 101, 239], [1, 13]], ["Sigmoid", "ReLU"], scale=0.45,
          head_scale=1.0, seed=112, kernel_size=2),
]
BY_NAME = {c.name: c for c in CASES}


def _layer_weights(lc: dict) -> list:
    """(kind, count) of one fused-family array's weights in the .nam stream order: rechannel, then per layer the dilated
    convolution (weights, bias), the input mixin and the 1x1 (weights, bias), then the head (weights, bias)"""
    c, cin = lc["channels"], lc["input_size"]
    ks = lc.get("kernel_sizes") or [lc["kernel_size"]] * len(lc["dilations"])
    head = lc.get("head") or {"out_channels": lc["head_size"], "kernel_size": 1, "bias": lc["head_bias"]}
    out = [("rechannel", cin * c)]
    for k in ks:
        out += [("conv", k * c * c + c), ("mixin", c), ("1x1", c * c + c)]
    out.append(("head", head["out_channels"] * c * head["kernel_size"] + (head["out_channels"] if head["bias"] else 0)))
    return out


def weight_range(nam: dict, array: int, kind: str) -> tuple:
    """[start, stop) of the first block of `kind` ("conv": the first layer's dilated convolution and bias, or "head") of
    layer array `array` in the document's flat weights"""
    pos = 0
    for a, lc in enumerate(nam["config"]["layers"]):
        for k, n in _layer_weights(lc):
            if a == array and k == kind:
                return pos, pos + n
            pos += n
    raise KeyError((array, kind))


def check_layout(nam: dict) -> None:
    total = sum(n for lc in nam["config"]["layers"] for _k, n in _layer_weights(lc)) + 1  # + head_scale
    assert total == nam_config.expected_weight_count(nam) == len(nam["weights"])


def reseeded(case: Case) -> dict:
    """a second model of the case's shape for a bank: every weight but head_scale scaled by its own 1 + 5% N(0, 1)"""
    nam = json.loads(json.dumps(case.nam))
    w = np.asarray(nam["weights"], np.float32)
    w[:-1] *= (1.0 + 0.05 * np.random.default_rng(case.seed).standard_normal(len(w) - 1)).astype(np.float32)
    nam["weights"] = [float(v) for v in w]
    return nam
