"""The fused WaveNet family's cases (tests/fused_kernel_cases.py) on the host: each case takes the fused kernel with its
channel pair, and together they take every pair the kernels are compiled for; each case's output follows its input; a
model one ring tap or one weight away from the case gives an output far outside the tolerance; the compiled kernel's tile
geometry is 1024 x 1 or 512 x 2 as the case says; and the oracle matches the reference build on every case.

The reference's outputs come from tests/golden/reference_outputs.npz under fused_cases/ (nam_fixtures.reference)."""
import copy

import numpy as np
import pytest

import neuralampmodelercore_b200 as nb
from oracle import oracle, ref
from tests import fused_kernel_cases as fc
from tests import nam_fixtures as fx

TOL = 1e-5
N, BLOCK, SEED = 4096, 256, 7  # one stream; the longest look-back (1400) is reached many times over
MARGIN = 10.0  # a mutant must move the output by at least this many tolerances

# kChannelPairs in csrc/nam_b200.cu: the (C0, C1) pairs wavenet_fused_kernel and wavenet_lat2_kernel are compiled for
CHANNEL_PAIRS = {(4, 0), (8, 0), (16, 0), (4, 4), (4, 8), (4, 16), (8, 4), (8, 8), (8, 16), (16, 4), (16, 8), (16, 16)}
IDS = [c.name for c in fc.CASES]


def _oracle(nam, fast=False):
    x = fc.signal(1, N, SEED)
    m = oracle.OracleModel.from_dict(nam, fast_tanh=fast)
    m.reset(48000.0, BLOCK)
    y = m.run(x[0], BLOCK)
    m.close()
    return y


def _reference_run(case, fast):
    x = fc.signal(1, N, SEED)
    r = ref.ReferenceModel.from_dict(case.nam, fast_tanh=fast)
    r.reset(48000.0, BLOCK)
    y = r.run(x[0], BLOCK)
    r.close()
    return y


@pytest.mark.parametrize("case", fc.CASES, ids=IDS)
def test_each_case_takes_the_fused_kernel_with_its_channel_pair(case):
    fc.check_layout(case.nam)
    info = nb.inspect(case.nam)
    assert info["kernel"] == "fused", info
    assert info["kernel_variant"] == case.pair[0] * 100 + case.pair[1], info


def test_the_cases_reach_every_channel_pair():
    assert {c.pair for c in fc.CASES} == CHANNEL_PAIRS
    # the low-latency kernels and the compiled short-call kernels refuse convolutional heads: every pair has a case without
    assert {c.pair for c in fc.CASES if not c.conv_head} == CHANNEL_PAIRS


def test_the_cases_cover_the_look_back_ranges_heads_and_activations():
    lbs = [c.lookback for c in fc.CASES]
    assert any(lb <= 64 for lb in lbs) and any(512 < lb <= 1024 for lb in lbs) and any(lb > 1024 for lb in lbs)
    kernels = {k for c in fc.CASES for lc in c.layers for k in (lc.get("kernel_sizes") or [lc["kernel_size"]])}
    assert set(range(1, 6)) <= kernels
    heads = [c for c in fc.CASES if c.conv_head]
    assert len({c.pair for c in heads}) >= 3 and (8, 0) in {c.pair for c in heads}
    assert any(c.pair[1] for c in heads)
    for c in heads:
        assert all((lc["head"]["kernel_size"] - 1) * lc["head"].get("head_dilation", 1) <= 64 for lc in c.layers)
    acts = {(a if isinstance(a, str) else a["type"]) for c in fc.CASES for a in (lc["activation"] for lc in c.layers)}
    assert acts == {"Tanh", "Hardtanh", "Fasttanh", "ReLU", "LeakyReLU", "PReLU", "Sigmoid", "SiLU", "Hardswish",
                    "LeakyHardtanh", "Softsign"}
    # per-channel PReLU slopes on a padded array: a pad channel's slope must not reach the output
    assert any(isinstance(lc["activation"], dict) and lc["activation"]["type"] == "PReLU"
               and len(lc["activation"]["negative_slopes"]) == lc["channels"] and lc["channels"] not in (4, 8, 16)
               for c in fc.CASES for lc in c.layers)
    # exact and padded channel counts in both array positions
    for a in (0, 1):
        counts = {c.layers[a]["channels"] for c in fc.CASES if len(c.layers) > a}
        assert {4, 8, 16} <= counts and {3, 6, 12, 13} <= counts, (a, counts)


@pytest.mark.parametrize("case", fc.CASES, ids=IDS)
def test_the_output_follows_the_input(case):
    y = _oracle(case.nam)
    std, peak = float(np.std(y)), float(np.max(np.abs(y)))
    assert 0.1 <= std <= 1.0 and peak <= 4.0, f"{case.name}: std over time {std:.3f}, max|y| {peak:.3f}"


@pytest.mark.parametrize("case", fc.CASES, ids=IDS)
def test_the_compiled_kernels_tile_geometry(case):
    rep = nb.jit_prepare(case.nam, fast_tanh=False)
    assert rep["ok"], rep["why_not"][:2000]
    assert rep["threads"] == case.spec_threads


def test_the_cases_compile_to_both_tile_geometries():
    assert {c.spec_threads for c in fc.CASES} == {512, 1024}


def _mutants(case):
    """(what, document): dilation + 1 in the first and the last layer of each array; the largest 1x1 bias of array 0's first
    layer (it feeds every later layer) x 1.001; with a convolutional head, the largest weight of the output head x 1.001"""
    for a, lc in enumerate(case.layers):
        for li in (0, len(lc["dilations"]) - 1):
            nam = copy.deepcopy(case.nam)
            nam["config"]["layers"][a]["dilations"][li] += 1
            yield f"array {a} layer {li} dilation + 1", nam
    w = np.asarray(case.nam["weights"])
    s, e = fc.weight_range(case.nam, 0, "1x1")
    picks = [("array 0 layer 0 1x1 bias", e - case.layers[0]["channels"], e)]
    if case.conv_head:
        picks.append(("output head weight",) + fc.weight_range(case.nam, len(case.layers) - 1, "head"))
    for what, s, e in picks:
        i = s + int(np.argmax(np.abs(w[s:e])))
        nam = copy.deepcopy(case.nam)
        nam["weights"][i] = float(np.float32(w[i] * 1.001))
        yield f"{what} [{i}] x 1.001", nam


@pytest.mark.parametrize("case", fc.CASES, ids=IDS)
def test_mutants_move_the_output_far_past_the_tolerance(case):
    y = _oracle(case.nam)
    tol = TOL * max(1.0, float(np.max(np.abs(y))))
    margins = {what: float(np.max(np.abs(_oracle(nam) - y))) / tol for what, nam in _mutants(case)}
    worst = min(margins, key=margins.get)
    print(f"{case.name}: smallest margin {margins[worst]:.1f} x the tolerance ({worst})")
    assert margins[worst] >= MARGIN, margins


REGIMES = [(c, False) for c in fc.CASES] + [(c, True) for c in fc.CASES if c.has_tanh]


@pytest.mark.parametrize("case,fast", REGIMES, ids=[f"{c.name}-{'fast' if f else 'exact'}_tanh" for c, f in REGIMES])
def test_oracle_matches_the_reference_build(case, fast):
    regime = "fast" if fast else "exact"
    yr = fx.reference(f"fused_cases/{case.name}/{regime}", lambda: _reference_run(case, fast))
    yo = fx.sample(_oracle(case.nam, fast))
    peak = float(np.max(np.abs(yr)))
    err = float(np.max(np.abs(yo - yr)))
    assert err <= TOL * max(1.0, peak), f"{case.name}: max|reference - oracle| = {err:.3e} (max|y| {peak:.3f})"
