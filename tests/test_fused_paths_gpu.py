"""Every launch path of the fused WaveNet family (launch_wavenet in csrc/nam_b200.cu) on every case of
tests/fused_kernel_cases.py, against the oracle (1e-5 relative to max(1, max|y|)), which test_fused_cases_host.py holds
to the reference build on the same cases.

Each case has one oracle run of 16 streams x N frames.  Each path runs a prefix of those streams through all N frames in
its own call lengths (among them 1, an odd length, one tile and one tile + 1, and where the path allows, a call longer
than the case's largest ring), in three ways:
- contiguous process_batch calls: the table-free instantiation;
- slot tables: process_streams over a new permutation of the slots each call, one of them ragged (a 0-frame entry
  among them), so the streams' clocks drift apart for the calls after it: the TBL instantiation;
- a 2-model bank of the case and a reseeded copy, the streams bound to them alternately: the TBL instantiation with a
  weight blob per stream; each stream meets the oracle of its own model.
The kernels each path launches are read from torch.profiler's CUDA activity, and the path's kernel must be among them,
so a change to the dispatch rules cannot quietly move a test off the path it was written for."""
import json
import os
import tempfile

import numpy as np
import pytest
import torch

import neuralampmodelercore_b200 as nb
from oracle import oracle
from tests import fused_kernel_cases as fc

pytestmark = pytest.mark.gpu

TOL = 1e-5
STREAMS = 16  # the compiled 64-frame short-call kernel packs 8 streams per CTA and runs only from two CTAs' worth up
N, SEED = 4608, 41


# (name, streams, handle options, $NAM_B200_LAT_KERNEL, max call / Reset size, tile frames (the compiled throughput kernel's:
# the case's, see _tile), the instantiation's template
# arguments after C0, C1 (wavenet_fused_kernel: S, NT, MINB, LQ, LS; wavenet_lat2_kernel: FW) or the compiled kernel's name)
PATHS = [
    ("lat2_64", 5, {"jit": 2}, "precompiled", 64, 64, "lat2 2"),
    ("lat2_128", 5, {"jit": 2}, "precompiled", 128, 128, "lat2 4"),
    ("short_4x64", 9, {"jit": 2}, "off", 96, 64, "fused 2 128 3 6 false"),
    ("short_4x128", 9, {"jit": 2}, "off", 192, 128, "fused 2 256 2 7 false"),
    ("small_128x1", 5, {"jit": 2}, "off", 128, 128, "fused 1 128 3 7 false"),
    ("lockstep_128", 3, {"jit": 2}, None, 0, 128, "fused 1 128 3 7 true"),
    ("lockstep_256", 3, {"jit": 2, "kernel_geometry": 1}, None, 0, 256, "fused 2 128 3 8 true"),
    ("lockstep_512", 3, {"jit": 2, "kernel_geometry": 2}, None, 0, 512, "fused 2 256 2 9 true"),
    ("wavefront", 3, {"jit": 2, "tile_mode": 1}, None, 0, 512, "fused 2 256 2 9 false"),
    ("persistent_256x2", 9, {"jit": 2, "tile_mode": 2}, None, 0, 512, "fused 2 256 2 9 false"),
    ("persistent_128x2", 9, {"jit": 2, "tile_mode": 2, "kernel_geometry": 1}, None, 0, 256, "fused 2 128 3 8 false"),
    ("persistent_2_sms", 9, {"jit": 2, "tile_mode": 2, "ctas_per_sm": 1}, None, 0, 512, "fused 2 256 2 9 false"),
    ("compiled", 9, {"jit": 1, "tile_mode": 2}, None, 0, 512, "wavenet_spec_kernel"),
    ("compiled_short64", 16, {"jit": 1}, "off", 64, 64, "wavenet_spec_short_kernel"),
    ("compiled_short128", 16, {"jit": 1}, "off", 128, 128, "wavenet_spec_short128_kernel"),
    ("compiled_short256", 16, {"jit": 1}, "off", 256, 256, "wavenet_spec_short256_kernel"),
    ("compiled_latency", 5, {"jit": 3}, "jit", 128, 128, "wavenet_lat_kernel"),
]
BY_PATH = {p[0]: p for p in PATHS}
# the low-latency kernels and the compiled short-call kernels have no convolutional head: such a model's short calls take
# the 128 x 1 geometry (few streams) or the 4 x 64 / 4 x 128 geometries (many)
NO_CONV_HEAD = {"lat2_64": "fused 1 128 3 7 false", "lat2_128": "fused 1 128 3 7 false", "compiled_short64": None,
                "compiled_short128": None, "compiled_short256": None, "compiled_latency": None}
COMPILED = {p[0] for p in PATHS if p[2]["jit"] in (1, 3)}


def _calls(case, max_call, tile):
    """lengths 1, an odd one, one tile, one tile + 1 (each capped at the path's longest call), then, where calls are not
    capped, one longer than the case's largest ring; the rest of the N frames in calls of at most one tile or 1024"""
    cap = max_call or N
    fixed = [1, min(cap, tile) - 1, min(cap, tile), min(cap, tile + 1)]
    if not max_call:
        fixed.append(case.ring + 389)
    calls = list(fixed)
    block = min(cap, max(tile, 1024) if not max_call else cap)
    while sum(calls) < N:
        calls.append(min(block, N - sum(calls)))
    return calls


def _expected(case, path):
    kind = BY_PATH[path][6]
    if case.conv_head and path in NO_CONV_HEAD:
        kind = NO_CONV_HEAD[path]
    return kind


def _kernel_name(case, kind, table):
    """the kernel's name as CUPTI reports it, without spaces"""
    if kind.startswith("wavenet_"):
        return kind
    family, *args = kind.split()
    c0, c1 = case.pair
    name = "wavenet_fused_kernel" if family == "fused" else "wavenet_lat2_kernel"
    return f"{name}<{c0},{c1},{','.join(args)},{'true' if table else 'false'}>"


class Kernels:
    """The CUDA kernels launched inside the block, with their grids, from torch.profiler's CUDA activity"""

    def __enter__(self):
        torch.cuda.synchronize()
        self.prof = torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA])
        self.prof.__enter__()
        return self

    def __exit__(self, *exc):
        torch.cuda.synchronize()
        self.prof.__exit__(*exc)
        with tempfile.TemporaryDirectory() as tmp:
            path = os.path.join(tmp, "trace.json")
            self.prof.export_chrome_trace(path)
            with open(path) as f:
                trace = json.load(f)
        self.launches = [(e["name"].replace(" ", ""), tuple(e.get("args", {}).get("grid", ())))
                         for e in trace.get("traceEvents", []) if e.get("cat") == "kernel"]
        return False

    def grids(self, name):
        return [g for n, g in self.launches if name in n]


@pytest.fixture(scope="module")
def oracle_runs():
    cache = {}

    def get(nam, fast):
        key = (json.dumps(nam), fast)
        if key not in cache:
            proto = oracle.OracleModel.from_dict(nam, fast_tanh=fast)
            proto.reset(48000.0, 256)
            cache[key] = proto.run_batch(fc.signal(STREAMS, N, SEED), 256)
            proto.close()
        return cache[key]

    return get


def _handle(nam, batch, opts, max_call, fast, bank_docs=None):
    if bank_docs is not None:
        d = nb.get_dsp_bank(bank_docs, batch=batch, fast_tanh=fast, **opts)
    else:
        d = nb.get_dsp(nam, batch=batch, fast_tanh=fast, **opts)
    if opts["jit"] == 1:
        assert d.jit_state == 1, d.jit_note()
    d.Reset(48000.0, max_call or N)
    return d


def _tile(case, path):
    """the frames of the path's tile; the compiled throughput kernel's is the case's (1024 x 1 or 512 x 2 threads x frames)"""
    return case.spec_threads if path == "compiled" else BY_PATH[path][5]


def _run(case, path, fast, mode, x, calls=None):
    """The outputs of `mode` ("contiguous", "table" or "bank") on `path`, each stream's as far as it got, and the kernels
    that ran"""
    name, k, opts, _lat, max_call, _tile_frames, _kind = BY_PATH[path]
    calls = calls or _calls(case, max_call, _tile(case, path))
    docs = [case.nam, fc.reseeded(case)] if mode == "bank" else None
    d = _handle(case.nam, k, opts, max_call, fast, docs)
    if docs:
        d.assign_streams(list(range(k)), [s % 2 for s in range(k)])
    if path == "persistent_2_sms":  # one CTA on each of 2 SMs
        d.set_reserved_sms(torch.cuda.get_device_properties(0).multi_processor_count - 2)
    if path == "compiled_latency":
        assert d.jit_lat_state == 1, d.jit_note()
    rng = np.random.default_rng(list(BY_PATH).index(name))
    pos = np.zeros(k, np.int64)
    out = [[] for _ in range(k)]
    with Kernels() as kern:
        for c, n in enumerate(calls):
            if mode == "table":
                streams = [int(s) for s in rng.permutation(k)]
                counts = [n] * k
                if c == 1:  # ragged: a 0-frame entry, the others from 1 to n frames
                    counts = [0] + [int(v) for v in rng.integers(1, n + 1, size=k - 1)]
                    counts[-1] = n
                xi = np.zeros((k, n), np.float32)
                for i, s in enumerate(streams):
                    xi[i, :counts[i]] = x[s, pos[s]:pos[s] + counts[i]]
                y = d.process_streams(streams, xi, n_frames=counts)
                for i, s in enumerate(streams):
                    out[s].append(y[i, :counts[i]])
                    pos[s] += counts[i]
            else:
                y = d.process_batch(np.ascontiguousarray(x[:k, pos[0]:pos[0] + n]))
                for s in range(k):
                    out[s].append(y[s])
                pos += n
    d.close()
    return [np.concatenate(o) for o in out], kern


REGIMES = [(c, False) for c in fc.CASES] + [(c, True) for c in fc.CASES if c.has_tanh]
REGIME_IDS = [f"{c.name}-{'fast' if f else 'exact'}_tanh" for c, f in REGIMES]


def _run_and_check(case, path, fast, mode, x, want):
    """one run of the path, each stream within the tolerance of its oracle output; returns the kernels that ran"""
    outs, kern = _run(case, path, fast, mode, x)
    assert all(len(y) > 0 for y in outs)
    for s, y in enumerate(outs):
        ref = want[s][:len(y)]
        scale = max(1.0, float(np.max(np.abs(ref))))
        err = float(np.max(np.abs(y - ref)))
        assert err <= TOL * scale, f"{path} ({mode}), stream {s}: {err:.3e} from the oracle (max|y| {scale:.2f})"
    return kern


@pytest.mark.parametrize("case,fast", REGIMES, ids=REGIME_IDS)
@pytest.mark.parametrize("path", [p[0] for p in PATHS])
def test_path_matches_the_oracle(case, fast, path, oracle_runs, monkeypatch):
    kind = _expected(case, path)
    if kind is None:
        pytest.skip(f"{path} has no kernel for a convolutional head")
    lat = BY_PATH[path][3]
    if lat is not None:
        monkeypatch.setenv("NAM_B200_LAT_KERNEL", lat)
    x = fc.signal(STREAMS, N, SEED)
    want = oracle_runs(case.nam, fast)
    modes = ["contiguous"] if path in COMPILED else ["contiguous", "table", "bank"]
    for mode in modes:
        want_m = want
        if mode == "bank":
            other = oracle_runs(fc.reseeded(case), fast)
            want_m = [want[s] if s % 2 == 0 else other[s] for s in range(STREAMS)]
        kern = _run_and_check(case, path, fast, mode, x, want_m)
        if not kern.launches:
            # The profiler can hand back a capture with no CUDA activity at all (it did once, with outputs that met the
            # oracle).  No launch path runs without a kernel, so an empty capture says nothing about dispatch: take the
            # capture again, from a second run whose outputs are checked as well.
            kern = _run_and_check(case, path, fast, mode, x, want_m)
        name = _kernel_name(case, kind, mode != "contiguous")
        grids = kern.grids(name)
        assert grids, f"{path} ({mode}): {name} did not run; the kernels were {sorted({n for n, _ in kern.launches})}"
        if path == "wavefront":  # one CTA per (stream, tile): the grid is larger than the stream count
            assert max(g[0] for g in grids) > BY_PATH[path][1], grids
        if path == "persistent_2_sms":  # 2 SMs' worth of CTAs, each walking several streams
            assert max(g[0] for g in grids) < BY_PATH[path][1], grids


@pytest.mark.parametrize("case", fc.CASES, ids=[c.name for c in fc.CASES])
def test_the_compiled_kernel_equals_the_persistent_fused_kernel(case):
    """with the library tanh both kernels add in the same order: bit for bit on the same calls, split around the compiled
    kernel's tile"""
    x = fc.signal(STREAMS, N, SEED)
    calls = _calls(case, 0, case.spec_threads)
    spec, _ = _run(case, "compiled", False, "contiguous", x, calls)
    fused, _ = _run(case, "persistent_256x2", False, "contiguous", x, calls)
    for s in range(len(spec)):
        assert np.array_equal(spec[s], fused[s]), f"stream {s}: {int(np.sum(spec[s] != fused[s]))} outputs differ"
