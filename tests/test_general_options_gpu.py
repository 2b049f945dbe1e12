"""Both forms of the general WaveNet kernel -- precompiled (wavenet_generic.cuh, jit = 2) and compiled per model by NVRTC
(wavenet_generic_spec.cuh, jit = 1) -- and the ConvNet kernel on every case of tests/general_kernel_cases.py: each option
of the reference's WaveNet, each limit of generic_desc.h, the read-only weight path and a look-back far beyond the
128-frame tile.  The yardstick is the oracle (1e-5 relative to max(1, max|y|)), which test_general_options_host.py holds to
the reference build on the same cases; stream 0 also meets the reference build's stored output directly.  The two forms
of the general kernel share the algorithm and the summation order, so they must agree to 1e-6."""
import numpy as np
import pytest

import neuralampmodelercore_b200 as nb
from oracle import oracle
from tests import general_kernel_cases as gk
from tests import nam_fixtures as fx

pytestmark = pytest.mark.gpu

TOL = 1e-5
SAME = 1e-6  # compiled vs precompiled general kernel
STREAMS = 5
REF_N, REF_SEED = 4096, 7  # the signal of test_general_options_host.py's reference outputs (stream 0 here)


def _ring(lookback: int) -> int:
    """the frames a convolution's ring keeps: look-back + one tile, rounded up to a power of two (generic_pack.cpp)"""
    r = 1
    while r < lookback + 128:
        r <<= 1
    return r


def _calls(case):
    """lengths 1, 127, 128, 129 (one frame short of, exactly and one past the tile), an odd length, then one call longer
    than the largest ring, then the rest of the signal"""
    fixed = [1, 127, 128, 129, 333, _ring(case.lookback) + 389]
    n = max(REF_N, sum(fixed))
    block = max(fixed[-1], 1024)
    calls = list(fixed)
    while sum(calls) < n:
        calls.append(min(block, n - sum(calls)))
    return calls, block


def _input(case, streams, n):
    x = gk.signal(case, streams, n, seed=REF_SEED + 100)
    x[0, :, :REF_N] = gk.signal(case, 1, REF_N, REF_SEED)[0]
    return x


def _oracle(case, x, block=512):
    outs = []
    for s in range(x.shape[0]):
        m = oracle.OracleModel.from_dict(case.nam)
        m.reset(48000.0, block)
        outs.append(np.concatenate([np.atleast_2d(m.process(np.ascontiguousarray(x[s, :, p:p + block])))
                                    for p in range(0, x.shape[2], block)], axis=1))
        m.close()
    return np.stack(outs)


def _run(case, x, calls, block, jit):
    d = nb.get_dsp(case.nam, batch=x.shape[0], jit=jit)
    assert d.jit_state == (1 if jit == 1 else 0), d.jit_note()
    d.Reset(48000.0, block)
    out, pos = [], 0
    for n in calls:
        xc = np.ascontiguousarray(x[:, :, pos:pos + n] if case.in_channels > 1 else x[:, 0, pos:pos + n])
        y = d.process_batch(xc)
        out.append(y if y.ndim == 3 else y[:, None, :])
        pos += n
    d.close()
    return np.concatenate(out, axis=2)


def _stored_reference(case):
    with np.load(fx.REFERENCE_OUTPUTS) as z:
        return z[f"general_options/{case.name}/exact"]


@pytest.mark.parametrize("case", gk.CASES, ids=[c.name for c in gk.CASES])
def test_kernels_match_the_oracle(case):
    calls, block = _calls(case)
    x = _input(case, STREAMS, sum(calls))
    want = _oracle(case, x)
    scale = max(1.0, float(np.max(np.abs(want))))
    pre = _run(case, x, calls, block, jit=2)
    err = float(np.max(np.abs(pre - want)))
    assert err <= TOL * scale, f"precompiled kernel: {err:.3e} from the oracle (max|y| {scale:.2f})"
    stored = _stored_reference(case)
    err_ref = float(np.max(np.abs(fx.sample(pre[0, :, :REF_N]) - stored)))
    assert err_ref <= TOL * scale, f"precompiled kernel: {err_ref:.3e} from the reference build's output"
    if case.compiled:
        comp = _run(case, x, calls, block, jit=1)
        err = float(np.max(np.abs(comp - want)))
        assert err <= TOL * scale, f"compiled kernel: {err:.3e} from the oracle"
        diff = float(np.max(np.abs(comp - pre)))
        assert diff <= SAME * scale, f"compiled and precompiled kernels differ by {diff:.3e}"


def test_seventy_streams():
    """70 streams of different signals (more than one 64-stream group, the last group partly filled): every stream is its
    own, on both forms"""
    case = gk.BY_NAME["parametric_primaries"]
    n, block = 1500, 512
    x = fx.synthetic_batch(70, n, seed=29) * 4.0
    proto = oracle.OracleModel.from_dict(case.nam)
    proto.reset(48000.0, 256)
    want = proto.run_batch(x, 256)
    calls = [block, 129, 1, 127, 128, block, n - 2 * block - 385]
    outs = {jit: _run(case, x[:, None, :], calls, block, jit)[:, 0] for jit in (2, 1)}
    scale = max(1.0, float(np.max(np.abs(want))))
    for jit, y in outs.items():
        err = float(np.max(np.abs(y - want)))
        assert err <= TOL * scale, f"jit={jit}: {err:.3e}"
    assert float(np.max(np.abs(outs[1] - outs[2]))) <= SAME * scale


@pytest.mark.parametrize("name", ["parametric_primaries", "film_input_mixin_pre_film", "condition_dsp_gated_head"])
def test_two_model_bank_on_the_shape_compiled_kernel(name):
    """a bank of the case and a reweighted copy, on the general kernel compiled for their shape (weights staged per stream,
    read through gspec::w): each stream within 1e-6 of an ordinary compiled handle of its model"""
    from tests.test_general_bank_gpu import _reweighted

    case = gk.BY_NAME[name]
    docs = [case.nam, _reweighted(case.nam, 2, seed=3)[1]]
    B, block, n = 4, 256, 768
    models = [0, 1, 1, 0]
    bank = nb.get_dsp_bank(docs, batch=B, jit=1)
    assert bank.jit_state == 1, bank.jit_note()
    bank.Reset(48000.0, block)
    bank.assign_streams(list(range(B)), models)
    x = gk.signal(case, B, n, seed=31)
    feed = (lambda a: a) if case.in_channels > 1 else (lambda a: a[:, 0])
    y = np.concatenate([bank.process_batch(np.ascontiguousarray(feed(x[..., p:p + block]))) for p in range(0, n, block)], axis=-1)
    bank.close()
    for k in range(2):
        rows = [s for s in range(B) if models[s] == k]
        h = nb.get_dsp(docs[k], batch=len(rows), jit=1)
        assert h.jit_state == 1, h.jit_note()
        h.Reset(48000.0, block)
        yk = np.concatenate([h.process_batch(np.ascontiguousarray(feed(x[rows][..., p:p + block]))) for p in range(0, n, block)],
                            axis=-1)
        h.close()
        scale = max(1.0, float(np.max(np.abs(yk))))
        assert float(np.max(np.abs(y[rows] - yk))) <= SAME * scale, f"model {k}"
