"""The model-specialised throughput kernel in the tile its model gets (a1_standard: 1024 frames, one 1024-thread CTA per
SM; a2_full and wavenet.nam: 512 frames, two CTAs per SM), bit for bit against the precompiled fused kernel on the same
calls: call lengths around the tile size, successive calls that leave the clock off
a tile boundary, ragged calls, slot tables whose streams sit at different clocks, a batch that does not fill whole
rounds of 132 CTAs, a convolutional head (a2_full) and a one-array model (wavenet.nam).

Both kernels add in the same order, so with the library tanh their outputs agree to the last bit (`jit=1`: the
specialised kernel, mandatory; `jit=2`: the precompiled kernels; `tile_mode=2` keeps small batches off the lock-step
mode so that every long call takes the kernel under test)."""
import numpy as np
import pytest

import neuralampmodelercore_b200 as nb
from tests import nam_fixtures as fx

pytestmark = pytest.mark.gpu


def _pair(nam, batch):
    spec = nb.get_dsp(nam, batch=batch, fast_tanh=False, jit=1, tile_mode=2)
    assert spec.jit_state == 1, spec.jit_note()
    fused = nb.get_dsp(nam, batch=batch, fast_tanh=False, jit=2, tile_mode=2)
    assert fused.jit_state == 0
    for d in (spec, fused):
        d.Reset(48000.0, 4096)
    return spec, fused


def _same(a, b, what):
    assert a.shape == b.shape
    if not np.array_equal(a, b):
        bad = np.argwhere(a != b)
        raise AssertionError(f"{what}: {len(bad)} outputs differ, first at {tuple(bad[0])}: {a[tuple(bad[0])]!r} vs "
                             f"{b[tuple(bad[0])]!r}")


def _run_calls(name, batch, lengths, seed):
    nam = fx.load_model(name)
    x = fx.synthetic_batch(batch, sum(lengths), seed=seed)
    spec, fused = _pair(nam, batch)
    pos = 0
    for n in lengths:
        xi = np.ascontiguousarray(x[:, pos:pos + n])
        _same(spec.process_batch(xi), fused.process_batch(xi), f"{name}: call of {n} frames at frame {pos}")
        pos += n
    spec.close()
    fused.close()


@pytest.mark.parametrize("n", [1, 1023, 1024, 1025, 3000, 4096])
def test_call_lengths_around_the_tile(n):
    # each length twice: the second call starts where the first left the clock
    _run_calls("wavenet_a1_standard", 8, [n, n], seed=n)


def test_successive_calls_off_the_tile_boundary():
    _run_calls("wavenet_a1_standard", 8, [1500, 700, 2049, 333, 1024, 4095], seed=21)


def test_batch_that_does_not_fill_whole_rounds():
    # 133 streams on 132 CTAs: one CTA takes a second stream
    _run_calls("wavenet_a1_standard", 133, [2500, 1100], seed=22)


@pytest.mark.parametrize("name", ["a2_full", "wavenet"])
def test_convolutional_head_and_one_array(name):
    _run_calls(name, 6, [1024, 1025, 1, 2047], seed=23)


def test_ragged_calls_and_slot_tables_at_different_clocks():
    nam = fx.load_model("wavenet_a1_standard")
    B = 12
    spec, fused = _pair(nam, B)
    rng = np.random.default_rng(24)
    calls = [
        (list(range(B)), [1024] * B),  # every stream
        ([3, 0, 7, 11], [1025, 1, 2048, 600]),  # a subset, ragged: the clocks drift apart
        ([5, 3, 9], [3000, 1023, 4096]),
        (list(range(B - 1, -1, -1)), [int(v) for v in rng.integers(0, 2500, B)]),  # every stream, reversed, ragged
        ([0, 7], [1024, 1024]),
    ]
    for i, (streams, frames) in enumerate(calls):
        x = fx.synthetic_batch(len(streams), max(frames), seed=30 + i)
        a = spec.process_streams(streams, x, n_frames=frames)
        b = fused.process_streams(streams, x, n_frames=frames)
        _same(a, b, f"call {i} (streams {streams}, frames {frames})")
    # every stream once more from where its own clock stands
    x = fx.synthetic_batch(B, 1500, seed=40)
    _same(spec.process_batch(x), fused.process_batch(x), "final call on every stream")
    spec.close()
    fused.close()
