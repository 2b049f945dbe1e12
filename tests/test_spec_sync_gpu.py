"""The specialised throughput kernel's per-layer synchronisation (history copies and ring stores around the barriers B0
and B1, the async-proxy fence only in the threads whose columns a ring store reads), bit for bit against the
precompiled fused kernel with the library tanh: many tiles of one stream in one call, rings whose every copy wraps,
8-only and 16-only channel models, a convolutional head, and ragged calls through slot tables.

`jit=1`: the specialised kernel, mandatory; `jit=2`: the precompiled kernels; `tile_mode=2` keeps small batches off the
lock-step mode so that every long call takes the kernel under test."""
import numpy as np
import pytest

import neuralampmodelercore_b200 as nb
from tests import nam_fixtures as fx

pytestmark = pytest.mark.gpu


def _pair(nam, batch, max_frames=4096):
    spec = nb.get_dsp(nam, batch=batch, fast_tanh=False, jit=1, tile_mode=2)
    assert spec.jit_state == 1, spec.jit_note()
    fused = nb.get_dsp(nam, batch=batch, fast_tanh=False, jit=2, tile_mode=2)
    assert fused.jit_state == 0
    for d in (spec, fused):
        d.Reset(48000.0, max_frames)
    return spec, fused


def _same(a, b, what):
    assert a.shape == b.shape
    if not np.array_equal(a, b):
        bad = np.argwhere(a != b)
        raise AssertionError(f"{what}: {len(bad)} outputs differ, first at {tuple(bad[0])}: {a[tuple(bad[0])]!r} vs "
                             f"{b[tuple(bad[0])]!r}")


def _run_calls(nam, batch, lengths, seed, what):
    x = fx.synthetic_batch(batch, sum(lengths), seed=seed)
    spec, fused = _pair(nam, batch, max(max(lengths), 4096))
    pos = 0
    for n in lengths:
        xi = np.ascontiguousarray(x[:, pos:pos + n])
        _same(spec.process_batch(xi), fused.process_batch(xi), f"{what}: call of {n} frames at frame {pos}")
        pos += n
    spec.close()
    fused.close()


def test_one_stream_walks_nine_tiles_in_one_call():
    # a1_standard takes 1024-frame tiles: 9 tiles and a partial one, then a call that starts off the tile boundary
    _run_calls(fx.load_model("wavenet_a1_standard"), 1, [9 * 1024 + 77, 3 * 1024], seed=51, what="a1_standard, 1 stream")


@pytest.mark.parametrize("seed", [1, 2])
def test_lookback_equal_to_ring_so_every_copy_wraps(seed):
    # kernel size 3 and power-of-two dilations: each layer's look-back 2 d is its whole ring, so every history load and
    # ring store that does not start at column 0 is split in two pieces
    nam = fx.random_wavenet(channels=(16, 8), dilations=[[1, 2, 4, 8, 16, 32, 64, 128, 256, 512]] * 2, seed=seed)
    _run_calls(nam, 5, [1000, 1024, 2100, 37, 1024], seed=60 + seed, what=f"random a1-shaped model {seed}")


@pytest.mark.parametrize("channels", [(8,), (8, 8), (16,), (16, 16)])
def test_models_of_one_channel_count(channels):
    dil = [[1, 3, 9, 27, 81, 243], [2, 4, 8, 16, 32, 64, 128]][: len(channels)]
    nam = fx.random_wavenet(channels=channels, dilations=dil, seed=len(channels) * 10 + channels[0])
    _run_calls(nam, 4, [1500, 1024, 3000], seed=70, what=f"channels {channels}")


def test_a2_full_convolutional_head():
    _run_calls(fx.load_model("a2_full"), 3, [4 * 1024 + 5, 1023, 700], seed=80, what="a2_full")


def test_ragged_calls_through_slot_tables():
    nam = fx.load_model("wavenet_a1_standard")
    B = 9
    spec, fused = _pair(nam, B)
    rng = np.random.default_rng(90)
    for i in range(6):
        streams = [int(v) for v in rng.choice(B, size=int(rng.integers(1, B + 1)), replace=False)]
        frames = [int(v) for v in rng.integers(0, 4097, len(streams))]
        x = fx.synthetic_batch(len(streams), max(frames + [1]), seed=91 + i)
        _same(spec.process_streams(streams, x, n_frames=frames), fused.process_streams(streams, x, n_frames=frames),
              f"call {i} (streams {streams}, frames {frames})")
    x = fx.synthetic_batch(B, 2222, seed=99)
    _same(spec.process_batch(x), fused.process_batch(x), "final call on every stream")
    spec.close()
    fused.close()
