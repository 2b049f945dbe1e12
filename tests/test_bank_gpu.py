"""GPU tests of model banks (nam_b200_create_bank_from_json, DSP via get_dsp_bank): one handle whose streams each run
their own model.  The yardstick is one ordinary jit = 2 handle per model, given every call the bank gets: each bank stream's
outputs and records must match, byte for byte, the same stream index on the handle of its model, and each stream must be
within 1e-5 of the oracle for its model."""
import copy

import numpy as np
import pytest

import neuralampmodelercore_b200 as nb
from neuralampmodelercore_b200 import _capi
from tests import nam_fixtures as fx
from tests.test_process_streams_gpu import TOL, _oracle_stream

pytestmark = pytest.mark.gpu
SHAPES = {"wavenet": "wavenet", "a1": "wavenet_a1_standard", "a2_lite": "a2_lite"}


def _family(shape: str, k: int, seed: int = 0) -> list:
    """k documents of one shape: the fixture's weights, each model seeded-perturbed (head_scale, the last weight, too),
    each with its own loudness"""
    base = fx.load_model(SHAPES[shape])
    docs = []
    for i in range(k):
        d = copy.deepcopy(base)
        rng = np.random.default_rng(1000 * seed + i)
        w = np.asarray(base["weights"], np.float32)
        d["weights"] = [float(v) for v in w * (1.0 + 0.05 * rng.standard_normal(w.shape)).astype(np.float32)]
        d.setdefault("metadata", {})
        d["metadata"] = dict(d["metadata"] or {}, loudness=-20.0 - i)
        docs.append(d)
    return docs


class Rig:
    """A bank and its yardstick handles, plus each stream's chunks since it was last bound (for the oracle)."""

    def __init__(self, docs, batch, block, **kw):
        self.docs, self.block = docs, block
        self.bank = nb.get_dsp_bank(docs, batch=batch, **kw)
        self.bank.Reset(48000.0, block)
        self.refs = []
        for d in docs:
            r = nb.get_dsp(d, batch=batch, **dict(kw, jit=2))
            r.Reset(48000.0, block)
            self.refs.append(r)
        self.model = np.zeros(batch, np.int64)
        self.ins = {s: [] for s in range(batch)}
        self.outs = {s: [] for s in range(batch)}

    def assign(self, streams, models):
        self.bank.assign_streams(streams, models)
        for s, k in zip(streams, models):
            self.refs[k].reset_streams([s])
            self.model[s] = k
            self.ins[s], self.outs[s] = [], []
        assert list(self.bank.stream_models(streams)) == list(models)

    def call(self, streams, counts, seed):
        """A ragged process_streams call on the bank and the same call on every yardstick handle"""
        n_max = max(counts)
        x = fx.synthetic_batch(len(streams), max(n_max, 1), seed=seed)[:, :n_max].copy()
        for i, c in enumerate(counts):
            x[i, c:] = 0.0
        y = self.bank.process_streams(streams, x, n_frames=counts)
        for k, ref in enumerate(self.refs):
            rows = [i for i, s in enumerate(streams) if self.model[s] == k]
            if rows:
                yk = ref.process_streams(streams, x, n_frames=counts)
                assert np.array_equal(y[rows], yk[rows]), f"model {k}: outputs differ from its ordinary handle"
        for i, (s, c) in enumerate(zip(streams, counts)):
            if c:
                self.ins[s].append(x[i, :c].copy())
                self.outs[s].append(y[i, :c].copy())
        return y

    def check_records(self, streams=None):
        streams = range(len(self.model)) if streams is None else streams
        for k, ref in enumerate(self.refs):
            sk = [s for s in streams if self.model[s] == k]
            if sk:
                assert np.array_equal(self.bank.export_streams(sk), ref.export_streams(sk)), f"model {k}: records differ"

    def check_oracle(self, streams):
        for s in streams:
            if self.ins[s]:
                ref = _oracle_stream(self.docs[self.model[s]], self.ins[s], self.block)
                err = float(np.max(np.abs(np.concatenate(self.outs[s]) - ref)))
                assert err <= TOL, f"stream {s} (model {self.model[s]}): {err:.3e} from the oracle"

    def close(self):
        self.bank.close()
        for r in self.refs:
            r.close()


@pytest.mark.parametrize("shape,k", [("wavenet", 3), ("a1", 4), ("a2_lite", 5)])
def test_seeded_schedules_match_each_models_handle_and_the_oracle(shape, k):
    B, block = 12, 512
    rig = Rig(_family(shape, k, seed=1), B, block)
    rig.assign(list(range(B)), [s % k for s in range(B)])  # interleaved: short-geometry slots mix models
    rng = np.random.default_rng(7)
    pool = [0, 1, 37, 63, 64, 65, 127, 128, 129, 300, 512]
    for c in range(6):
        n = int(rng.integers(2, B + 1))
        streams = [int(v) for v in rng.permutation(B)[:n]]
        counts = [int(v) for v in rng.choice(pool, size=n)] if c % 2 else [int(rng.choice(pool[1:]))] * n
        counts[0] = max(counts[0], 1)
        rig.call(streams, counts, seed=100 + c)
    rig.check_records()
    rig.check_oracle([0, 1, 2, B - 1])
    rig.close()


# (name, batch, max_frames, counts of one call, options, $NAM_B200_LAT_KERNEL)
PATHS = [
    ("short64", 16, 64, [64] * 16, {}, "off"),
    ("short128", 16, 128, [128, 100] * 8, {}, "off"),
    ("small128x1", 5, 128, [128, 64, 1, 0, 99], {}, "off"),
    ("persistent256x2", 12, 1024, [1024] * 6 + [700] * 6, {"tile_mode": 2}, None),
    ("persistent128x2", 12, 1024, [1024, 513] * 6, {"tile_mode": 2, "kernel_geometry": 1}, None),
    ("lockstep", 3, 4096, [4096, 1000, 0], {}, None),
    ("wavefront", 3, 2048, [2048, 1500, 600], {"tile_mode": 1}, None),
    ("lat2", 6, 64, [64, 64, 33, 0, 64, 1], {}, "precompiled"),
]


@pytest.mark.parametrize("name,batch,block,counts,kw,lat", PATHS, ids=[p[0] for p in PATHS])
def test_every_kernel_path_with_mixed_models(name, batch, block, counts, kw, lat, monkeypatch):
    if lat is not None:
        monkeypatch.setenv("NAM_B200_LAT_KERNEL", lat)
    k = 3
    rig = Rig(_family("a1", k, seed=2), batch, block, **kw)
    models = [s % k for s in range(batch)]
    if batch >= 8:
        models[:4] = [1, 1, 1, 1]  # one homogeneous slot of four streams
    rig.assign(list(range(batch)), models)
    for c in range(2):
        rig.call(list(range(batch)), counts, seed=300 + c)
        rig.call(list(range(batch))[::-1], counts[::-1], seed=310 + c)
    rig.check_records()
    rig.check_oracle([0, 1, batch - 1])
    rig.close()


def test_pipelined_host_path_on_pinned_buffers():
    """Large host-buffer calls are split into chunks of streams, each a sub-range of the bank's table"""
    B, n, k = 2200, 1024, 3
    rig = Rig(_family("a1", k, seed=3), B, n)
    rig.assign(list(range(B)), [s % k for s in range(B)])
    lib = _capi.load()
    x = fx.synthetic_batch(B, n, seed=9)
    y = np.empty_like(x)
    assert lib.nam_b200_pin_host_buffer(x.ctypes.data, x.nbytes) == 0
    assert lib.nam_b200_pin_host_buffer(y.ctypes.data, y.nbytes) == 0
    try:
        before = rig.bank.launch_count()
        rig.bank.process_batch(x, y)
        assert rig.bank.launch_count() - before >= 2  # (one launch per chunk)
        for kk, ref in enumerate(rig.refs):
            rows = [s for s in range(B) if rig.model[s] == kk]
            yk = ref.process_batch(x)
            assert np.array_equal(y[rows], yk[rows])
    finally:
        lib.nam_b200_unpin_host_buffer(x.ctypes.data)
        lib.nam_b200_unpin_host_buffer(y.ctypes.data)
    for s in (0, 1, 2, B - 1):
        ref = _oracle_stream(rig.docs[rig.model[s]], [x[s]], n)
        assert float(np.max(np.abs(y[s] - ref))) <= TOL
    rig.check_records([0, 1, 2, 1000, B - 1])
    rig.close()


def test_planar_process_runs_stream_0s_model():
    rig = Rig(_family("wavenet", 3, seed=4), 2, 64)
    rig.assign([0], [2])
    x = fx.synthetic_batch(1, 256, seed=11)[0].astype(np.float64)
    for c in range(4):
        chunk = x[64 * c:64 * (c + 1)]
        ya, yb = np.zeros(64), np.zeros(64)
        rig.bank.process([chunk], [ya], 64)
        rig.refs[2].process([chunk], [yb], 64)
        assert np.array_equal(ya, yb)
    rig.close()


def test_reset_gives_each_stream_its_models_fresh_state():
    B, k = 6, 3
    docs = _family("a1", k, seed=5)
    rig = Rig(docs, B, 256)
    rig.assign(list(range(B)), [2, 0, 1, 2, 1, 0])
    rig.call(list(range(B)), [256] * B, seed=1)
    rig.bank.Reset(48000.0, 256)
    for s in range(B):
        fresh = nb.get_dsp(docs[rig.model[s]], batch=1, jit=2)
        fresh.Reset(48000.0, 256)
        assert np.array_equal(rig.bank.export_streams([s]), fresh.export_streams([0])), f"stream {s}"
        fresh.close()
    assert list(rig.bank.stream_models(range(B))) == [2, 0, 1, 2, 1, 0]
    rig.close()


def test_assign_moves_one_stream_and_leaves_the_others_bit_identical():
    B, k = 6, 3
    rig = Rig(_family("a1", k, seed=6), B, 256)
    rig.call(list(range(B)), [256] * B, seed=2)
    before = rig.bank.export_streams(range(B))
    rig.assign([3], [2])
    after = rig.bank.export_streams(range(B))
    for s in range(B):
        if s != 3:
            assert np.array_equal(before[s], after[s])
    assert np.array_equal(after[3], rig.refs[2].export_streams([3])[0])
    rig.call([3, 0], [256, 128], seed=3)
    rig.check_records()
    rig.check_oracle([3, 0])
    # reset_streams returns a stream to its current model's fresh state
    rig.bank.reset_streams([3])
    rig.refs[2].reset_streams([3])
    rig.check_records([3])
    rig.close()


def test_assign_refusals_name_the_entry():
    docs = _family("wavenet", 3)
    bank = nb.get_dsp_bank(docs, batch=4)
    with pytest.raises(RuntimeError, match="before reset"):
        bank.assign_streams([0], [1])
    bank.Reset(48000.0, 64)
    with pytest.raises(ValueError, match=r"models\[1\] = 3"):
        bank.assign_streams([0, 1], [1, 3])
    with pytest.raises(ValueError, match=r"models\[0\] = -1"):
        bank.assign_streams([2], [-1])
    with pytest.raises(ValueError, match=r"streams\[1\] = 0: duplicate"):
        bank.assign_streams([0, 0], [1, 2])
    with pytest.raises(ValueError, match="stream index outside"):
        bank.assign_streams([4], [1])
    assert list(bank.stream_models(range(4))) == [0, 0, 0, 0]
    bank.close()


def test_records_move_between_a_bank_and_ordinary_handles():
    k = 3
    docs = _family("a1", k, seed=7)
    rig = Rig(docs, 6, 256)
    rig.assign([1, 4], [1, 2])
    rig.call([1, 4], [256, 200], seed=4)
    # bank -> ordinary handle of the stream's model -> both continue identically
    one = nb.get_dsp(docs[1], batch=2, jit=2)
    one.Reset(48000.0, 256)
    one.import_streams([0], rig.bank.export_streams([1]))
    x = fx.synthetic_batch(1, 256, seed=5)
    ya = rig.bank.process_streams([1], x)
    yb = one.process_streams([0], x)
    assert np.array_equal(ya, yb)
    assert np.array_equal(rig.bank.export_streams([1]), one.export_streams([0]))
    # ordinary handle -> bank: the record of model 2 rebinds the stream to model 2
    two = nb.get_dsp(docs[2], batch=1, jit=2)
    two.Reset(48000.0, 256)
    two.process_streams([0], fx.synthetic_batch(1, 256, seed=6))
    rec = two.export_streams([0])
    rig.bank.import_streams([5], rec)
    assert list(rig.bank.stream_models([5])) == [2]
    x = fx.synthetic_batch(1, 128, seed=7)
    assert np.array_equal(rig.bank.process_streams([5], x), two.process_streams([0], x))
    assert np.array_equal(rig.bank.export_streams([5]), two.export_streams([0]))
    # a record of a model outside the bank is refused, naming the fingerprint
    other = nb.get_dsp(_family("a1", 4, seed=8)[3], batch=1, jit=2)
    other.Reset(48000.0, 256)
    with pytest.raises(ValueError, match="none of the 3 models of this bank"):
        rig.bank.import_streams([0], other.export_streams([0]))
    for h in (one, two, other):
        h.close()
    rig.close()


def test_duplicate_documents_import_to_the_lowest_index():
    docs = _family("wavenet", 2)
    bank = nb.get_dsp_bank([docs[0], docs[1], docs[1]], batch=3)
    bank.Reset(48000.0, 64)
    bank.assign_streams([2], [2])
    bank.import_streams([0], bank.export_streams([2]))
    assert list(bank.stream_models([0, 2])) == [1, 2]
    bank.close()


def test_copy_streams_carries_the_binding():
    rig = Rig(_family("a1", 3, seed=9), 4, 256)
    rig.assign([0, 1, 2], [1, 2, 0])
    rig.call([0, 1, 2], [256, 256, 256], seed=8)
    rec = rig.bank.export_streams([0, 1])
    rig.bank.copy_streams([0], [3])
    assert list(rig.bank.stream_models([3])) == [1]
    assert np.array_equal(rig.bank.export_streams([3])[0], rec[0])
    rig.bank.copy_streams([0, 1], [1, 0])  # swap
    assert list(rig.bank.stream_models([0, 1])) == [2, 1]
    assert np.array_equal(rig.bank.export_streams([1, 0]), rec)
    rig.bank.close()
    for r in rig.refs:
        r.close()


def test_ordinary_handles_are_banks_of_one():
    docs = _family("a1", 1)
    a, b = nb.get_dsp(docs[0], batch=4, jit=2), nb.get_dsp(docs[0], batch=4, jit=2)
    for h in (a, b):
        h.Reset(48000.0, 256)
        h.process_batch(fx.synthetic_batch(4, 256, seed=12))
    assert a.bank_size == 1 and list(a.stream_models(range(4))) == [0] * 4
    na, nb_ = a.launch_count(), b.launch_count()
    a.assign_streams([2, 0], [0, 0])
    b.reset_streams([2, 0])
    assert a.launch_count() - na == b.launch_count() - nb_
    assert np.array_equal(a.export_streams(range(4)), b.export_streams(range(4)))
    with pytest.raises(ValueError, match=r"models\[0\] = 1"):
        a.assign_streams([1], [1])
    # a bank of one document is the ordinary handle
    one = nb.get_dsp_bank(docs, batch=4, jit=2)
    one.Reset(48000.0, 256)
    assert one.bank_size == 1
    x = fx.synthetic_batch(4, 256, seed=13)
    b.Reset(48000.0, 256)
    assert np.array_equal(one.process_batch(x), b.process_batch(x))
    for h in (a, b, one):
        h.close()


def test_bank_jit_note_and_model_info():
    docs = _family("a1", 3, seed=10)
    bank = nb.get_dsp_bank(docs, batch=4, jit=3)
    bank.Reset(48000.0, 128)
    assert bank.bank_size == 3
    assert "model bank" in bank.jit_note()
    fields = [f for f, _ in nb._capi.Info._fields_ if f not in ("struct_size", "reserved")]
    for k, d in enumerate(docs):
        ref = nb.get_dsp(d, batch=4, jit=2)
        ref.Reset(48000.0, 128)
        got, want = bank.model_info(k), ref.info
        for f in fields:
            assert getattr(got, f) == getattr(want, f), (k, f)
        ref.close()
    with pytest.raises(ValueError, match="outside"):
        bank.model_info(3)
    bank.close()
