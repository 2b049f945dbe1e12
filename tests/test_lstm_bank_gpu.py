"""GPU tests of LSTM model banks: one handle whose streams each run their own LSTM capture of one shape.  The yardstick is
one ordinary jit = 2 handle per model, given every call the bank gets (reset_streams(fresh=True) on it is the counterpart of
assign_streams): each bank stream's outputs and records must match, byte for byte, the same stream index on the handle of
its model, and sampled streams must be within 1e-5 of the oracle for their model, fed the same calls, Resets and prewarms.

The shapes cover every LSTM kernel: lane groups of G = 4 / 8 / 16 / 32 (lstm_group.cuh; at H = 64 at most 3 models' weights
fit in one CTA's shared memory, so a CTA of 4 streams with 4 models makes two passes) and one thread per stream (H = 70, and
a 2-in / 3-out cell), where a CTA makes one pass per distinct model.  The random cells expect 4 kHz, so that their
prewarm (half a second of samples, lstm.cpp:127-134) stays short on the slow thread-per-stream kernel."""
import copy

import numpy as np
import pytest

import neuralampmodelercore_b200 as nb
from oracle import nam_config, oracle
from tests import nam_fixtures as fx

pytestmark = pytest.mark.gpu
TOL = 1e-5


def _lstm(H, nl, seed, in_ch=1, out_ch=1) -> dict:
    config = {"input_size": in_ch, "hidden_size": H, "num_layers": nl}
    if in_ch != 1 or out_ch != 1:
        config.update(in_channels=in_ch, out_channels=out_ch)
    nam = {"version": "0.5.4", "architecture": "LSTM", "sample_rate": 4000.0, "config": config, "weights": []}
    n = nam_config.expected_weight_count(nam)
    nam["weights"] = [float(v) for v in np.random.default_rng(seed).uniform(-0.4, 0.4, n)]
    return nam


# shape -> (hidden, layers, in, out); "lstm" is the example capture, reweighted per model
SHAPES = {"lstm": None, "h5": (5, 2, 1, 1), "h16": (16, 2, 1, 1), "h64": (64, 1, 1, 1), "h70": (70, 1, 1, 1),
          "2in3out": (5, 2, 2, 3)}


def _family(shape: str, k: int, seed: int = 0) -> list:
    """k documents of one shape, every weight (h0 / c0 and the head included) different per model"""
    if SHAPES[shape] is None:
        base = fx.load_model("lstm")
        docs = []
        for i in range(k):
            d = copy.deepcopy(base)
            rng = np.random.default_rng(1000 * seed + i)
            w = np.asarray(base["weights"], np.float32)
            d["weights"] = [float(v) for v in w * (1.0 + 0.1 * rng.standard_normal(w.shape)).astype(np.float32)]
            docs.append(d)
        return docs
    H, nl, ci, co = SHAPES[shape]
    return [_lstm(H, nl, 1000 * seed + i, ci, co) for i in range(k)]


def _oracle(doc, events, block, prewarm=True):
    """One oracle instance fed a stream's history since it was bound: arrays are process calls ([n] or [channels, n]),
    "reset" is a Reset after history (an LSTM keeps h, c and prewarms on top), None a standalone prewarm."""
    m = oracle.OracleModel.from_dict(doc)
    m.reset(48000.0, block, prewarm=prewarm)
    ys = []
    for e in events:
        if e is None:
            for _ in range(0, m.prewarm_samples, block):
                m.process(np.zeros((m.in_channels, block), np.float32))
        elif isinstance(e, str):
            m.reset(48000.0, block, prewarm=prewarm)
        else:
            y = m.process(np.ascontiguousarray(e))
            ys.append(np.atleast_2d(y) if e.ndim == 2 else np.asarray(y).reshape(-1))
    m.close()
    return np.concatenate(ys, axis=-1) if ys else None


class Rig:
    """A bank and its yardstick handles, plus each stream's history since it was last bound (for the oracle)."""

    def __init__(self, docs, batch, block, **kw):
        self.docs, self.block, self.kw = docs, block, kw
        self.bank = nb.get_dsp_bank(docs, batch=batch, **kw)
        self.bank.Reset(48000.0, block)
        self.refs = []
        for d in docs:
            r = nb.get_dsp(d, batch=batch, **dict(kw, jit=2))
            r.Reset(48000.0, block)
            self.refs.append(r)
        self.ci, self.co = self.bank.in_channels, self.bank.out_channels
        self.model = np.zeros(batch, np.int64)
        self.events = {s: [] for s in range(batch)}
        self.outs = {s: [] for s in range(batch)}

    def _rebound(self, s):
        self.events[s], self.outs[s] = [], []

    def assign(self, streams, models):
        self.bank.assign_streams(streams, models)
        for k in sorted(set(int(v) for v in models)):
            self.refs[k].reset_streams([s for s, kk in zip(streams, models) if kk == k], fresh=True)
        for s, k in zip(streams, models):
            self.model[s] = k
            self._rebound(s)
        assert list(self.bank.stream_models(streams)) == list(models)

    def reset_streams(self, streams, fresh):
        self.bank.reset_streams(streams, fresh=fresh)
        for k in sorted(set(int(self.model[s]) for s in streams)):
            self.refs[k].reset_streams([s for s in streams if self.model[s] == k], fresh=fresh)
        for s in streams:
            if fresh:
                self._rebound(s)
            else:
                self.events[s].append("reset")

    def reset(self):
        for h in [self.bank] + self.refs:
            h.Reset(48000.0, self.block)
        for s in self.events:
            self.events[s].append("reset")

    def prewarm(self):
        for h in [self.bank] + self.refs:
            h.prewarm()
        for s in self.events:
            self.events[s].append(None)

    def input(self, n, frames, seed):
        x = fx.synthetic_batch(n * self.ci, max(frames, 1), seed=seed)[:, :frames]
        return np.ascontiguousarray(x.reshape(n, self.ci, frames) if self.ci > 1 else x)

    def call(self, streams, counts, seed):
        """A ragged process_streams call on the bank and the same call on every yardstick handle"""
        x = self.input(len(streams), max(counts), seed)
        for i, c in enumerate(counts):
            x[i, ..., c:] = 0.0
        y = self.bank.process_streams(streams, x, n_frames=counts)
        for k, ref in enumerate(self.refs):
            rows = [i for i, s in enumerate(streams) if self.model[s] == k]
            if rows:
                yk = ref.process_streams(streams, x, n_frames=counts)
                assert np.array_equal(y[rows], yk[rows]), f"model {k}: outputs differ from its ordinary handle"
        for i, (s, c) in enumerate(zip(streams, counts)):
            if c:
                self.events[s].append(x[i, ..., :c].copy())
                self.outs[s].append(y[i, ..., :c].copy())
        return y

    def call_batch(self, frames, seed):
        """A contiguous process_batch call over every stream: the same launches as the yardstick's call"""
        B = len(self.model)
        x = self.input(B, frames, seed)
        before = self.bank.launch_count()
        y = self.bank.process_batch(x)
        launches = self.bank.launch_count() - before
        for k, ref in enumerate(self.refs):
            rows = [s for s in range(B) if self.model[s] == k]
            if rows:
                before = ref.launch_count()
                yk = ref.process_batch(x)
                assert ref.launch_count() - before == launches
                assert np.array_equal(y[rows], yk[rows]), f"model {k}: outputs differ from its ordinary handle"
        for s in range(B):
            self.events[s].append(x[s].copy())
            self.outs[s].append(y[s].copy())

    def check_records(self, streams=None):
        streams = range(len(self.model)) if streams is None else streams
        for k, ref in enumerate(self.refs):
            sk = [s for s in streams if self.model[s] == k]
            if sk:
                assert np.array_equal(self.bank.export_streams(sk), ref.export_streams(sk)), f"model {k}: records differ"

    def check_oracle(self, streams):
        prewarm = self.kw.get("prewarm", True) is not False
        for s in streams:
            if self.outs[s]:
                ref = _oracle(self.docs[self.model[s]], self.events[s], self.block, prewarm)
                err = float(np.max(np.abs(np.concatenate(self.outs[s], axis=-1) - ref)))
                assert err <= TOL, f"stream {s} (model {self.model[s]}): {err:.3e} from the oracle"

    def close(self):
        for h in [self.bank] + self.refs:
            h.close()


BINDINGS = {
    "grouped": lambda B, k: [s * k // B for s in range(B)],
    "round_robin": lambda B, k: [s % k for s in range(B)],
    "scattered": lambda B, k: [int(v) for v in np.random.default_rng(5).integers(0, k, B)],
}


@pytest.mark.parametrize("binding", sorted(BINDINGS))
@pytest.mark.parametrize("shape", list(SHAPES))
def test_seeded_schedules_match_each_models_handle_and_the_oracle(shape, binding):
    B, block, k = 70, 128, 4  # 70 streams: full and partial CTAs of every kernel
    rig = Rig(_family(shape, k, seed=1), B, block)
    models = BINDINGS[binding](B, k)
    rig.assign(list(range(B)), models)
    rng = np.random.default_rng(7)
    pool = [0, 1, 37, 64, 100, block]
    for c in range(5):
        n = int(rng.integers(2, B + 1))
        streams = [int(v) for v in rng.permutation(B)[:n]]
        counts = [int(v) for v in rng.choice(pool, size=n)] if c % 2 else [int(rng.choice(pool[1:]))] * n
        counts[0] = max(counts[0], 1)
        rig.call(streams, counts, seed=100 + c)
    rig.call_batch(block, seed=200)
    rig.check_records()
    rig.check_oracle(sorted({0, 1, 33, B - 1} | {models.index(m) for m in set(models)}))
    rig.close()


@pytest.mark.parametrize("shape,k", [("lstm", 40), ("h16", 8), ("2in3out", 9)])
def test_many_models_round_robin(shape, k):
    """lstm.nam: a CTA of 32 streams holds 32 models' copies at once; H = 16: 8 copies of ~3.3k floats; 2-in/3-out: the
    thread-per-stream kernel makes 9 passes per CTA"""
    B, block = 70, 64
    rig = Rig(_family(shape, k, seed=2), B, block)
    rig.assign(list(range(B)), [s % k for s in range(B)])
    rig.call(list(range(B)), [block] * B, seed=1)
    rig.call(list(range(B))[::-1], [(7 * s) % (block + 1) for s in range(B)], seed=2)
    rig.check_records()
    rig.check_oracle([0, 1, k - 1, B - 1])
    rig.close()


@pytest.mark.parametrize("shape", ["lstm", "h64", "h70", "2in3out"])
def test_lifecycle_reset_reset_streams_assign_prewarm(shape):
    B, block, k = 12, 128, 3
    rig = Rig(_family(shape, k, seed=3), B, block)
    rig.assign(list(range(B)), [s % k for s in range(B)])
    rig.call(list(range(B)), [block] * B, seed=1)
    rig.call([5, 0, 7, 2], [block, 37, 0, 1], seed=2)
    rig.reset()  # a second Reset after history: each stream keeps h, c and is prewarmed on top with its own model
    rig.call(list(range(B)), [block] * B, seed=3)
    rig.check_records()
    rig.reset_streams([1, 5], fresh=False)
    rig.reset_streams([2, 7], fresh=True)
    rig.check_records([1, 2, 5, 7])
    rig.call(list(range(B)), [100] * B, seed=4)
    rig.assign([3], [(rig.model[3] + 1) % k])  # to another model and back
    rig.call([3, 4], [block, block], seed=5)
    rig.assign([3], [0])
    rig.call([3, 4], [64, block], seed=6)
    rig.prewarm()  # standalone: every stream with its own model, from its current state
    rig.call(list(range(B)), [block] * B, seed=7)
    rig.check_records()
    rig.check_oracle(list(range(B)))
    # the runtime fast-tanh switch: calls, and the fresh state reset_streams / assign_streams hand out, as on the yardstick
    for h in [rig.bank] + rig.refs:
        h.set_fast_tanh(True)
    rig.call(list(range(B)), [block] * B, seed=8)
    rig.reset_streams([4, 9], fresh=True)
    rig.assign([6], [(rig.model[6] + 2) % k])
    rig.call(list(range(B)), [block] * B, seed=9)
    rig.check_records()
    for h in [rig.bank] + rig.refs:
        h.set_fast_tanh(False)
    rig.reset_streams([4], fresh=True)
    rig.call([4, 6], [block, block], seed=10)
    rig.check_records()
    rig.close()


@pytest.mark.parametrize("shape", ["lstm", "h70"])
def test_without_prewarm_each_stream_starts_from_its_models_initial_state(shape):
    B, block, k = 10, 64, 3
    rig = Rig(_family(shape, k, seed=4), B, block, prewarm=False)
    rig.call([0, 1], [block, block], seed=1)  # bound to model 0 since creation: model 0's h0 / c0
    rig.assign(list(range(2, B)), [s % k for s in range(2, B)])
    rig.call(list(range(B)), [block] * B, seed=2)
    rig.reset()
    rig.reset_streams([3], fresh=False)
    rig.reset_streams([4], fresh=True)
    rig.call(list(range(B)), [block] * B, seed=3)
    rig.check_records()
    rig.check_oracle(list(range(B)))
    rig.close()


def test_records_move_between_a_bank_and_ordinary_handles():
    k, block = 3, 128
    docs = _family("lstm", k, seed=5)
    rig = Rig(docs, 6, block)
    rig.assign([1, 4], [1, 2])
    rig.call([1, 4], [block, 100], seed=1)
    # bank -> ordinary handle of the stream's model -> both continue identically
    one = nb.get_dsp(docs[1], batch=2, jit=2)
    one.Reset(48000.0, block)
    one.import_streams([0], rig.bank.export_streams([1]))
    x = fx.synthetic_batch(1, block, seed=2)
    assert np.array_equal(rig.bank.process_streams([1], x), one.process_streams([0], x))
    assert np.array_equal(rig.bank.export_streams([1]), one.export_streams([0]))
    # ordinary handle -> bank: the record of model 2 rebinds the stream to model 2
    two = nb.get_dsp(docs[2], batch=1, jit=2)
    two.Reset(48000.0, block)
    two.process_streams([0], fx.synthetic_batch(1, block, seed=3))
    rig.bank.import_streams([5], two.export_streams([0]))
    assert list(rig.bank.stream_models([5])) == [2]
    x = fx.synthetic_batch(1, 77, seed=4)
    assert np.array_equal(rig.bank.process_streams([5], x), two.process_streams([0], x))
    assert np.array_equal(rig.bank.export_streams([5]), two.export_streams([0]))
    # a record of a model outside the bank is refused, naming the fingerprint
    other = nb.get_dsp(_family("lstm", 4, seed=6)[3], batch=1, jit=2)
    other.Reset(48000.0, block)
    with pytest.raises(ValueError, match="none of the 3 models of this bank"):
        rig.bank.import_streams([0], other.export_streams([0]))
    for h in (one, two, other):
        h.close()
    rig.close()


def test_copy_streams_carries_the_binding_and_zero_frame_positions_keep_their_state():
    rig = Rig(_family("h16", 3, seed=7), 5, 128)
    rig.assign([0, 1, 2], [1, 2, 0])
    rig.call([0, 1, 2], [128, 128, 128], seed=1)
    rec = rig.bank.export_streams([0, 1])
    rig.bank.copy_streams([0], [3])
    assert list(rig.bank.stream_models([3])) == [1]
    assert np.array_equal(rig.bank.export_streams([3])[0], rec[0])
    rig.bank.copy_streams([0, 1], [1, 0])  # swap
    assert list(rig.bank.stream_models([0, 1])) == [2, 1]
    assert np.array_equal(rig.bank.export_streams([1, 0]), rec)
    # a copied stream runs its source's model: it continues like the source on that model's handle
    x = fx.synthetic_batch(1, 128, seed=2)
    one = nb.get_dsp(rig.docs[1], batch=1, jit=2)
    one.Reset(48000.0, 128)
    one.import_streams([0], rec[:1])
    assert np.array_equal(rig.bank.process_streams([3], x), one.process_streams([0], x))
    # positions with 0 frames keep their state bit for bit, whatever their CTA mates run
    before = rig.bank.export_streams(range(5))
    rig.bank.process_streams([4, 2, 1], np.ones((3, 90), np.float32), n_frames=[90, 0, 0])
    after = rig.bank.export_streams(range(5))
    for s in (0, 1, 2, 3):
        assert np.array_equal(before[s], after[s]), s
    assert not np.array_equal(before[4], after[4])
    one.close()
    rig.bank.close()
    for r in rig.refs:
        r.close()


def test_default_jit_bank_runs_the_precompiled_kernels():
    docs = _family("lstm", 3, seed=8)
    bank = nb.get_dsp_bank(docs, batch=256)  # (an ordinary handle of this batch would compile lstm_spec kernels)
    bank.Reset(48000.0, 64)
    note = bank.jit_note()
    assert "model bank" in note and "precompiled" in note, note
    ref = nb.get_dsp(docs[0], batch=256, jit=2)
    ref.Reset(48000.0, 64)
    x = fx.synthetic_batch(256, 64, seed=9)
    assert np.array_equal(bank.process_batch(x), ref.process_batch(x))
    bank.close()
    ref.close()


@pytest.mark.parametrize("shape", ["lstm", "h70"])
def test_ordinary_lstm_without_prewarm_starts_every_stream_from_h0_c0(shape):
    """Every reference DSP object starts from the trained h0 / c0 (lstm.cpp:24-28), also when Reset runs no prewarm"""
    doc = _family(shape, 1, seed=9)[0] if shape != "lstm" else fx.load_model("lstm")
    B, block = 4, 64
    d = nb.get_dsp(doc, batch=B, prewarm=False)
    d.Reset(48000.0, block)
    x = fx.synthetic_batch(B, 256, seed=10)
    got = np.concatenate([d.process_batch(np.ascontiguousarray(x[:, p:p + block])) for p in range(0, 256, block)], axis=1)
    for s in range(B):
        ref = _oracle(doc, [x[s, p:p + block] for p in range(0, 256, block)], block, prewarm=False)
        assert float(np.max(np.abs(got[s] - ref))) <= TOL, s
    d.close()
