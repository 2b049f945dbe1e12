"""GPU tests of model banks of general-kernel WaveNets and of ConvNets.  The yardstick is test_bank_gpu's: one ordinary
jit = 2 handle per model, given every call the bank gets; each bank stream's outputs and records must match the same stream
of its model's handle byte for byte, and each stream must be within 1e-5 of the oracle for its model."""
import copy

import numpy as np
import pytest

import neuralampmodelercore_b200 as nb
from tests import nam_fixtures as fx
from tests.test_bank_gpu import Rig
from tests.test_multichannel_gpu import _randomise, _signal, _wavenet_2in_3out
from tests.test_process_streams_gpu import TOL, _oracle_stream
from tests.test_reference_build import _convnet

pytestmark = pytest.mark.gpu


def _reweighted(base: dict, k: int, seed: int) -> list:
    docs = []
    for i in range(k):
        d = copy.deepcopy(base)
        w = np.asarray(base["weights"], np.float32)
        rng = np.random.default_rng(1000 * seed + i)
        d["weights"] = [float(v) for v in w * (1.0 + 0.05 * rng.standard_normal(w.shape)).astype(np.float32)]
        cd = d["config"].get("condition_dsp")
        if cd:  # the nested document's weights (its head_scale, the last one, too) are per model as well
            wc = np.asarray(cd["weights"], np.float32)
            cd["weights"] = [float(v) for v in wc * (1.0 + 0.05 * rng.standard_normal(wc.shape)).astype(np.float32)]
        d["metadata"] = dict(d.get("metadata") or {}, loudness=-20.0 - i)
        docs.append(d)
    return docs


def _wide_general():
    """a general-kernel WaveNet (gated, bottleneck != channels) whose blob exceeds the 200 KB the kernel stages in shared
    memory: the read-only path"""
    layer = {"input_size": 1, "condition_size": 1, "head_size": 1, "channels": 64, "bottleneck": 32, "kernel_size": 3,
             "dilations": [1, 2, 4, 8, 16], "activation": "Tanh", "gated": True, "head_bias": False}
    return _randomise(fx.make_wavenet_nam([layer], []), seed=3, scale=0.08, last=0.7)


def family(shape: str, k: int, seed: int = 0) -> list:
    if shape == "convnet":
        return [_convnet(6, [1, 2, 4, 8], True, "Tanh", 10 * seed + i) for i in range(k)]
    if shape == "mc":
        return [_randomise(_wavenet_2in_3out(), seed=20 * seed + i, last=0.5 + 0.1 * i) for i in range(k)]
    base = {"a2_max": lambda: fx.load_model("wavenet_a2_max"), "cond": lambda: fx.load_model("wavenet_condition_dsp"),
            "wide": _wide_general}[shape]()
    return _reweighted(base, k, seed)


class GRig(Rig):
    """Rig for mono and multi-channel models: inputs [n, in_channels, frames] when the model has several channels"""

    def __init__(self, docs, batch, block, **kw):
        super().__init__(docs, batch, block, **kw)
        self.ci = self.bank.in_channels

    def _input(self, n, frames, seed):
        if self.ci == 1:
            return fx.synthetic_batch(n, frames, seed=seed)
        return _signal(n, self.ci, frames, seed)

    def call(self, streams, counts, seed):
        n_max = max(counts)
        x = self._input(len(streams), max(n_max, 1), seed)[..., :n_max].copy()
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
                self.ins[s].append(x[i, ..., :c].copy())
                self.outs[s].append(y[i, ..., :c].copy())
        return y

    def contiguous(self, seed):
        """a process_batch call over every stream (the bank's identity table), the same on every yardstick"""
        B = len(self.model)
        x = self._input(B, self.block, seed)
        y = self.bank.process_batch(x)
        for k, ref in enumerate(self.refs):
            rows = [s for s in range(B) if self.model[s] == k]
            if rows:
                assert np.array_equal(y[rows], ref.process_batch(x)[rows]), f"model {k}: contiguous call differs"
        for s in range(B):
            self.ins[s].append(x[s].copy())
            self.outs[s].append(y[s].copy())

    def check_oracle(self, streams):
        for s in streams:
            if self.ins[s]:
                ref = _oracle_stream(self.docs[self.model[s]], self.ins[s], self.block)
                err = float(np.max(np.abs(np.concatenate(self.outs[s], axis=-1) - ref)))
                assert err <= TOL, f"stream {s} (model {self.model[s]}): {err:.3e} from the oracle"


def _binding(kind: str, B: int, K: int) -> list:
    if kind == "grouped":
        return [min(s * K // B, K - 1) for s in range(B)]
    if kind == "round_robin":
        return [s % K for s in range(B)]
    return [int(v) for v in np.random.default_rng(5).integers(0, K, size=B)]  # scattered


@pytest.mark.parametrize("binding", ["grouped", "round_robin", "scattered"])
@pytest.mark.parametrize("shape", ["a2_max", "cond", "mc", "convnet"])
def test_streams_match_their_models_handles_and_the_oracle(shape, binding):
    B, K, block = 10, 3, 256
    rig = GRig(family(shape, K, seed=1), B, block)
    rig.assign(list(range(B)), _binding(binding, B, K))
    rng = np.random.default_rng(11)
    for c in range(3):
        streams = [int(v) for v in rng.permutation(B)[:int(rng.integers(4, B + 1))]]
        counts = [int(v) for v in rng.choice([0, 1, 64, 127, 128, 129, 256], size=len(streams))]
        counts[0] = max(counts[0], 1)
        rig.call(streams, counts, seed=200 + c)
    rig.contiguous(seed=210)
    rig.check_records()
    rig.check_oracle([0, B // 2, B - 1])
    rig.close()


@pytest.mark.parametrize("shape", ["a2_max", "convnet"])
def test_reset_prewarm_reset_streams_and_assignment(shape):
    B, K, block = 6, 3, 128
    docs = family(shape, K, seed=2)
    rig = GRig(docs, B, block)
    models = [2, 0, 1, 2, 1, 0]
    rig.assign(list(range(B)), models)
    rig.call(list(range(B)), [block] * B, seed=1)
    # a second Reset: every stream in the fresh state of its own model
    rig.bank.Reset(48000.0, block)
    for s in range(B):
        fresh = nb.get_dsp(docs[models[s]], batch=1, jit=2)
        fresh.Reset(48000.0, block)
        assert np.array_equal(rig.bank.export_streams([s]), fresh.export_streams([0])), f"stream {s}"
        fresh.close()
    for ref in rig.refs:
        ref.Reset(48000.0, block)
    rig.ins = {s: [] for s in range(B)}
    rig.outs = {s: [] for s in range(B)}
    rig.call(list(range(B)), [block, 0, 77, block, 1, block], seed=2)
    # a standalone prewarm runs every stream from its current state with its own model
    rig.bank.prewarm()
    for ref in rig.refs:
        ref.prewarm()
    rig.check_records()
    # reset_streams, and assignment away and back
    rig.bank.reset_streams([0, 4])
    for s in (0, 4):
        rig.refs[rig.model[s]].reset_streams([s])
    rig.check_records()
    rig.assign([1, 3], [2, 0])
    rig.call([1, 3, 5], [block, 100, block], seed=3)
    rig.assign([1, 3], [0, 2])
    rig.call([1, 3], [block, block], seed=4)
    rig.check_records()
    rig.check_oracle([1, 3])
    rig.close()


def test_records_move_between_a_bank_and_ordinary_handles_and_copies_carry_the_binding():
    K, block = 3, 256
    docs = family("cond", K, seed=3)
    rig = GRig(docs, 6, block)
    rig.assign([1, 4], [1, 2])
    rig.call([1, 4], [block, 200], seed=4)
    one = nb.get_dsp(docs[1], batch=2, jit=2)
    one.Reset(48000.0, block)
    one.import_streams([0], rig.bank.export_streams([1]))
    x = fx.synthetic_batch(1, block, seed=5)
    assert np.array_equal(rig.bank.process_streams([1], x), one.process_streams([0], x))
    assert np.array_equal(rig.bank.export_streams([1]), one.export_streams([0]))
    two = nb.get_dsp(docs[2], batch=1, jit=2)
    two.Reset(48000.0, block)
    two.process_streams([0], fx.synthetic_batch(1, block, seed=6))
    rig.bank.import_streams([5], two.export_streams([0]))
    assert list(rig.bank.stream_models([5])) == [2]
    x = fx.synthetic_batch(1, 128, seed=7)
    assert np.array_equal(rig.bank.process_streams([5], x), two.process_streams([0], x))
    # copies carry the binding
    rec = rig.bank.export_streams([5])
    rig.bank.copy_streams([5], [0])
    assert list(rig.bank.stream_models([0])) == [2]
    assert np.array_equal(rig.bank.export_streams([0]), rec)
    x = fx.synthetic_batch(2, 128, seed=8)
    y = rig.bank.process_streams([0, 5], x)
    assert np.array_equal(y[:1], two.process_streams([0], x[:1]))
    for h in (one, two):
        h.close()
    rig.close()


def test_kernel_geometry_4_and_the_default_jit():
    B, K, block = 8, 3, 256
    docs = family("a2_max", K, seed=4)
    rig = GRig(docs, B, block, kernel_geometry=4)
    rig.assign(list(range(B)), _binding("round_robin", B, K))
    rig.call(list(range(B)), [block, 0, 3, 200, block, block, 1, 129], seed=9)
    rig.check_records()
    rig.check_oracle([0, 3])
    rig.close()
    bank = nb.get_dsp_bank(docs, batch=4, jit=2)
    bank.Reset(48000.0, 128)
    assert bank.jit_state == 0 and "precompiled" in bank.jit_note()
    bank.close()


def _run(h, x, block):
    h.Reset(48000.0, block)
    return np.concatenate([h.process_batch(np.ascontiguousarray(x[..., p:p + block])) for p in range(0, x.shape[-1], block)],
                          axis=-1)


@pytest.mark.parametrize("shape", ["a2_max", "cond", "mc"])
def test_shape_compiled_kernel_matches_each_models_compiled_handle_and_the_oracle(shape):
    """jit = 1 creates the bank on the kernel compiled for its shape; each stream is within 1e-6 of an ordinary handle of
    its model on that model's specialised kernel, and within 1e-5 of the oracle"""
    B, K, block, n = 9, 3, 256, 768
    docs = family(shape, K, seed=6)
    bank = nb.get_dsp_bank(docs, batch=B, jit=1)
    assert bank.jit_state == 1 and "compiled for the bank's shape" in bank.jit_note(), bank.jit_note()
    models = [s % K for s in range(B)]
    bank.Reset(48000.0, block)
    bank.assign_streams(list(range(B)), models)
    ci = bank.in_channels
    x = fx.synthetic_batch(B, n, seed=21) if ci == 1 else _signal(B, ci, n, 21)
    y = np.concatenate([bank.process_batch(np.ascontiguousarray(x[..., p:p + block])) for p in range(0, n, block)], axis=-1)
    worst = {}
    for k in range(K):
        rows = [s for s in range(B) if models[s] == k]
        h = nb.get_dsp(docs[k], batch=len(rows), jit=1)
        assert h.jit_state == 1
        yk = _run(h, np.ascontiguousarray(x[rows]), block)
        h.close()
        worst[k] = float(np.max(np.abs(y[rows] - yk)))
        assert worst[k] <= 1e-6, worst
        ref = _oracle_stream(docs[k], [x[rows[0], ..., p:p + block] for p in range(0, n, block)], block)
        assert float(np.max(np.abs(y[rows[0]] - ref))) <= TOL
    print("shape-compiled bank vs compiled handles, max |diff| per model:", worst)
    bank.close()


def test_shape_compiled_stream_does_not_depend_on_its_neighbours():
    B, K, block = 6, 3, 256
    docs = family("a2_max", K, seed=7)
    x = fx.synthetic_batch(B, 2 * block, seed=22)
    outs = []
    for models in ([0] * B, [0, 1, 2, 1, 2, 1], [0, 2, 2, 2, 2, 2]):
        bank = nb.get_dsp_bank(docs, batch=B, jit=1)
        assert bank.jit_state == 1
        bank.Reset(48000.0, block)
        bank.assign_streams(list(range(B)), models)
        outs.append(_run_no_reset(bank, x, block))
        bank.close()
    assert np.array_equal(outs[0][0], outs[1][0]) and np.array_equal(outs[0][0], outs[2][0])


def _run_no_reset(h, x, block):
    return np.concatenate([h.process_batch(np.ascontiguousarray(x[..., p:p + block])) for p in range(0, x.shape[-1], block)],
                          axis=-1)


def test_default_jit_bank_of_a_throughput_batch_runs_the_shape_compiled_kernel():
    B, K, block = 256, 4, 128
    docs = family("a2_max", K, seed=8)
    bank = nb.get_dsp_bank(docs, batch=B)
    assert bank.jit_state == 1, bank.jit_note()
    bank.Reset(48000.0, block)
    models = [s % K for s in range(B)]
    bank.assign_streams(list(range(B)), models)
    x = fx.synthetic_batch(B, 2 * block, seed=23)
    y = _run_no_reset(bank, x, block)
    for k in range(K):
        rows = [s for s in range(B) if models[s] == k]
        h = nb.get_dsp(docs[k], batch=len(rows), jit=1)  # (64 streams: the default jit would not compile the model)
        assert h.jit_state == 1
        assert float(np.max(np.abs(y[rows] - _run(h, np.ascontiguousarray(x[rows]), block)))) <= 1e-6
        h.close()
    bank.close()


def test_read_only_blob_path():
    docs = family("wide", 2, seed=5)
    assert 4 * len(docs[0]["weights"]) > 200 * 1024  # (the general kernel stages at most 200 KB in shared memory)
    assert nb.bank_check(docs)["ok"] is True
    # (it is a general-family model: a fused-family model beside it is refused for its kernel)
    assert "model 1: kernel: served by the fused kernel" in nb.bank_check([docs[0], fx.random_wavenet(seed=0)])["reason"]
    # its blob does not fit the shape-compiled kernel either: required jit fails with the reason, preferred falls back
    with pytest.raises(Exception, match="shared memory|too many weights"):
        nb.get_dsp_bank(docs, batch=4, jit=1)
    B, block = 4, 256
    rig = GRig(docs, B, block)
    rig.assign(list(range(B)), [1, 0, 1, 0])
    rig.call(list(range(B)), [block, 100, 0, block], seed=10)
    rig.call([3, 0], [block, block], seed=11)
    rig.check_records()
    rig.check_oracle([0, 1])
    rig.close()
