"""GPU tests of growing model banks (nam_b200_bank_add_models, nam_b200_bank_replace_model, options.bank_capacity).

The yardstick is a bank created with all its documents: a bank created with two documents and grown to five mid-session
must give, call for call, the same output bytes and export the same record bytes.  That bank in turn is held to one
ordinary jit = 2 handle per model and to the oracle by the Rig of test_bank_gpu (test_lstm_bank_gpu for LSTMs)."""
import os
from pathlib import Path

import numpy as np
import pytest

import neuralampmodelercore_b200 as nb
from neuralampmodelercore_b200 import _capi
from tests import nam_fixtures as fx
from tests import test_lstm_bank_gpu as lstm_bank
from tests.test_bank_gpu import Rig, _family
from tests.test_general_bank_gpu import family as general_family

pytestmark = pytest.mark.gpu

class OracleRig(Rig):
    """The shape-compiled general kernel orders its sums unlike the precompiled one, so a bank on it is held to the oracle
    alone (as in test_general_bank_gpu), not to jit = 2 handles byte for byte"""

    def __init__(self, docs, batch, block, **kw):
        super().__init__(docs, batch, block, **kw)
        for r in self.refs:
            r.close()
        self.refs = []

    def assign(self, streams, models):
        self.bank.assign_streams(streams, models)
        for s, k in zip(streams, models):
            self.model[s] = k
            self.ins[s], self.outs[s] = [], []


# name -> (documents of one shape, Rig class, options, streams)
FAMILIES = {
    "wavenet": (lambda k, seed: _family("wavenet", k, seed), Rig, {}, 48),
    "a1": (lambda k, seed: _family("a1", k, seed), Rig, {}, 48),
    "a2_max_jit2": (lambda k, seed: general_family("a2_max", k, seed), Rig, {"jit": 2}, 48),
    # (the default jit compiles the general kernel for the bank's shape from max_batch 256 on)
    "a2_max_shape_compiled": (lambda k, seed: general_family("a2_max", k, seed), OracleRig, {}, 256),
    "convnet": (lambda k, seed: general_family("convnet", k, seed), Rig, {}, 48),
    "lstm": (lambda k, seed: lstm_bank._family("lstm", k, seed), lstm_bank.Rig, {}, 64),
    "h70": (lambda k, seed: lstm_bank._family("h70", k, seed), lstm_bank.Rig, {}, 40),
}


def _x(n, counts, seed):
    """The input a Rig's ragged call of these counts feeds (mono models)"""
    n_max = max(counts)
    x = fx.synthetic_batch(n, max(n_max, 1), seed=seed)[:, :n_max].copy()
    for i, c in enumerate(counts):
        x[i, c:] = 0.0
    return x


def _call_both(grown, rig, streams, counts, seed):
    """The same ragged call on the grown bank and on the rig's created bank (which the rig holds to its yardsticks)"""
    y = rig.call(streams, counts, seed)
    assert np.array_equal(grown.process_streams(streams, _x(len(streams), counts, seed), n_frames=counts), y)


def _schedule(grown, rig, B, seed):
    rng = np.random.default_rng(seed)
    for c in range(2):
        n = int(rng.integers(B // 2, B + 1))
        streams = [int(v) for v in rng.permutation(B)[:n]]
        counts = [int(v) for v in rng.choice([0, 1, 17, 40, 63, 64], size=n)]
        counts[0] = 64
        _call_both(grown, rig, streams, counts, seed=seed + c)


def _assign_both(grown, rig, streams, models):
    rig.assign(streams, models)
    grown.assign_streams(streams, models)


def _jit_cache_files() -> int:
    d = Path(os.environ.get("NAM_B200_JIT_CACHE") or (_capi.lib_path().parent / "jit_cache"))
    return sum(1 for p in d.rglob("*") if p.is_file()) if d.exists() else 0


def _prewarm_blocks(h, block) -> int:
    return -(-h.GetPrewarmSamples() // block) if h.GetPrewarmSamples() > 0 else 0


@pytest.mark.parametrize("name", list(FAMILIES))
def test_grown_bank_equals_created_bank_and_adding_disturbs_nothing(name):
    make, rig_cls, kw, B = FAMILIES[name]
    block = 64
    docs = make(5, 1)
    rig = rig_cls(docs, B, block, **kw)
    grown = nb.get_dsp_bank(docs[:2], batch=B, capacity=6, **kw)
    grown.Reset(48000.0, block)
    assert (grown.bank_size, grown.bank_capacity) == (2, 6)
    if name == "a2_max_shape_compiled":
        assert grown.jit_state == 1 and rig.bank.jit_state == 1, grown.jit_note()
    _assign_both(grown, rig, list(range(B)), [s % 2 for s in range(B)])
    _schedule(grown, rig, B, seed=10)

    # adding: no stream's record moves by a bit, the only launches are the new rows' prewarm, nothing is compiled
    before, cached = grown.export_streams(range(B)), _jit_cache_files()
    launches = grown.launch_count()
    assert grown.add_models(docs[2:]) == [2, 3, 4]
    assert grown.launch_count() - launches == _prewarm_blocks(grown, block)
    assert grown.bank_size == 5
    assert np.array_equal(grown.export_streams(range(B)), before)
    assert _jit_cache_files() == cached

    moved = list(range(0, B, 3))
    _assign_both(grown, rig, moved, [2 + (i % 3) for i in range(len(moved))])
    _schedule(grown, rig, B, seed=20)
    assert np.array_equal(grown.export_streams(range(B)), rig.bank.export_streams(range(B)))
    for k in range(5):
        got, want = grown.model_info(k), rig.bank.model_info(k)
        assert (got.loudness, got.n_weights) == (want.loudness, want.n_weights)
    rig.check_records()
    rig.check_oracle([moved[0], moved[1], moved[2], 1])
    grown.close()
    rig.close()


# (name, family, max_frames, options, when): when the documents are added relative to the grown bank's Reset
TIMINGS = [
    ("before_reset", "a1", 64, {}, "before"),
    ("after_reset_64", "a1", 64, {}, "after"),
    ("after_reset_4096", "a1", 4096, {}, "after"),
    ("no_prewarm", "a1", 64, {"prewarm": False}, "after"),
    ("general_4096", "a2_max_jit2", 4096, {"jit": 2}, "after"),
    ("lstm_before_reset", "lstm", 64, {}, "before"),
    ("lstm_no_prewarm", "lstm", 64, {"prewarm": False}, "after"),
    ("lstm_after_fast_tanh_switch", "lstm", 64, {}, "switch"),
]


@pytest.mark.parametrize("name,fam,block,kw,when", TIMINGS, ids=[t[0] for t in TIMINGS])
def test_when_models_are_added(name, fam, block, kw, when):
    docs = FAMILIES[fam][0](5, 2)
    B = 8
    created = nb.get_dsp_bank(docs, batch=B, **kw)
    grown = nb.get_dsp_bank(docs[:2], batch=B, capacity=5, **kw)
    if when == "before":
        grown.add_models(docs[2:])
    for h in (created, grown):
        h.Reset(48000.0, block)
    if when == "switch":
        for h in (created, grown):
            h.set_fast_tanh(True)
            h.assign_streams([0], [1])  # (the model rows are rebuilt in the new regime before this copy)
    if when != "before":
        assert grown.add_models(docs[2:]) == [2, 3, 4]
    models = [s % 5 for s in range(B)]
    for h in (created, grown):
        h.assign_streams(list(range(B)), models)
    assert np.array_equal(grown.export_streams(range(B)), created.export_streams(range(B)))
    counts = [block, block // 2, 1, block, 0, block, 3, block]
    x = _x(B, counts, seed=5)
    assert np.array_equal(grown.process_streams(list(range(B)), x, n_frames=counts),
                          created.process_streams(list(range(B)), x, n_frames=counts))
    assert np.array_equal(grown.export_streams(range(B)), created.export_streams(range(B)))
    created.close()
    grown.close()


def test_replace_model():
    import torch

    docs = _family("a1", 3, seed=3)
    new = _family("a1", 4, seed=4)[3]
    B, block = 8, 256
    bank = nb.get_dsp_bank(docs, batch=B, capacity=4, jit=2)
    bank.Reset(48000.0, block)
    bank.assign_streams([0, 1, 2], [0, 1, 1])
    old_ref, new_ref = nb.get_dsp(docs[2], batch=B, jit=2), nb.get_dsp(new, batch=B, jit=2)
    for h in (old_ref, new_ref):
        h.Reset(48000.0, block)

    # refused while a stream is bound: the handle is unchanged
    bank.assign_streams([5, 3], [2, 2])
    records, info = bank.export_streams(range(B)), bank.model_info(2)
    with pytest.raises(RuntimeError, match=r"2 stream\(s\) are bound to model 2 \(the lowest: stream 3\)"):
        bank.replace_model(2, new)
    assert np.array_equal(bank.export_streams(range(B)), records)
    assert bank.model_info(2).loudness == info.loudness
    old_record = old_ref.export_streams([0])

    # an asynchronous call on a side CUDA stream runs stream 5 (model 2); stream 5 moves and model 2 is replaced while that
    # call may still be in flight: its outputs are the old model's
    x = fx.synthetic_batch(1, block, seed=6)
    xd = torch.from_numpy(x).cuda()
    yd = torch.zeros_like(xd)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(50_000_000)  # (keeps the call queued while the host moves on)
        bank.process_streams_device([5], xd.data_ptr(), yd.data_ptr(), block, cuda_stream=side.cuda_stream)
    bank.assign_streams([5, 3], [0, 0])
    bank.replace_model(2, new)
    side.synchronize()
    assert np.array_equal(yd.cpu().numpy(), old_ref.process_streams([5], x))

    # streams assigned to the recycled index run the new document
    bank.assign_streams([4, 6], [2, 2])
    assert bank.model_info(2).loudness == new_ref.info.loudness
    new_ref.reset_streams([4, 6])
    x = fx.synthetic_batch(2, block, seed=7)
    assert np.array_equal(bank.process_streams([4, 6], x), new_ref.process_streams([4, 6], x))
    assert np.array_equal(bank.export_streams([4, 6]), new_ref.export_streams([4, 6]))

    # records: the old document's is refused, the new one's binds its stream to model 2
    with pytest.raises(ValueError, match="none of the 3 models of this bank"):
        bank.import_streams([7], old_record)
    bank.import_streams([7], new_ref.export_streams([4]))
    assert list(bank.stream_models([7])) == [2]
    # model 0 may be replaced as well; get_info follows it
    bank.assign_streams(list(range(B)), [1] * B)
    bank.replace_model(0, new)
    assert bank.info.loudness == new_ref.info.loudness
    for h in (bank, old_ref, new_ref):
        h.close()


def _refused(bank, control, call, match, exc=ValueError):
    """`call` on `bank` raises and leaves it exactly as `control`, which got every other call `bank` got"""
    B = bank.batch
    with pytest.raises(exc, match=match):
        call()
    assert (bank.bank_size, bank.bank_capacity) == (control.bank_size, control.bank_capacity)
    assert np.array_equal(bank.stream_models(range(B)), control.stream_models(range(B)))
    assert np.array_equal(bank.export_streams(range(B)), control.export_streams(range(B)))
    x = _x(B, [64] * B, seed=9)
    assert np.array_equal(bank.process_streams(list(range(B)), x), control.process_streams(list(range(B)), x))


def test_refusals_leave_the_handle_unchanged():
    docs = _family("wavenet", 5, seed=5)
    B = 6
    bank, control = (nb.get_dsp_bank(docs[:2], batch=B, capacity=5) for _ in range(2))
    for h in (bank, control):
        h.Reset(48000.0, 64)
        h.assign_streams([1, 4], [1, 1])
        h.process_streams(list(range(B)), _x(B, [64] * B, seed=1))
    other_shape = _family("a1", 1)[0]
    _refused(bank, control, lambda: bank.add_models([docs[2], docs[3], other_shape]), r"model 4 differs from model 0",
             RuntimeError)
    _refused(bank, control, lambda: bank.add_models([docs[2], lstm_bank._family("lstm", 1)[0]]), r"model 3: architecture",
             nb.UnsupportedModelError)
    _refused(bank, control, lambda: bank.add_models(docs[1:5]), r"4 documents do not fit: the bank holds 2 of its "
                                                                  r"bank_capacity = 5")
    _refused(bank, control, lambda: bank.add_models([]), r"n = 0")
    ordinary = nb.get_dsp(docs[0], batch=B)
    with pytest.raises(ValueError, match=r"bank_capacity = 1"):
        ordinary.add_models([docs[1]])
    assert ordinary.bank_size == 1 and ordinary.bank_capacity == 1
    with pytest.raises(nb.UnsupportedModelError, match="not a model bank"):
        ordinary.replace_model(0, docs[1])
    for cap in (1, -1):
        with pytest.raises(ValueError, match=rf"bank_capacity = {cap}"):
            nb.get_dsp_bank(docs[:2], batch=B, capacity=cap)
    for h in (bank, control, ordinary):
        h.close()


def test_one_document_with_room_is_a_bank():
    docs = _family("a1", 5, seed=6)
    B, block = 40, 64
    one = nb.get_dsp_bank(docs[:1], batch=B, capacity=4, jit=3)
    one.Reset(48000.0, block)
    assert (one.bank_size, one.bank_capacity, one.jit_state) == (1, 4, 0)
    assert "model bank" in one.jit_note(), one.jit_note()
    rig = Rig(docs[:4], B, block)
    _assign_both(one, rig, list(range(B)), [0] * B)
    _schedule(one, rig, B, seed=30)
    assert one.add_models(docs[1:4]) == [1, 2, 3]
    _assign_both(one, rig, list(range(0, B, 2)), [1 + (s // 2) % 3 for s in range(0, B, 2)])
    _schedule(one, rig, B, seed=40)
    assert np.array_equal(one.export_streams(range(B)), rig.bank.export_streams(range(B)))
    rig.check_records()
    one.close()
    rig.close()
    # with capacity 0 or 1 a bank of one document is get_dsp
    x = fx.synthetic_batch(4, block, seed=8)
    plain = nb.get_dsp(docs[0], batch=4)
    plain.Reset(48000.0, block)
    want = plain.process_batch(x)
    for cap in (0, 1):
        h = nb.get_dsp_bank(docs[:1], batch=4, capacity=cap)
        h.Reset(48000.0, block)
        assert (h.bank_size, h.bank_capacity) == (1, 1)
        assert np.array_equal(h.process_batch(x), want)
        h.close()
    plain.close()
