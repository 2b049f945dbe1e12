"""CPU-only tests of the per-stream state record (include/nam_b200.h, nam_b200_state_layout_json): its segments against
sizes derived independently from the oracle's config parser (oracle/nam_config.py), the pinned sizes of SURVEY.md
section 8, and the model fingerprint the record carries."""
import json

import numpy as np
import pytest

import neuralampmodelercore_b200 as nb
from oracle import nam_config
from tests import nam_fixtures as fx
from tests.test_reference_build import CONVNETS, _convnet

FIXTURES = ["wavenet", "wavenet_a1_standard", "lstm", "a2_full", "a2_lite", "wavenet_a2_max", "wavenet_condition_dsp",
            "slimmable_wavenet"]


def _wavenet_segments(fm: nam_config.FlatModel) -> list:
    """(channels, columns) of every convolution with a look-back, walking the flattened cfg like
    nam_config.expected_weight_count: layer convolutions, then each array's head convolution, then the post-stack head;
    a condition_dsp's segments after the main network's."""
    it = iter(fm.cfg.tolist())
    nxt = lambda: next(it)  # noqa: E731
    assert nxt() == nam_config.ARCH_WAVENET
    _in_ch, n_arrays, with_head = nxt(), nxt(), nxt()
    segs, last_head = [], 0
    for _ in range(n_arrays):
        (_inp, _cs, ch, bn, hs, hk, hd, _hb, _gi, _gm, _l1a, _l1g, h1a, h1o, _h1g) = [nxt() for _ in range(15)]
        for _f in range(8):
            nxt(), nxt(), nxt()
        for _l in range(nxt()):
            k, d, _g = nxt(), nxt(), nxt()
            for _a in range(2):  # activation and secondary activation: code, n_params
                nxt(), nxt()
            segs.append((ch, (k - 1) * d))
        segs.append((h1o if h1a else bn, (hk - 1) * hd))
        last_head = hs
    if with_head:
        hc, _ho, nk = nxt(), nxt(), nxt()
        cin = last_head
        for _i in range(nk):
            k = nxt()
            segs.append((cin, k - 1))
            cin = hc
    if fm.condition_dsp is not None:
        segs += _wavenet_segments(fm.condition_dsp)
    return [s for s in segs if s[1] > 0]


def expected_payload_floats(nam: dict) -> int:
    fm = nam_config.flatten(nam)
    c = fm.raw_config
    if fm.architecture == "WaveNet":
        return sum(ch * cols for ch, cols in _wavenet_segments(fm))
    if fm.architecture == "LSTM":
        return int(c["num_layers"]) * 2 * int(c["hidden_size"])
    if fm.architecture == "Linear":
        return int(c["receptive_field"]) - 1
    if fm.architecture == "ConvNet":
        cin, total = int(c.get("in_channels", 1)), 0
        for d in c["dilations"]:  # kernel-2 convolutions: look-back = dilation
            total += cin * int(d)
            cin = int(c["channels"])
        return total
    raise AssertionError(fm.architecture)


def _linear(rf=200, seed=3):
    rng = np.random.default_rng(seed)
    return {"version": "0.5.4", "architecture": "Linear", "config": {"receptive_field": rf, "bias": True},
            "weights": [float(v) for v in rng.uniform(-0.1, 0.1, rf + 1)], "sample_rate": 48000}


def _documents():
    docs = {name: fx.load_model(name) for name in FIXTURES if name != "slimmable_wavenet"}
    docs.update({f"convnet{i}": _convnet(**kw) for i, kw in enumerate(CONVNETS)})
    docs["linear"] = _linear()
    return docs


@pytest.mark.parametrize("name", list(_documents().keys()))
def test_layout_totals_match_config_derivation(name):
    nam = _documents()[name]
    lay = nb.state_layout(nam)
    segs = lay["segments"]
    assert lay["payload_floats"] == expected_payload_floats(nam)
    assert sum(s["channels"] * s["columns"] for s in segs) == lay["payload_floats"]
    assert lay["record_bytes"] == lay["header_bytes"] + 4 * lay["payload_floats"] and lay["header_bytes"] == 64
    off = 0
    for s in segs:  # contiguous, in order, none empty
        assert s["offset"] == off and s["columns"] > 0 and s["channels"] > 0
        off += s["channels"] * s["columns"]
    if nam["architecture"] == "WaveNet":
        fm = nam_config.flatten(nam)
        assert [(s["channels"], s["columns"]) for s in segs] == _wavenet_segments(fm)


def test_pinned_sizes():
    """SURVEY.md section 8: wavenet.nam 50 floats, a1_standard 49,104 (= 196,416 B), lstm.nam 6 (h[3], c[3])."""
    assert nb.state_layout(fx.load_model("wavenet"))["payload_floats"] == 50
    assert nb.state_layout(fx.load_model("wavenet_a1_standard"))["payload_floats"] == 49104
    lstm = nb.state_layout(fx.load_model("lstm"))
    assert lstm["payload_floats"] == 6 and [s["name"] for s in lstm["segments"]] == ["layer0.h", "layer0.c"]
    # A2-Full: SURVEY.md's 50,768 floats include the kernel-16 head convolution's 15 columns of 8 channels
    a2 = nb.state_layout(fx.load_model("a2_full"))
    layers = sum(s["channels"] * s["columns"] for s in a2["segments"] if ".layer" in s["name"])
    heads = [s for s in a2["segments"] if s["name"].endswith(".head")]
    assert [(s["channels"], s["columns"]) for s in heads] == [(8, 15)]
    assert a2["payload_floats"] == layers + 8 * 15 == 50768


def test_condition_dsp_segments_follow_the_main_network():
    lay = nb.state_layout(fx.load_model("wavenet_a2_max"))
    names = [s["name"] for s in lay["segments"]]
    cond = [i for i, n in enumerate(names) if n.startswith("condition_dsp.")]
    assert cond and cond == list(range(cond[0], len(names)))


def test_fingerprint_identity(tmp_path):
    nam = fx.load_model("wavenet")
    fp = nb.state_layout(nam)["fingerprint"]
    assert isinstance(fp, int) and 0 <= fp < 2 ** 64
    p = tmp_path / "m.nam"
    p.write_text(json.dumps(nam, indent=2))
    assert nb.state_layout(p)["fingerprint"] == fp  # file vs dict
    reordered = {"config": {k: nam["config"][k] for k in reversed(list(nam["config"]))}, **{k: v for k, v in nam.items() if k != "config"}}
    assert nb.state_layout(reordered)["fingerprint"] == fp  # key order is not part of the model
    meta = {**nam, "metadata": {"loudness": -20.0}, "sample_rate": 44100}
    assert nb.state_layout(meta)["fingerprint"] == fp  # neither are metadata and the sample rate
    one = json.loads(json.dumps(nam))
    one["weights"][7] = float(np.nextafter(np.float32(one["weights"][7]), np.float32(np.inf)))
    assert nb.state_layout(one)["fingerprint"] != fp  # a single weight, one ulp
    cfg = json.loads(json.dumps(nam))
    cfg["config"]["head_scale"] = cfg["config"]["head_scale"] + 1.0
    assert nb.state_layout(cfg)["fingerprint"] != fp
    assert nb.state_layout(fx.load_model("wavenet_a1_standard"))["fingerprint"] != fp


def test_container_describes_its_default_submodel():
    subs = nb.submodels(fx.load_model("slimmable_wavenet"))
    assert len(subs) >= 2
    whole = nb.state_layout(fx.load_model("slimmable_wavenet"))
    assert whole == nb.state_layout(subs[-1][1])
    assert nb.state_layout(subs[0][1])["fingerprint"] != whole["fingerprint"]
