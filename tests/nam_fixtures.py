"""Test helpers: committed model fixtures (tests/golden/models/*.npz), the decoded example input and
the synthetic benchmark signal of SURVEY.md section 8(d).  Nothing here reads the reference's source tree."""
from __future__ import annotations

import json
import os
from pathlib import Path

import numpy as np

GOLDEN = Path(__file__).resolve().parent / "golden"


def _restore(obj, arrays):
    if isinstance(obj, dict):
        if set(obj.keys()) == {"__weights__"}:
            return [float(v) for v in arrays[f"w{obj['__weights__']}"]]
        return {k: _restore(v, arrays) for k, v in obj.items()}
    if isinstance(obj, list):
        return [_restore(v, arrays) for v in obj]
    return obj


def load_model(name: str) -> dict:
    """The .nam document (dict with version/architecture/config/weights...) of a committed fixture."""
    with np.load(GOLDEN / "models" / f"{name}.npz") as z:
        header = json.loads(bytes(z["header"]).decode())
        arrays = {k: z[k] for k in z.files if k != "header"}
    return _restore(header, arrays)


def input_wav() -> np.ndarray:
    """example_audio/input.wav decoded to float32: 1 s of silence then 1 s of a 220 Hz, 0.5-amplitude sine."""
    with np.load(GOLDEN / "input_wav.npz") as z:
        return z["x"].astype(np.float32)


def oracle_golden(name: str, regime: str) -> dict:
    with np.load(GOLDEN / "oracle_outputs.npz") as z:
        return {k.split(".")[-1]: z[k] for k in z.files if k.startswith(f"{name}.{regime}.")}


def decimate(y: np.ndarray) -> dict:
    return {"head": y[:512], "transition": y[46000:50096], "strided": y[::37]}


REFERENCE_OUTPUTS = GOLDEN / "reference_outputs.npz"


def sample(y: np.ndarray) -> np.ndarray:
    """The part of an output (time on the last axis) that tests/golden/reference_outputs.npz keeps: all of it up to
    1024 frames, else the first 128 frames and every 16th frame after them."""
    y = np.asarray(y, dtype=np.float32)
    n = y.shape[-1]
    return y if n <= 1024 else y[..., np.r_[0:128, 128:n:16]]


def reference(key: str, compute) -> np.ndarray:
    """What the reference (NeuralAmpModelerCore itself, oracle/_ref) computes for the test case `key`, sampled as by
    `sample()`, from tests/golden/reference_outputs.npz.  `compute` is the case's recipe against the reference build
    (oracle.ref): with NAM_REFERENCE_RECORD=1, where oracle/_ref is built, it runs and its result replaces the stored one."""
    if os.environ.get("NAM_REFERENCE_RECORD") == "1":
        y = sample(compute())
        store = {}
        if REFERENCE_OUTPUTS.exists():
            with np.load(REFERENCE_OUTPUTS) as z:
                store = {k: z[k] for k in z.files}
        store[key] = y
        np.savez_compressed(REFERENCE_OUTPUTS, **store)
        return y
    with np.load(REFERENCE_OUTPUTS) as z:
        return z[key]


def synthetic_batch(batch: int, n: int, seed: int = 1234, rate: float = 48000.0) -> np.ndarray:
    """Per stream b: g_b*(0.25 sin(2pi 220 t + phi_b) + 0.10 sin(2pi 1230 t)) + 0.01*noise  (SURVEY.md 8d;
    the two-tone is the reference's own bench signal, tools/bench_a2_fast.cpp:245-249)."""
    t = np.arange(n, dtype=np.float64) / rate
    b = np.arange(batch, dtype=np.float64)[:, None]
    g = 0.5 + b / (2.0 * batch)
    phi = 2.0 * np.pi * b / batch
    x = g * (0.25 * np.sin(2 * np.pi * 220.0 * t[None, :] + phi) + 0.10 * np.sin(2 * np.pi * 1230.0 * t[None, :]))
    rng = np.random.default_rng(seed)
    x = x + 0.01 * rng.standard_normal((batch, n))
    return np.ascontiguousarray(x, dtype=np.float32)


def make_wavenet_nam(layers: list[dict], weights, head_scale: float = 1.0, version: str = "0.5.4",
                     sample_rate: float | None = 48000.0, **config_extra) -> dict:
    nam = {
        "version": version,
        "architecture": "WaveNet",
        "config": {"layers": layers, "head": None, "head_scale": head_scale, **config_extra},
        "weights": [float(w) for w in weights],
    }
    if sample_rate is not None:
        nam["sample_rate"] = sample_rate
    return nam


def random_wavenet(channels=(16, 8), kernel_size=3, dilations=None, activation="Tanh", seed=0, scale=0.3,
                   head_bias_last=True, kernel_sizes=None, head_kernel=None, head_dilation=None) -> dict:
    """Random-weight plain WaveNet in the a1 family (tools/create_wavenet.py-style), weights U(-scale, scale)
    like tools/test/test_a2_fast.cpp:109-117."""
    from oracle import nam_config

    dilations = dilations or [[1, 2, 4, 8], [1, 2, 4, 8]]
    layers = []
    for a, c in enumerate(channels):
        last = a + 1 == len(channels)
        lc = {
            "input_size": 1 if a == 0 else channels[a - 1],
            "condition_size": 1,
            "head_size": 1 if last else channels[a + 1],
            "channels": c,
            "dilations": list(dilations[a]),
            "activation": activation,
            "gated": False,
            "head_bias": bool(last and head_bias_last),
        }
        if head_kernel is not None:  # A2-style nested head config (model.cpp:961-1036)
            lc["head"] = {"out_channels": lc.pop("head_size"), "kernel_size": int(head_kernel), "bias": lc.pop("head_bias")}
            if head_dilation is not None:
                lc["head"]["head_dilation"] = int(head_dilation)
        if kernel_sizes is not None:
            lc["kernel_sizes"] = list(kernel_sizes[a])
        else:
            lc["kernel_size"] = kernel_size
        layers.append(lc)
    nam = make_wavenet_nam(layers, [], head_scale=0.02)
    n = nam_config.expected_weight_count(nam)
    rng = np.random.default_rng(seed)
    w = rng.uniform(-scale, scale, size=n).astype(np.float32)
    w[-1] = 0.02  # head_scale is the last weight
    nam["weights"] = [float(v) for v in w]
    return nam


def make_container(submodels, version: str = "0.7.0", sample_rate: float | None = 48000.0) -> dict:
    """A "SlimmableContainer" document (NAM/container.cpp:146-169; example_models/A2.nam has this form):
    `submodels` = [(max_value, nam_dict), ...]."""
    nam = {
        "version": version,
        "architecture": "SlimmableContainer",
        "config": {"submodels": [{"max_value": float(v), "model": m} for v, m in submodels]},
        "weights": [],
    }
    if sample_rate is not None:
        nam["sample_rate"] = sample_rate
    return nam
