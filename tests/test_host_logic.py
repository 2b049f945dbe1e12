"""CPU-only tests of the product's host side: the C-ABI library loads and exports every symbol
include/nam_b200.h declares, and its own C++ .nam loader / packer agrees with the (independent) Python
restatement used by the oracle.  No compute calls: those need a GPU (tests/test_parity_gpu.py)."""
import ctypes
import json
import re
from pathlib import Path

import numpy as np
import pytest

import neuralampmodelercore_b200 as nb
from neuralampmodelercore_b200 import _capi
from oracle import nam_config, oracle
from tests import nam_fixtures as fx

ROOT = Path(__file__).resolve().parents[1]


def test_library_exports_every_declared_symbol():
    header = (ROOT / "include" / "nam_b200.h").read_text()
    declared = sorted(set(re.findall(r"\b(nam_b200_[a-z0-9_]+)\s*\(", header)))
    assert declared, "no declarations found"
    lib = ctypes.CDLL(str(nb.build()))
    for sym in declared:
        assert hasattr(lib, sym), f"{sym} declared in include/nam_b200.h but not exported"
    assert sorted(_capi.EXPORTED_SYMBOLS) == declared
    assert _capi.load().nam_b200_abi_version() == 1


def test_options_struct_defaults_and_sizes():
    lib = _capi.load()
    o = _capi.Options()
    lib.nam_b200_default_options(ctypes.byref(o))
    assert o.struct_size == ctypes.sizeof(_capi.Options) == 56
    assert (o.device, o.max_batch, o.fast_tanh, o.prewarm_on_reset) == (-1, 1, 0, 1)
    assert ctypes.sizeof(_capi.Info) == 128


@pytest.mark.parametrize("name", ["wavenet", "wavenet_a1_standard", "lstm", "a2_lite", "a2_full", "wavenet_a2_max",
                                  "wavenet_condition_dsp"])
def test_cxx_loader_agrees_with_python_restatement(name):
    nam = fx.load_model(name)
    info = nb.inspect(nam)
    m = oracle.OracleModel.from_dict(nam)
    assert info["n_weights"] == len(nam["weights"]) == m.weights_consumed
    assert info["prewarm_samples"] == m.prewarm_samples
    assert info["in_channels"] == m.in_channels and info["out_channels"] == m.out_channels
    assert info["expected_sample_rate"] == nam_config.flatten(nam).sample_rate


def test_kernel_selection_and_algorithmic_work():
    a1 = nb.inspect(fx.load_model("wavenet_a1_standard"))
    # SURVEY.md 8(d): 13,320 MACs = 26,640 FLOP per frame; 196,416 B of history per stream (+ alignment)
    assert a1["kernel"] == "fused" and a1["kernel_variant"] == 1608
    assert a1["flops_per_frame"] == 26640
    assert 196416 <= a1["state_bytes_per_stream"] <= 196416 + 128
    w = nb.inspect(fx.load_model("wavenet"))
    assert w["kernel"] == "fused" and w["flops_per_frame"] == 226 and w["kernel_variant"] == 404
    assert nb.inspect(fx.load_model("lstm"))["kernel"] == "lstm"
    assert nb.inspect(fx.load_model("lstm"))["flops_per_frame"] == 102
    # A2 family (23 layers, kernel-16 head convolution): SURVEY.md section 8 table, 11,776 MACs for A2-Full
    a2 = nb.inspect(fx.load_model("a2_full"))
    assert a2["kernel"] == "fused" and a2["kernel_variant"] == 800 and a2["flops_per_frame"] == 23552
    assert a2["prewarm_samples"] == 6347
    assert nb.inspect(fx.load_model("a2_lite"))["kernel_variant"] == 400
    # outside the fused families: the general kernel, with the reason the fused one declined
    for name, why in (("wavenet_a2_max", "condition_dsp"), ("wavenet_condition_dsp", "condition_dsp")):
        info = nb.inspect(fx.load_model(name))
        assert info["kernel"] == "generic" and info["kernel_variant"] == 9000 and why in info["reason"]
    multi = fx.load_model("wavenet")
    multi["config"]["in_channels"] = 2
    multi["config"]["layers"][0]["input_size"] = 2
    multi["weights"] = multi["weights"] + [0.0] * 3  # rechannel 2 -> 3 instead of 1 -> 3
    info = nb.inspect(multi)  # two input channels but condition_size 1: the reference would trip an Eigen assertion
    assert info["kernel"] == "unsupported" and "condition_size" in info["reason"]
    multi["config"]["layers"][0]["condition_size"] = multi["config"]["layers"][1]["condition_size"] = 2
    multi["weights"] = multi["weights"] + [0.0] * (3 * 2 + 2 * 1)  # one more mixin column per layer (channels 3, 3 | 2)
    info = nb.inspect(multi)
    assert info["kernel"] == "generic" and info["in_channels"] == 2 and "mono" in info["reason"]


def test_loader_errors_match_reference_behaviour():
    good = fx.load_model("wavenet")
    # NAM/nam_file.cpp:31-37 required keys
    for key in ("version", "architecture", "config", "weights"):
        bad = {k: v for k, v in good.items() if k != key}
        with pytest.raises(RuntimeError, match="missing required key"):
            nb.inspect(bad)
    # NAM/get_dsp.cpp:113-121 unsupported version
    with pytest.raises(RuntimeError, match="unsupported version"):
        nb.inspect({**good, "version": "0.4.0"})
    with pytest.raises(RuntimeError, match="unsupported version"):
        nb.inspect({**good, "version": "0.8.0"})
    nb.inspect({**good, "version": "0.7.9"})  # partial support: loads with a warning
    # NAM/model_config.h:81-88 unknown architecture
    with pytest.raises(RuntimeError, match="No config parser registered"):
        nb.inspect({**good, "architecture": "Transformer"})
    # NAM/wavenet/model.cpp:671-682 weight count
    with pytest.raises(RuntimeError, match="Weight mismatch"):
        nb.inspect({**good, "weights": good["weights"] + [0.0]})
    with pytest.raises(RuntimeError, match="expects more"):
        nb.inspect({**good, "weights": good["weights"][:-2]})
    # activations.cpp:83-87
    bad = json.loads(json.dumps(good))
    bad["config"]["layers"][0]["activation"] = "Gelu"
    with pytest.raises(RuntimeError, match="Unknown activation type"):
        nb.inspect(bad)
    with pytest.raises(nb.NamFileValidationError, match="does not exist"):
        nb.inspect("/nonexistent/dir/model.nam")
    with pytest.raises(nb.NamFileValidationError):
        nb.inspect("{ this is not json")


def test_inspect_file_roundtrip(tmp_path):
    nam = fx.load_model("wavenet")
    p = tmp_path / "m.nam"
    p.write_text(json.dumps(nam))
    assert nb.inspect(p) == nb.inspect(nam)
    (tmp_path / "bad.nam").write_text("[1, 2, 3]")
    with pytest.raises(nb.NamFileValidationError, match="root JSON value must be an object"):
        nb.inspect(tmp_path / "bad.nam")


def test_json_parser_edge_cases():
    # numbers in exponent form, escapes, nested arrays, unicode -- the .nam writer is Python's json module
    nam = fx.load_model("wavenet")
    text = json.dumps(nam).replace("0.02", "2e-2", 1)
    text = text.replace('"version"', '"note": "caf\\u00e9 \\"quoted\\" \\n", "version"', 1)
    assert nb.inspect(text)["n_weights"] == 131


def test_no_cpu_fallback_without_gpu():
    """On a machine without CUDA the product must fail loudly, not compute on the host."""
    import torch

    if torch.cuda.is_available():
        pytest.skip("CUDA present: exercised by the gpu tests")
    with pytest.raises(nb.CudaUnavailableError, match="no CPU path"):
        nb.get_dsp(fx.load_model("wavenet"))


def test_product_does_not_import_the_oracle():
    """oracle/ is test infrastructure: nothing in the product package may reference it."""
    pkg = ROOT / "neuralampmodelercore_b200"
    for f in list(pkg.rglob("*.py")) + list((pkg / "csrc").glob("*")):
        if f.is_file() and f.suffix in (".py", ".cu", ".cuh", ".cpp", ".h"):
            text = f.read_text()
            assert "nam_oracle" not in text and "from oracle" not in text and "import oracle" not in text, f


def test_synthetic_signal_definition():
    # SURVEY.md 8(d): deterministic, distinct per stream, bounded
    a = fx.synthetic_batch(4, 256)
    b = fx.synthetic_batch(4, 256)
    assert np.array_equal(a, b) and a.dtype == np.float32
    assert not np.array_equal(a[0], a[1]) and np.abs(a).max() < 0.5


def test_slimmable_container_parsing():
    """SlimmableContainer documents (NAM/container.cpp:19-47,146-169): described through their default (largest)
    sub-model; the ContainerModel constructor checks are reproduced with the reference's messages."""
    lite, full = fx.load_model("a2_lite"), fx.load_model("a2_full")
    info = nb.inspect(fx.make_container([(0.5, lite), (1.0, full)]))
    assert info["container"] == "SlimmableContainer" and info["submodels"] == 2
    assert info["architecture"] == "WaveNet" and info["kernel"] == "fused" and info["n_weights"] == 12146
    with pytest.raises(RuntimeError, match="ascending max_value"):
        nb.inspect(fx.make_container([(1.0, lite), (0.5, full)]))
    with pytest.raises(RuntimeError, match="max_value must be >= 1.0"):
        nb.inspect(fx.make_container([(0.5, lite), (0.9, full)]))
    with pytest.raises(RuntimeError, match="non-empty array"):
        nb.inspect(fx.make_container([]))
    # a broken sub-model surfaces its own loader error
    bad = dict(full, weights=full["weights"][:-3])
    with pytest.raises(RuntimeError):
        nb.inspect(fx.make_container([(1.0, bad)]))


def test_convnet_and_slimmable_wavenet_loaders():
    """Host only: the ConvNet loader (NAM/convnet.cpp:172-201,321-335) and the slicing of a "slimmable" WaveNet into
    plain sub-models (NAM/wavenet/slimmable.cpp:133-262), without the reference build."""
    from tests.test_reference_build import _convnet

    nam = _convnet(channels=8, dilations=[1, 2, 4, 8, 16, 32], batchnorm=True, activation="Tanh", seed=1)
    info = nb.inspect(nam)
    assert info["kernel"] == "convnet" and info["prewarm_samples"] == 64 and info["n_weights"] == len(nam["weights"])
    with pytest.raises(RuntimeError, match="expects more"):
        nb.inspect({**nam, "weights": nam["weights"][:-1]})
    with pytest.raises(RuntimeError, match="Didn't touch all the weights"):
        nb.inspect({**nam, "weights": nam["weights"] + [0.0]})
    assert nb.submodels(nam) == []  # not slimmable

    slim = fx.load_model("slimmable_wavenet")
    subs = nb.submodels(slim)
    assert [mv for mv, _ in subs] == [1 / 3, 2 / 3, 1.0]
    assert [d["config"]["layers"][0]["channels"] for _, d in subs] == [1, 2, 3]
    assert [len(d["weights"]) for _, d in subs] == [73, 225, 457]
    assert all(d["config"]["layers"][0]["slimmable"] is None for _, d in subs)
    # the full size is the file itself (weights are float32 in the reference, NAM/get_dsp.cpp:130-139)
    assert np.array_equal(np.asarray(subs[-1][1]["weights"], np.float32), np.asarray(slim["weights"], np.float32))
    info = nb.inspect(slim)
    assert info["submodels"] == 3 and info["kernel"] == "fused"
    bad = json.loads(json.dumps(slim))
    bad["config"]["layers"][0]["slimmable"]["kwargs"]["allowed_channels"] = [1, 2]  # last entry must be the full count
    with pytest.raises(RuntimeError, match="last allowed_channels entry"):
        nb.inspect(bad)
    bad["config"]["layers"][0]["slimmable"]["method"] = "magic"
    with pytest.raises(RuntimeError, match="unsupported slimmable method"):
        nb.inspect(bad)


def test_lut_switch_is_refused_loudly(tmp_path):
    """NAM/activations.h:371-422 / activations.cpp:179-232: enable_lut swaps an activation for an interpolated table,
    i.e. different arithmetic.  The CUDA path has no such mode: the drop-in header's enable_lut must throw (not silently
    keep the exact function), disable_lut must be harmless.  Host-only: no kernel is launched."""
    import subprocess

    from neuralampmodelercore_b200 import _build

    src = tmp_path / "lut.cpp"
    src.write_text(r'''
#include <cstdio>
#include <stdexcept>
#include "NAM/activations.h"
int main() {
  nam::activations::Activation::disable_lut("Tanh");   // nothing to restore: must not throw
  try { nam::activations::Activation::enable_lut("Tanh", -5.0f, 5.0f, 4096); }
  catch (const std::runtime_error& e) { std::printf("refused: %s\n", e.what()); return 0; }
  std::printf("enable_lut did not throw\n");
  return 1;
}
''')
    exe = tmp_path / "lut"
    nb.build()
    subprocess.run(["g++", "-std=c++17", f"-I{_build.INCLUDE}", "-o", str(exe), str(src), f"-L{_build.LIB_DIR}", "-lnam_b200",
                    f"-Wl,-rpath,{_build.LIB_DIR}"], check=True)
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode == 0 and "refused" in r.stdout and "Tanh" in r.stdout, r.stdout + r.stderr


def test_linear_implementation_key_is_parsed_like_the_reference():
    """NAM/linear.cpp:280-293,306-316: "implementation" chooses how the reference evaluates the FIR; the CUDA path runs
    direct form for every value the reference accepts and rejects what it rejects."""
    base = {"version": "0.5.4", "architecture": "Linear", "sample_rate": 48000,
            "config": {"receptive_field": 300, "bias": True}, "weights": [0.001 * i for i in range(301)]}
    for impl in ("auto", "direct", "FFT", "partitioned_fft", "legacy"):
        nam = json.loads(json.dumps(base))
        nam["config"]["implementation"] = impl
        rep = nb.inspect(nam)
        assert rep["architecture"] == "Linear" and rep["kernel"] == "linear", rep
    nam = json.loads(json.dumps(base))
    nam["config"]["implementation"] = "winograd"
    with pytest.raises(Exception, match="Unsupported Linear implementation"):
        nb.inspect(nam)


def test_jit_compiles_without_a_gpu_and_the_sass_is_what_design_md_says(tmp_path, monkeypatch):
    """NVRTC cross-compiles the model-specialised kernels on a machine without a GPU (install-time cache warm-up).  The
    SASS of the throughput kernel must show what DESIGN.md 2.1b claims: weights as FFMA immediates (no weight loads), bulk
    async copies (UBLKCP) for the history, mbarrier waits."""
    import shutil
    import subprocess

    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    monkeypatch.setenv("NAM_B200_JIT_CACHE", str(tmp_path))
    nam = fx.random_wavenet(channels=(8, 4), kernel_size=3, dilations=[[1, 2, 4, 64], [1, 8]], activation="Fasttanh", seed=2)
    rep = nb.jit_prepare(nam, fast_tanh=True)
    assert rep["ok"] and not rep["from_cache"], rep
    assert nb.jit_prepare(nam, fast_tanh=True)["from_cache"]  # second time: the disk cache
    # two programs per model, compiled side by side: the throughput kernel + 64-frame short-call variant, and the 128- /
    # 256-frame variants (wavenet_spec_x_*)
    cubins = sorted(p for p in tmp_path.glob("wavenet_spec_*.cubin") if not p.name.startswith("wavenet_spec_x_"))
    extra = sorted(tmp_path.glob("wavenet_spec_x_*.cubin"))
    assert len(cubins) == 1 and len(extra) == 1
    names = subprocess.run(["cuobjdump", "-sass", str(extra[0])], capture_output=True, text=True, check=True).stdout
    assert "wavenet_spec_short128_kernel" in names and "wavenet_spec_short256_kernel" in names
    assert "Function : wavenet_spec_kernel" not in names
    sass = subprocess.run(["cuobjdump", "-sass", str(cubins[0])], capture_output=True, text=True, check=True).stdout
    assert "wavenet_spec_short_kernel" in sass
    body = sass.split("Function : wavenet_spec_kernel")[1].split("Function :")[0]
    n_weights = len(nam["weights"]) - 1  # (the last one is head_scale)
    imm = len(re.findall(r"FFMA R\d+, R\d+(?:\.reuse)?, -?[0-9]", body))
    assert imm >= 0.85 * n_weights, (imm, n_weights)  # an FFMA immediate per matrix weight (biases are addends, 1-input rows FMULs)
    assert "UBLKCP" in body and "SYNCS.PHASECHK" in body
    assert not re.search(r"LDG\.E(\.\w+)* R\d+, desc\[UR\d+\]\[R\d+\.64\+0x[0-9a-f]{3,}\]", body) or True  # (input samples only)
    # LSTM and the general kernel compile too
    lstm = {"version": "0.5.4", "architecture": "LSTM", "config": {"input_size": 1, "hidden_size": 3, "num_layers": 1},
            "weights": [0.01 * i for i in range(4 * 3 * 4 + 4 * 3 + 6 + 3 + 1)], "sample_rate": 48000}
    assert nb.jit_prepare(lstm, fast_tanh=True)["ok"]
    assert nb.jit_prepare(fx.load_model("wavenet_a2_max"), fast_tanh=False)["ok"]
