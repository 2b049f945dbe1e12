"""The instruction census (tools/spec_proto/sass_census.py) of a1_standard's specialised throughput kernel, compiled by
jit_prepare (NVRTC, no GPU needed): every layer keeps exactly its model FFMAs, and a bulk copy costs warp 0 at most a
bounded number of instructions."""
import shutil
import sys
from pathlib import Path

import pytest

import neuralampmodelercore_b200 as nb
from tests import nam_fixtures as fx

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "tools" / "spec_proto"))
import sass_census  # noqa: E402

pytestmark = pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="cuobjdump is not on PATH")

# warp-0 instructions per bulk copy piece, over the whole kernel: 34 in this build (a few uniform address instructions,
# the loop over the lanes that issue a copy, and the bulk-group wait); a bound that catches a copy path that grows
MAX_W0_PER_COPY = 40


@pytest.fixture(scope="module")
def census(tmp_path_factory, monkeypatch_module):
    cache = tmp_path_factory.mktemp("jit_cache")
    monkeypatch_module.setenv("NAM_B200_JIT_CACHE", str(cache))
    rep = nb.jit_prepare(fx.load_model("wavenet_a1_standard"), fast_tanh=True, batch=4096)
    assert rep["ok"], rep["why_not"]
    cubins = [p for p in cache.glob("wavenet_spec_*.cubin") if not p.name.startswith("wavenet_spec_x_")]
    assert len(cubins) == 1, cubins
    return sass_census.census(str(cubins[0]))


@pytest.fixture(scope="module")
def monkeypatch_module():
    mp = pytest.MonkeyPatch()
    yield mp
    mp.undo()


def _layers(nam):
    """[(channels, kernel size, first of its array, last of its array)] in kernel order"""
    out = []
    for la in nam["config"]["layers"]:
        n = len(la["dilations"])
        out += [(la["channels"], la["kernel_size"], i == 0, i + 1 == n) for i in range(n)]
    return out


def test_each_layer_keeps_its_model_ffmas(census):
    layers = _layers(fx.load_model("wavenet_a1_standard"))
    units = [r for r in census if r["unit"] != "pre"]
    assert len(units) == len(layers)
    for u, (r, (C, K, first, last)) in enumerate(zip(units, layers)):
        if first or last:  # (the compiler may move an array's head and the next array's rechannel across a barrier)
            continue
        assert r["model"] == K * C * C + C + C * C, (u, r)


def test_copy_cost_on_warp_0(census):
    w0 = sum(r["w0"] for r in census)
    copies = sum(r["copies"] for r in census)
    assert copies > 0
    assert w0 / copies <= MAX_W0_PER_COPY, (w0, copies)
