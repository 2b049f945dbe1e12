"""In-tree build of libnam_b200.so with nvcc for sm_90a (H100) (no JIT cache, no torch extension machinery).

The shared library is written to neuralampmodelercore_b200/lib/ so it travels with the repo snapshot
to the GPU box; it is git-ignored (*.so) so history stays source-only.
"""
from __future__ import annotations

import os
import shutil
import subprocess
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
LIB_DIR = PKG / "lib"
LIB_PATH = LIB_DIR / "libnam_b200.so"
INCLUDE = PKG.parent / "include"

SOURCES = ["nam_b200.cu", "nam_model_spec.cpp", "json_lite.cpp", "wavenet_pack.cpp", "generic_pack.cpp", "nam_dsp_shim.cpp",
           "jit_spec.cpp"]


def _obj_name(src: Path) -> str:
    return src.name + ".o"

GENCODE = "arch=compute_90a,code=sm_90a"

NVCC_FLAGS = [
    "-gencode",
    GENCODE,
    "-O3",
    "-lineinfo",
    "-std=c++17",
    "-Xcompiler",
    "-fPIC",
    "-shared",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and Path(cand).exists():
            return cand
    raise RuntimeError("nvcc not found: libnam_b200.so cannot be built")


def sources() -> list[Path]:
    return [CSRC / s for s in SOURCES if (CSRC / s).exists()]


def _stale() -> bool:
    if not LIB_PATH.exists():
        return True
    t = LIB_PATH.stat().st_mtime
    deps = list(CSRC.glob("*")) + list(INCLUDE.rglob("*.h"))
    return any(p.stat().st_mtime > t for p in deps if p.is_file())


def embed_spec_source() -> None:
    """wavenet_spec.cuh / lstm_spec.cuh -> csrc/*_src.inc, C++ raw string literals: the library carries the sources of the
    model-specialised kernels and hands them to NVRTC at model-load time (jit_spec.cpp)."""
    for stem in ("wavenet_spec", "lstm_spec", "wavenet_lat", "wavenet_generic_spec"):
        _embed(stem)
    _embed("generic_desc", ".h")


def _embed(stem: str, ext: str = ".cuh") -> Path:
    src = (CSRC / f"{stem}{ext}").read_text()
    delim = "NAMB200SPEC"
    assert f"){delim}\"" not in src
    # a string literal may not exceed 64 KiB on some compilers: split into adjacent literals
    parts, chunk = [], 12000
    for i in range(0, len(src), chunk):
        parts.append(f'R"{delim}({src[i:i + chunk]}){delim}"')
    inc = CSRC / f"{stem}_src.inc"
    text = f"// generated from {stem}{ext} by _build.py -- do not edit\n" + "\n".join(parts) + "\n"
    if not inc.exists() or inc.read_text() != text:
        inc.write_text(text)
    return inc


def _compile_object(src: Path, obj: Path, verbose: bool) -> str:
    cmd = [_nvcc(), *[f for f in NVCC_FLAGS if f != "-shared"], f"-I{INCLUDE}", "-c", "-o", str(obj), str(src)]
    if verbose:
        cmd[1:1] = ["-Xptxas", "-v"]
    proc = subprocess.run(cmd, capture_output=True, text=True)
    if proc.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + proc.stdout + proc.stderr)
    return proc.stderr


def build(force: bool = False, verbose: bool = False) -> Path:
    """Compile every CUDA/C++ source of the product into lib/libnam_b200.so (cross-compiles without a GPU).
    One object per source under lib/obj/ (recompiled when the source or any header is newer), compiled in parallel,
    then linked: touching the JIT host code does not recompile the kernels."""
    from concurrent.futures import ThreadPoolExecutor

    embed_spec_source()
    if not force and not _stale():
        return LIB_PATH
    LIB_DIR.mkdir(exist_ok=True)
    obj_dir = LIB_DIR / "obj"
    obj_dir.mkdir(exist_ok=True)
    import re

    def closure(path: Path, seen: set) -> set:
        """Files reachable through #include "..." (searched next to the includer, in csrc/ and in include/)."""
        for name in re.findall(r'#include\s+"([^"]+)"', path.read_text()):
            for base in (path.parent, CSRC, INCLUDE):
                cand = (base / name).resolve()
                if cand.is_file() and cand not in seen:
                    seen.add(cand)
                    closure(cand, seen)
                    break
        return seen

    jobs = []
    for src in sources():
        obj = obj_dir / _obj_name(src)
        deps = [src, *closure(src, set())]
        if force or not obj.exists() or any(d.stat().st_mtime > obj.stat().st_mtime for d in deps):
            jobs.append((src, obj))
    with ThreadPoolExecutor(max_workers=max(1, min(len(jobs), os.cpu_count() or 1))) as ex:
        logs = list(ex.map(lambda j: _compile_object(j[0], j[1], verbose), jobs))
    tmp = LIB_DIR / "libnam_b200.so.tmp"
    cmd = [_nvcc(), "-shared", "-Xcompiler", "-fPIC", "-gencode", GENCODE, "-o", str(tmp),
           *[str(obj_dir / _obj_name(s)) for s in sources()], "-ldl"]
    proc = subprocess.run(cmd, capture_output=True, text=True)
    if proc.returncode != 0:
        raise RuntimeError("link failed:\n" + " ".join(cmd) + "\n" + proc.stdout + proc.stderr)
    os.replace(tmp, LIB_PATH)
    if verbose:
        print("\n".join(logs))
    return LIB_PATH
