"""Instruction census of the specialised throughput kernel (wavenet_spec_kernel), per history unit, from its SASS.

    python tools/spec_proto/sass_census.py <cubin> [--json]

The cubin is one the library built (jit_prepare writes it to the JIT cache: `wavenet_spec_<hash>.cubin`) or a
tools/spec_proto build (`nvcc -cubin`).  A history unit (a layer, or an array's convolutional head) starts at its B0, the
CTA barrier that is followed by the wait for the unit's history, and runs to the next unit's B0; the last unit runs to
the end of the tile loop.  The code in front of the first B0 (the tile's start: first history request, input load,
rechannel) is reported as unit "pre".  Per unit:
  total      non-NOP instructions
  ffma       FFMA instructions
  model      FFMAs with a model weight as immediate (every model FFMA has one; those of the fast tanh have a register or
             a fast-tanh constant)
  w0         instructions on paths that only warp 0 runs: branches skipped by the other warps that hold a bulk copy
             (UBLKCP), a bulk-group wait (DEPBAR) or the history mbarrier's expect-tx arrival
  copies     bulk copy instructions (UBLKCP), one per contiguous piece; w0 / copies is the cost of a copy
  cctl       CCTL.IVALL (what a full bulk-group wait compiles to)
Static counts: the tile body is straight-line code with one frame per thread, so they are close to per-frame counts.
"""
import argparse
import json
import re
import struct
import subprocess
import sys

# the fast-tanh constants (wavenet_spec.cuh, fast_tanh2) as float32
FAST_TANH_CONSTANTS = [struct.unpack("f", struct.pack("f", v))[0]
                       for v in (2.45550750702956, 0.821226666969744, 0.893229853513558, 0.814642734961073,
                                 2.44506634652299)]

_LINE = re.compile(r"/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;")


def sass_instructions(cubin, function="wavenet_spec_kernel"):
    """[(address, text)] of `function`'s non-NOP instructions."""
    out = subprocess.run(["cuobjdump", "-sass", "-fun", function, cubin], capture_output=True, text=True, check=True).stdout
    ins = []
    for m in _LINE.finditer(out):
        text = m.group(2).strip()
        if text.split()[0] in ("NOP",):
            continue
        ins.append((int(m.group(1), 16), text))
    if not ins:
        raise RuntimeError(f"no SASS for {function} in {cubin}")
    return ins


def _opcode(text):
    t = text.split()
    return t[1] if t[0].startswith("@") else t[0]


def _is_model_ffma(text):
    if _opcode(text) != "FFMA":
        return False
    imms = re.findall(r"(?<![\w.])-?\d+\.\d+(?:e[-+]?\d+)?", text)
    return bool(imms) and not any(abs(abs(float(t)) - c) <= 1e-6 * c for t in imms for c in FAST_TANH_CONSTANTS)


def census(cubin, function="wavenet_spec_kernel"):
    ins = sass_instructions(cubin, function)
    addr_index = {a: i for i, (a, _) in enumerate(ins)}
    ops = [_opcode(t) for _, t in ins]

    # unit starts: a BAR.SYNC followed, within a few instructions, by a try-wait on an mbarrier (the history wait)
    starts = []
    for i, op in enumerate(ops):
        if op.startswith("BAR.SYNC") and any(o.startswith("SYNCS.PHASECHK") for o in ops[i + 1:i + 6]):
            starts.append(i)
    end = next(i for i in range(len(ops) - 1, -1, -1) if ops[i] == "EXIT")
    # the tile loop's back edge: the last backward branch before EXIT ends the last unit
    for i in range(end - 1, starts[-1], -1):
        m = re.search(r"BRA\s+(?:`\(.*\)\s*)?0x([0-9a-f]+)", ins[i][1])
        if m and int(m.group(1), 16) < ins[i][0] and int(m.group(1), 16) < ins[starts[0]][0]:
            end = i + 1
            break

    # warp-0 paths: the span a conditional forward branch skips, when it holds a bulk copy, a bulk-group wait or the
    # history expect-tx arrival
    w0 = set()
    for i, (a, text) in enumerate(ins):
        if not text.startswith("@") or _opcode(text) != "BRA" or ".U.ANY" in text:
            continue
        m = re.search(r"0x([0-9a-f]+)", text.split("BRA", 1)[1])
        if not m:
            continue
        tgt = int(m.group(1), 16)
        if tgt <= a or tgt not in addr_index:
            continue
        span = range(i + 1, addr_index[tgt])
        if any(ops[j].startswith("BAR.SYNC") for j in span):  # (the branch around a whole tile loop)
            continue
        if any(ops[j].startswith(("UBLKCP", "DEPBAR")) or ops[j] == "SYNCS.ARRIVE.TRANS64" for j in span):
            w0.update(span)

    def row(name, lo, hi):
        r = dict(unit=name, total=hi - lo, ffma=0, model=0, w0=0, copies=0, cctl=0)
        for j in range(lo, hi):
            op, text = ops[j], ins[j][1]
            r["ffma"] += op == "FFMA"
            r["model"] += _is_model_ffma(text)
            r["w0"] += j in w0
            r["copies"] += op.startswith("UBLKCP")
            r["cctl"] += op.startswith("CCTL")
        return r

    rows = [row("pre", 0, starts[0])]
    bounds = starts + [end]
    for u in range(len(starts)):
        rows.append(row(str(u), bounds[u], bounds[u + 1]))
    return rows


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("cubin")
    ap.add_argument("--function", default="wavenet_spec_kernel")
    ap.add_argument("--json", action="store_true")
    a = ap.parse_args(argv)
    rows = census(a.cubin, a.function)
    if a.json:
        json.dump(rows, sys.stdout, indent=1)
        print()
        return
    keys = ["total", "ffma", "model", "w0", "copies", "cctl"]
    print(f"{'unit':>5} " + " ".join(f"{k:>7}" for k in keys) + f" {'w0/copy':>8}")
    for r in rows:
        per = f"{r['w0'] / r['copies']:.1f}" if r["copies"] else "-"
        print(f"{r['unit']:>5} " + " ".join(f"{r[k]:>7}" for k in keys) + f" {per:>8}")
    tot = {k: sum(r[k] for r in rows) for k in keys}
    print(f"{'all':>5} " + " ".join(f"{tot[k]:>7}" for k in keys) + f" {tot['w0'] / max(tot['copies'], 1):>8.1f}")


if __name__ == "__main__":
    main()
