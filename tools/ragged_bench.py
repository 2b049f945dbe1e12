"""Ragged calls on one GPU: wavenet_a1_standard, a handle of 4096 streams, device buffers, CUDA events.  Two length mixes --
"jitter", each stream's count drawn from {32, 48, 64, 96, 128}, and "long", uniform in [1024, 4096] -- and three arms:

  ragged      one nam_b200_process_streams_ragged_f32_device call over all streams;
  per_length  one nam_b200_process_streams_f32_device call per distinct length (inputs pre-gathered per length);
  pad_to_max  one process_streams call of n_max frames on a separate handle: the cost of ignoring the raggedness (its
              result is not the ragged one).

Every arm's rate counts valid samples only (sum of the counts) per second.  Each arm is timed with CUDA events over --iters
calls after warm-up, the arms alternated --repeats times; the spread (min..max) of the repeats is reported.  Prints the
card's name and power limit first, then one JSON line per (mix, arm).

    python tools/ragged_bench.py [--iters 10] [--warmup 2] [--repeats 3]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))


def card() -> str:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.TimeoutExpired):
        return "unknown (nvidia-smi unavailable)"


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--streams", type=int, default=4096)
    ap.add_argument("--mixes", nargs="*", default=["jitter", "long"])
    args = ap.parse_args()

    import numpy as np
    import torch

    import neuralampmodelercore_b200 as nb
    from tests import nam_fixtures as fx

    if not torch.cuda.is_available():
        raise SystemExit("ragged_bench: no CUDA device")
    print(json.dumps({"card": card(), "torch_device": torch.cuda.get_device_name(0)}), flush=True)
    nam = fx.load_model("wavenet_a1_standard")
    B = args.streams
    rng = np.random.default_rng(1)
    mixes = {"jitter": rng.choice([32, 48, 64, 96, 128], size=B), "long": rng.integers(1024, 4097, size=B)}
    stream = torch.cuda.Stream()
    s = stream.cuda_stream
    all_streams = np.arange(B, dtype=np.int32)
    for mix in args.mixes:
        counts = mixes[mix].astype(np.int32)
        n_max = int(counts.max())
        valid = int(counts.sum())
        a = nb.get_dsp(nam, batch=B, device=0, fast_tanh=True)
        a.Reset(48000.0, n_max)
        p = nb.get_dsp(nam, batch=B, device=0, fast_tanh=True)
        p.Reset(48000.0, n_max)
        x = torch.from_numpy(fx.synthetic_batch(B, n_max, seed=2)).cuda()
        y = torch.empty_like(x)
        groups = []  # (streams, input [k_rows, k], output) per distinct length
        for k in sorted(set(counts.tolist())):
            rows = np.nonzero(counts == k)[0].astype(np.int32)
            xi = x[torch.from_numpy(rows).long().cuda(), :k].contiguous()
            groups.append((rows, k, xi, torch.empty_like(xi)))
        torch.cuda.synchronize()

        def ragged():
            a.process_streams_device(all_streams, x.data_ptr(), y.data_ptr(), counts, cuda_stream=s)

        def per_length():
            for rows, k, xi, yi in groups:
                a.process_streams_device(rows, xi.data_ptr(), yi.data_ptr(), k, cuda_stream=s)

        def pad_to_max():
            p.process_streams_device(all_streams, x.data_ptr(), y.data_ptr(), n_max, cuda_stream=s)

        arms = {"ragged": ragged, "per_length": per_length, "pad_to_max": pad_to_max}

        def timed(fn):
            for _ in range(args.warmup):
                fn()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(args.iters):
                fn()
            e1.record(stream)
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / args.iters * 1e-3

        rates = {k: [] for k in arms}
        for _ in range(args.repeats):
            for name, fn in arms.items():
                rates[name].append(valid / timed(fn) / 1e6)
        for name in arms:
            r = rates[name]
            print(json.dumps({"mix": mix, "arm": name, "streams": B, "n_max": n_max, "valid_samples": valid,
                              "distinct_lengths": len(groups), "msamples_per_s": round(float(np.median(r)), 2),
                              "spread": [round(min(r), 2), round(max(r), 2)]}), flush=True)
        a.close()
        p.close()


if __name__ == "__main__":
    main()
