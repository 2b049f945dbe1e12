"""Slot-table calls on one GPU: wavenet_a1_standard, a handle of 4096 streams, device buffers, calls of 4096 and of 64
frames, four arms -- contiguous (nam_b200_process_f32_device), the identity table, a random permutation of all streams and
a random half of them (nam_b200_process_streams_f32_device).  Each arm is timed with CUDA events over --iters calls after
warm-up, the arms alternated --repeats times; the spread (min..max) of the repeats is reported.  The host time of a
table call's submission (table build, checks, upload, launch) is measured separately with a host clock around the call
alone.  Prints the card's name and power limit first, then one JSON line per (frames, arm).

    python tools/process_streams_bench.py [--iters 20] [--warmup 3] [--repeats 3]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
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
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--streams", type=int, default=4096)
    ap.add_argument("--frames", type=int, nargs="*", default=[4096, 64])
    args = ap.parse_args()

    import numpy as np
    import torch

    import neuralampmodelercore_b200 as nb
    from tests import nam_fixtures as fx

    if not torch.cuda.is_available():
        raise SystemExit("process_streams_bench: no CUDA device")
    print(json.dumps({"card": card(), "torch_device": torch.cuda.get_device_name(0)}), flush=True)
    nam = fx.load_model("wavenet_a1_standard")
    B = args.streams
    rng = np.random.default_rng(1)
    arms = {
        "contiguous": None,
        "identity_table": np.arange(B, dtype=np.int32),
        "permutation": rng.permutation(B).astype(np.int32),
        "random_half": rng.permutation(B)[:B // 2].astype(np.int32),
    }
    stream = torch.cuda.Stream()
    s = stream.cuda_stream
    for n in args.frames:
        d = nb.get_dsp(nam, batch=B, device=0, fast_tanh=True)
        d.Reset(48000.0, n)
        x = torch.from_numpy(fx.synthetic_batch(B, n, seed=2)).cuda()
        y = torch.empty_like(x)
        torch.cuda.synchronize()

        def call(streams):
            if streams is None:
                d.process_batch_device(x.data_ptr(), y.data_ptr(), B, n, cuda_stream=s)
            else:
                d.process_streams_device(streams, x.data_ptr(), y.data_ptr(), n, cuda_stream=s)

        def timed(streams):
            for _ in range(args.warmup):
                call(streams)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(args.iters):
                call(streams)
            e1.record(stream)
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / args.iters * 1e-3

        def host_us(streams):
            # host time of the submission alone: the stream is drained first, so the call does not wait on earlier work
            ts = []
            for _ in range(args.iters):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                call(streams)
                ts.append(time.perf_counter() - t0)
            torch.cuda.synchronize()
            return float(np.median(ts)) * 1e6

        rates = {k: [] for k in arms}
        for _ in range(args.repeats):
            for name, streams in arms.items():
                t = timed(streams)
                m = B if streams is None else len(streams)
                rates[name].append(m * n / t / 1e6)
        for name, streams in arms.items():
            r = rates[name]
            print(json.dumps({"frames": n, "arm": name, "streams": B if streams is None else len(streams),
                              "msamples_per_s": round(float(np.median(r)), 2), "spread": [round(min(r), 2), round(max(r), 2)],
                              "host_submit_us": round(host_us(streams), 1)}), flush=True)
        d.close()


if __name__ == "__main__":
    main()
