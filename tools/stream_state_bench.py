"""Per-stream state control on one GPU: device export, device import and reset_streams of wavenet_a1_standard streams
(196 KB of history each) at 1, 64 and 4096 streams, timed with CUDA events over many iterations after warm-up.  Bytes
moved come from the record layout (nam_b200_state_layout_json); bandwidth is reported against the 3.35 TB/s HBM3
figure of NVIDIA's H100 SXM data sheet.  Prints the card's name and power limit first, then one JSON line per case.

    python tools/stream_state_bench.py [--iters 50] [--warmup 5]
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

HBM3_BYTES_PER_S = 3.35e12


def card() -> str:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.TimeoutExpired):
        return "unknown (nvidia-smi unavailable)"


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--streams", type=int, nargs="*", default=[1, 64, 4096])
    args = ap.parse_args()

    import numpy as np
    import torch

    import neuralampmodelercore_b200 as nb
    from tests import nam_fixtures as fx

    if not torch.cuda.is_available():
        raise SystemExit("stream_state_bench: no CUDA device")
    print(json.dumps({"card": card(), "torch_device": torch.cuda.get_device_name(0)}), flush=True)
    nam = fx.load_model("wavenet_a1_standard")
    lay = nb.state_layout(nam)
    payload = 4 * lay["payload_floats"]
    rb = lay["record_bytes"]
    max_n = max(args.streams)
    d = nb.get_dsp(nam, batch=max_n, device=0, fast_tanh=True)
    d.Reset(48000.0, 64)
    d.process_batch(fx.synthetic_batch(max_n, 64, seed=1))
    buf = torch.empty(max_n * rb, dtype=torch.uint8, device="cuda")
    # a stream of its own: the device variants run on it and the events below bracket them (0 would mean the handle's
    # stream, which the events would not wait for)
    stream = torch.cuda.Stream()
    s = stream.cuda_stream

    def timed(fn, host_clock=False):
        for _ in range(args.warmup):
            fn()
        torch.cuda.synchronize()
        if host_clock:  # synchronous calls (they end in a synchronise of the handle's stream)
            t0 = time.perf_counter()
            for _ in range(args.iters):
                fn()
            return (time.perf_counter() - t0) / args.iters
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(args.iters):
            fn()
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.iters * 1e-3  # s per operation

    for n in args.streams:
        streams = np.arange(n, dtype=np.int32)
        d.export_streams_device(streams, buf.data_ptr(), rb, s)
        torch.cuda.synchronize()
        cases = {
            # state read, records written (CUDA events on `stream`)
            "export_device": (lambda: d.export_streams_device(streams, buf.data_ptr(), rb, s), n * (payload + rb), False),
            # records read, state written; the n headers go to the host and are checked first (CUDA events on `stream`,
            # which therefore include that round trip)
            "import_device": (lambda: d.import_streams_device(streams, buf.data_ptr(), rb, s), n * (rb + payload), False),
            # the kept record read once per stream, state written; synchronous (host clock)
            "reset_streams": (lambda: d.reset_streams(streams), n * (payload + payload), True),
        }
        for name, (fn, nbytes, host_clock) in cases.items():
            t = timed(fn, host_clock)
            print(json.dumps({"op": name, "streams": n, "record_bytes": rb, "bytes_moved": nbytes, "us_per_op": round(t * 1e6, 2),
                              "GB_per_s": round(nbytes / t / 1e9, 1), "share_of_hbm3_3.35TB_s": round(nbytes / t / HBM3_BYTES_PER_S, 3)}),
                  flush=True)
    d.close()


if __name__ == "__main__":
    main()
