"""Cost of the sample-rate conversion on a server-sized handle: 4096 streams of a1_standard on device buffers, host calls
of 64 and 4096 frames, a 44.1 kHz host converted to the capture's 48 kHz against a handle reset at 48 kHz (nothing to
convert).  The two arms alternate, so that drift of a shared machine lands on both.

  python tools/resample_bench.py [--streams 4096] [--reps 3] [--out DIR]

Prints one JSON object (--out DIR also writes it to DIR/resample_bench.json): per call size and arm the host Msamples/s of each repetition (median and spread), the device
time of the two conversion kernels and the history update (torch.profiler, a separate run), and the card's name and
power limit read in the same run."""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import neuralampmodelercore_b200 as nb  # noqa: E402
from tests import nam_fixtures as fx  # noqa: E402

RS_KERNELS = ("resample_kernel", "resample_history_kernel")


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return [s.strip() for s in q.split(",")]
    except Exception as e:  # (no nvidia-smi: the name from torch, the limit not measured)
        return [torch.cuda.get_device_name(0), f"not measured ({e})", "not measured"]


def timed(d, x, y, frames, calls, st):
    """host Msamples/s of `calls` device calls of `frames` frames on every stream (CUDA events)."""
    b = x.shape[0]
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.cuda.stream(st):
        for _ in range(3):
            d.process_batch_device(x.data_ptr(), y.data_ptr(), b, frames, cuda_stream=st.cuda_stream)
        e0.record(st)
        for _ in range(calls):
            d.process_batch_device(x.data_ptr(), y.data_ptr(), b, frames, cuda_stream=st.cuda_stream)
        e1.record(st)
    e1.synchronize()
    ms = e0.elapsed_time(e1)
    return b * frames * calls / (ms * 1e-3) / 1e6


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON to DIR/resample_bench.json")
    a = ap.parse_args()
    nam = fx.load_model("wavenet_a1_standard")
    nam["sample_rate"] = 48000.0  # (the fixture leaves its rate unknown; a capture trained at 48 kHz)
    st = torch.cuda.Stream()
    name, power, clock = card()
    result = {"card": name, "power_limit": power, "max_sm_clock": clock, "streams": a.streams, "model": "wavenet_a1_standard",
              "sizes": {}}
    for frames, calls in ((64, 600), (4096, 24)):
        arms = {}
        for host in (44100.0, 48000.0):
            d = nb.get_dsp(nam, batch=a.streams, resample=True)
            d.Reset(host, frames)
            arms[host] = d
        x = torch.from_numpy(fx.synthetic_batch(a.streams, frames, seed=1)).cuda()
        y = torch.empty_like(x)
        runs = {44100.0: [], 48000.0: []}
        for _ in range(a.reps):
            for host in (44100.0, 48000.0):
                runs[host].append(timed(arms[host], x, y, frames, calls, st))
        # kernel times of the conversion, from a profiled run of its own
        d = arms[44100.0]
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            timed(d, x, y, frames, calls, st)
        per = {}
        for ev in prof.key_averages():
            if any(k in ev.key for k in RS_KERNELS):
                per[ev.key.split("(")[0]] = round(ev.device_time_total / (calls + 3), 2)  # us per call
        conv = runs[44100.0]
        base = runs[48000.0]
        result["sizes"][str(frames)] = {
            "calls_timed": calls,
            "msamples_per_s_44k1_converted": {"median": round(statistics.median(conv), 1), "runs": [round(v, 1) for v in conv]},
            "msamples_per_s_48k_no_conversion": {"median": round(statistics.median(base), 1), "runs": [round(v, 1) for v in base]},
            "conversion_kernels_us_per_call": per or "not measured",
            "resample_ratio": list(d.resample_ratio),
        }
        for h in arms.values():
            h.close()
    if a.out:
        out = Path(a.out)
        out.mkdir(parents=True, exist_ok=True)
        (out / "resample_bench.json").write_text(json.dumps(result, indent=1))
    print(json.dumps(result))


if __name__ == "__main__":
    main()
