"""Model banks on one GPU: K a1_standard-shaped models (the fixture's weights, seeded-perturbed per model) behind one handle
of 4096 streams, device buffers, CUDA events.  Workloads: K in {1, 8, 64, 512}, calls of 64 and of 4096 frames, streams
bound to models grouped (streams of a model contiguous) or round-robin (stream s runs model s % K: every short-geometry
slot mixes models, the worst case for blob reloads).  Arms:

  bank      one nam_b200_process_f32_device call over all 4096 streams of the bank;
  handles   K ordinary jit = 2 handles, each running its own 4096 / K streams (K launches; K <= --handles-max-k only,
            the others print "not measured");
  jit2      one ordinary handle of model 0 with jit = 2: the precompiled-kernel ceiling;
  jit       one ordinary handle of model 0 with the default jit: the model-specialised kernel a bank gives up.

--arch lstm runs the same workloads on LSTM banks instead (rows carry "shape"): "lstm" = lstm.nam reweighted per model
(the lane-group kernel, G = 4: 32 streams per CTA) and "h70" = a random one-layer cell of hidden size 70 (one thread per
stream, 64 streams per CTA, one pass per distinct model of a CTA).  The thread-per-stream kernel takes ~1 s per
4096-frame call of 4096 such streams, so h70 runs only calls of up to --h70-max-frames frames; the others print "not
measured".  LSTM handles are made with prewarm off (Reset's 24000-sample prewarm is not what is timed).

--arch general runs wavenet_a2_max.nam reweighted per model (the general kernel; "shape": "a2_max"), --arch convnet a
ConvNet of 8 channels, dilations 1..128 and BatchNorm ("shape": "convnet").  A general bank runs the precompiled general
kernel with jit = 2 ("bank") and the general kernel compiled for the bank's shape with the default jit ("bank_jit", checked
within 1e-5 of the jit = 2 bank); its "handles" arm uses the default jit (each handle compiles its own model-specialised
kernel, so keep --handles-max-k small), and "jit" is the ordinary handle's model-specialised general kernel.

Before timing, every K checks the bank's first call against fresh ordinary handles of its models at the timed sizes (up to
--check-models models; the bank's row reports bytes_equal and max_abs_diff, and the run stops above 1e-5).  Each arm is timed over --iters calls after --warmup, the arms alternated --repeats
times; the rate is Msamples/s (streams x frames / s) with the spread (min..max) of the repeats.  Prints the card's name and
power limit first, then one JSON line per (K, frames, binding, arm).

    python tools/bank_bench.py [--arch wavenet|lstm|general|convnet] [--ks 1 8 64 512] [--frames 64 4096] [--iters 10] [--warmup 2]
                               [--repeats 3]
"""
from __future__ import annotations

import argparse
import copy
import json
import os
import subprocess
import sys
import tempfile
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


def family(k: int, shape: str = "a1") -> list:
    import numpy as np

    from tests import nam_fixtures as fx

    if shape == "h70":
        return [{"version": "0.5.4", "architecture": "LSTM", "sample_rate": 48000.0,
                 "config": {"input_size": 1, "hidden_size": 70, "num_layers": 1},
                 "weights": [float(v) for v in np.random.default_rng(i).uniform(-0.3, 0.3, 4 * 70 * 71 + 4 * 70 + 2 * 70 + 71)]}
                for i in range(k)]
    if shape == "convnet":
        from tests.test_reference_build import _convnet

        return [_convnet(8, [1, 2, 4, 8, 16, 32, 64, 128], True, "Tanh", i) for i in range(k)]
    base = fx.load_model({"a1": "wavenet_a1_standard", "lstm": "lstm", "a2_max": "wavenet_a2_max"}[shape])
    w0 = np.asarray(base["weights"], np.float32)
    docs = []
    for i in range(k):
        d = copy.deepcopy(base)
        rng = np.random.default_rng(i)
        d["weights"] = [float(v) for v in w0 * (1.0 + 0.05 * rng.standard_normal(w0.shape)).astype(np.float32)]
        docs.append(d)
    return docs


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", type=int, nargs="*", default=[1, 8, 64, 512])
    ap.add_argument("--frames", type=int, nargs="*", default=[64, 4096])
    ap.add_argument("--streams", type=int, default=4096)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--handles-max-k", type=int, default=64)
    ap.add_argument("--check-models", type=int, default=8)
    ap.add_argument("--arch", choices=["wavenet", "lstm", "general", "convnet"], default="wavenet")
    ap.add_argument("--h70-max-frames", type=int, default=64)
    args = ap.parse_args()
    os.environ.setdefault("NAM_B200_JIT_CACHE", tempfile.mkdtemp(prefix="nam_b200_jit_"))  # (the tree may be read-only)

    import numpy as np
    import torch

    import neuralampmodelercore_b200 as nb

    if not torch.cuda.is_available():
        raise SystemExit("bank_bench: no CUDA device")
    print(json.dumps({"card": card(), "torch_device": torch.cuda.get_device_name(0)}), flush=True)
    B = args.streams
    F = max(args.frames)
    stream = torch.cuda.Stream()
    cs = stream.cuda_stream
    x = torch.randn(B, F, device="cuda") * 0.1
    y = torch.empty(B, F, device="cuda")

    def timed(run, n):
        """ms per call of run() over n calls (CUDA events on the bench's stream)"""
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(stream):
            e0.record()
            for _ in range(n):
                run()
            e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1) / n

    def device_call(d, rows, n_frames):
        """a contiguous device call of handle d over rows [r0, r1) of the buffers"""
        r0, r1 = rows
        return lambda: d.process_batch_device(x[r0].data_ptr(), y[r0].data_ptr(), r1 - r0, n_frames, F, F, cuda_stream=cs)

    shapes = {"wavenet": ["a1"], "lstm": ["lstm", "h70"], "general": ["a2_max"], "convnet": ["convnet"]}[args.arch]
    for shape in shapes:
        run_shape(args, shape, B, F, x, y, stream, timed, device_call)


def run_shape(args, shape, B, F, x, y, stream, timed, device_call) -> None:
    import numpy as np

    import neuralampmodelercore_b200 as nb

    tag = {} if shape == "a1" else {"shape": shape}  # (the WaveNet rows keep their fields)
    opts = {"prewarm": False} if shape in ("lstm", "h70") else {}
    handle_jit = 0 if shape in ("a2_max", "convnet") else 2  # (the "handles" arm)
    singles = {}
    for jit in (2, 0):
        d = nb.get_dsp(family(1, shape)[0], batch=B, jit=jit, **opts)
        d.Reset(48000.0, F)
        singles[jit] = d

    for K in args.ks:
        docs = family(K, shape)
        bank = nb.get_dsp_bank(docs, batch=B, jit=2, **opts)
        bank.Reset(48000.0, F)
        # a general bank with the default jit: the general kernel compiled for the bank's shape
        bank_jit = nb.get_dsp_bank(docs, batch=B, **opts) if shape == "a2_max" else None
        per = B // K
        handles = []
        if K <= args.handles_max_k and K > 1:
            for d in docs:
                h = nb.get_dsp(d, batch=per, jit=handle_jit, **opts)
                h.Reset(48000.0, F)
                handles.append(h)
        for binding in ("grouped", "round_robin"):
            models = np.arange(B) // per if binding == "grouped" else np.arange(B) % K
            models = np.minimum(models, K - 1).astype(np.int32)
            for n_frames in args.frames:
                if shape == "h70" and n_frames > args.h70_max_frames:
                    for a in ("bank", "handles", "jit2", "jit"):
                        print(json.dumps({**tag, "K": K, "frames": n_frames, "binding": binding, "arm": a,
                                          "msamples_per_s": None, "note": "not measured"}), flush=True)
                    continue
                bank.Reset(48000.0, F)
                bank.assign_streams(np.arange(B), models)
                if shape in ("lstm", "h70"):  # (an LSTM keeps h, c across Reset: every stream restarts from its model's h0 / c0)
                    bank.reset_streams(np.arange(B), fresh=True)
                # correctness at the timed size: the bank's first call against fresh ordinary handles of its models
                bank_run = device_call(bank, (0, B), n_frames)
                bank_run()
                stream.synchronize()
                got = y[:, :n_frames].cpu().numpy()
                xs = x[:, :n_frames].cpu().numpy()
                check = {"max_abs_diff": 0.0, "bytes_equal": True}
                for k in range(min(K, args.check_models)):
                    rows = np.nonzero(models == k)[0]
                    h = nb.get_dsp(docs[k], batch=len(rows), jit=2, **opts)
                    h.Reset(48000.0, F)
                    want = h.process_batch(np.ascontiguousarray(xs[rows]))
                    h.close()
                    check["bytes_equal"] &= bool(np.array_equal(got[rows], want))
                    check["max_abs_diff"] = max(check["max_abs_diff"], float(np.max(np.abs(got[rows] - want))))
                if check["max_abs_diff"] > 1e-5:
                    raise SystemExit(f"bank_bench: K={K} {binding} {n_frames} frames: outputs differ from the ordinary handles {check}")
                arms = {}
                if bank_jit is not None:
                    bank_jit.Reset(48000.0, F)
                    bank_jit.assign_streams(np.arange(B), models)
                    arms["bank_jit"] = device_call(bank_jit, (0, B), n_frames)
                    arms["bank_jit"]()
                    stream.synchronize()
                    check["bank_jit_state"] = bank_jit.jit_state
                    check["bank_jit_max_abs_diff"] = float(np.max(np.abs(y[:, :n_frames].cpu().numpy() - got)))
                    if check["bank_jit_max_abs_diff"] > 1e-5:
                        raise SystemExit(f"bank_bench: K={K} {binding} {n_frames} frames: the default-jit bank differs {check}")
                arms.update({"bank": bank_run,
                        "jit2": device_call(singles[2], (0, B), n_frames),
                        "jit": device_call(singles[0], (0, B), n_frames)})
                if handles and binding == "grouped":
                    calls = [device_call(h, (k * per, (k + 1) * per), n_frames) for k, h in enumerate(handles)]
                    arms["handles"] = lambda: [c() for c in calls]
                rates = {a: [] for a in arms}
                for a, run in arms.items():
                    timed(run, args.warmup)
                for _ in range(args.repeats):
                    for a, run in arms.items():
                        ms = timed(run, args.iters)
                        rates[a].append(B * n_frames / (ms * 1e-3) / 1e6)
                for a in ("bank", "bank_jit", "handles", "jit2", "jit"):
                    if a == "bank_jit" and bank_jit is None:
                        continue
                    row = {**tag, "K": K, "frames": n_frames, "binding": binding, "arm": a}
                    if a in rates:
                        r = sorted(rates[a])
                        row.update(msamples_per_s=round(r[len(r) // 2], 1), spread=[round(r[0], 1), round(r[-1], 1)])
                    else:
                        row.update(msamples_per_s=None, note="not measured" if a == "handles" else "")
                    if a == "bank":
                        row.update(checked_models=min(K, args.check_models), **check)
                    print(json.dumps(row), flush=True)
        for h in handles:
            h.close()
        bank.close()
        if bank_jit is not None:
            bank_jit.close()
    for d in singles.values():
        d.close()


if __name__ == "__main__":
    main()
