"""Growing model banks on one GPU: a1_standard-shaped models (tools/bank_bench.py's family: the fixture's weights,
seeded-perturbed per model) behind one bank of 4096 streams.  Rows:

  add_models     wall time of DSP.add_models for 1 and for 64 documents into a reset bank of 8 models and capacity 512, at
                 max_frames 64 and 4096 (parsing, packing, uploads and the new rows' prewarm: everything the call does);
  replace_model  wall time of DSP.replace_model of an unbound model of that bank;
  rebuild        what growing replaces: create and reset a bank of K + 1 = 9 documents, then move all 4096 sessions over with
                 export_streams + import_streams (host records) or their _device variants (records in device memory);
  rate           Msamples/s of one process_f32_device call over all 4096 streams (CUDA events, --iters calls) at 64 and
                 4096 frames, streams bound to the 8 models in contiguous blocks, for a bank created with 8 documents at
                 capacity 8 and at capacity 512, and for a bank created with 2 documents at capacity 8 and grown to 8;
                 plus one row of the grown bank with round-robin binding (stream s runs model s % 8) at 64 frames.

Every arm runs --repeats times, the arms alternated; each row gives the median and the spread (min, max).  Prints the card's
name and power limit first, then one JSON line per row.

    python tools/bank_grow_bench.py [--streams 4096] [--repeats 3] [--iters 20]
"""
from __future__ import annotations

import argparse
import json
import statistics
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))


def summary(xs: list) -> dict:
    return {"median": round(statistics.median(xs), 3), "spread": [round(min(xs), 3), round(max(xs), 3)], "n": len(xs)}


def wall_ms(f) -> float:
    t0 = time.perf_counter()
    f()
    return (time.perf_counter() - t0) * 1e3


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=4096)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()

    import numpy as np
    import torch

    import neuralampmodelercore_b200 as nb
    from bank_bench import card, family

    if not torch.cuda.is_available():
        print("no CUDA device: nothing measured", file=sys.stderr)
        return 1
    print(f"card: {card()}", flush=True)
    B, K, CAP = args.streams, 8, 512
    # the bank's 8, one to add, 64 to add, one to replace with; as JSON texts, so that the timed calls do not include
    # Python's serialisation of the documents
    docs = [json.dumps(d) for d in family(K + 1 + 64 + 1)]
    grouped = [s * K // B for s in range(B)]
    results: dict = {}

    def record(key, value):
        results.setdefault(key, []).append(value)

    def reset_bank(frames, k=K, capacity=CAP):
        h = nb.get_dsp_bank(docs[:k], batch=B, capacity=capacity)
        h.Reset(48000.0, frames)
        h.assign_streams(list(range(B)), [s * k // B for s in range(B)])
        return h

    # call-rate banks, kept across repeats
    rate_banks = {"created_cap8": reset_bank(64, K, K), "created_cap512": reset_bank(64, K, CAP)}
    grown = reset_bank(64, 2, K)
    grown.add_models(docs[2:K])
    grown.assign_streams(list(range(B)), grouped)
    rate_banks["grown_cap8"] = grown
    x = {f: torch.from_numpy(np.ascontiguousarray(np.tile(
        np.sin(np.arange(f, dtype=np.float32) * 0.03)[None, :], (B, 1)))).cuda() for f in (64, 4096)}
    y = {f: torch.empty_like(x[f]) for f in x}

    rs = torch.cuda.Stream()  # (the events and the calls on one stream of their own)

    def rate(h, frames) -> float:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(rs):
            for _ in range(2):
                h.process_batch_device(x[frames].data_ptr(), y[frames].data_ptr(), B, frames, cuda_stream=rs.cuda_stream)
            e0.record()
            for _ in range(args.iters):
                h.process_batch_device(x[frames].data_ptr(), y[frames].data_ptr(), B, frames, cuda_stream=rs.cuda_stream)
            e1.record()
        rs.synchronize()
        return B * frames * args.iters / (e0.elapsed_time(e1) * 1e-3) / 1e6

    for r in range(args.repeats):
        for frames in (64, 4096):
            # growing a reset bank, and recycling an index
            h = reset_bank(frames)
            record(("add_models", 1, frames), wall_ms(lambda: h.add_models(docs[K:K + 1])))
            record(("add_models", 64, frames), wall_ms(lambda: h.add_models(docs[K + 1:K + 65])))
            record(("replace_model", 1, frames), wall_ms(lambda: h.replace_model(K, docs[K + 65])))
            h.close()
            # the alternative: a new bank of K + 1 documents, every session moved over
            old = reset_bank(frames)
            t0 = time.perf_counter()
            new = nb.get_dsp_bank(docs[:K + 1], batch=B)
            new.Reset(48000.0, frames)
            create_ms = (time.perf_counter() - t0) * 1e3
            streams = list(range(B))
            recs = None

            def host_move():
                nonlocal recs
                recs = old.export_streams(streams)
                new.import_streams(streams, recs)

            host_ms = wall_ms(host_move)
            rb = old.state_record_bytes
            buf = torch.empty(B * rb, dtype=torch.uint8, device="cuda")

            side = torch.cuda.Stream()

            def device_move():  # (both on one CUDA stream: the import reads what the export wrote)
                old.export_streams_device(streams, buf.data_ptr(), cuda_stream=side.cuda_stream)
                new.import_streams_device(streams, buf.data_ptr(), cuda_stream=side.cuda_stream)
                side.synchronize()

            device_ms = wall_ms(device_move)
            assert np.array_equal(new.export_streams([0, B - 1]), recs[[0, B - 1]])
            record(("rebuild_create_reset", K + 1, frames), create_ms)
            record(("rebuild_host_move", K + 1, frames), create_ms + host_ms)
            record(("rebuild_device_move", K + 1, frames), create_ms + device_ms)
            del buf, recs
            old.close()
            new.close()
            # call rates, the arms alternated
            for name in (["created_cap8", "created_cap512", "grown_cap8"] if r % 2 == 0
                         else ["grown_cap8", "created_cap512", "created_cap8"]):
                h = rate_banks[name]
                if h.GetMaxBufferSize() != frames:
                    h.Reset(48000.0, frames)
                    h.assign_streams(list(range(B)), grouped)
                record(("rate", name, frames), rate(h, frames))
            if frames == 64:
                g = rate_banks["grown_cap8"]
                g.assign_streams(list(range(B)), [s % K for s in range(B)])
                record(("rate", "grown_cap8_round_robin", 64), rate(g, 64))
                g.assign_streams(list(range(B)), grouped)
        print(f"repeat {r + 1}/{args.repeats} done", file=sys.stderr, flush=True)

    for (row, what, frames), xs in results.items():
        line = {"row": row, "max_frames" if row != "rate" else "frames": frames, "streams": B}
        if row == "rate":
            line.update(arm=what, msamples_per_s=summary(xs))
        else:
            line.update(models=what, capacity=CAP if row in ("add_models", "replace_model") else K + 1, wall_ms=summary(xs))
        print(json.dumps(line), flush=True)
    for h in rate_banks.values():
        h.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
