#!/usr/bin/env python
"""Recording K transmissions from one stream: K b2s_recorder pushes one after another against one b2s_recorder_bank push.

Input: config 4's record leg (bench.py --config 4): 40 MS/s CS8 from synth (four keyed FM carriers, 32768-point frames, 2048 frames
= 67.1 M samples, resident on the device), recorded at 32 kS/s. K = 4 uses config 4's shifts; K = 16 adds twelve more across the band.
Per K, after warm-up, (a) and (b) alternate for --reps repetitions, each timed with CUDA events around work that ends in the library's
synchronise; the medians are reported. Every repetition asserts that (a) and (b) produced the same bytes per channel. Prints one JSON
line with the card's name and power limit read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--ks", type=int, nargs="+", default=[4, 16])
    args = ap.parse_args()

    import numpy as np
    import torch

    import __graft_entry__ as ge
    import bench

    b2s, synth = ge.load_b2s(), ge.load_synth()
    if not torch.cuda.is_available():
        raise SystemExit("recorder_bank_bench.py needs a CUDA device: the recorders have no CPU fallback")
    wl = bench.WORKLOADS[4]
    n, fs, frames, bw = wl["n"], wl["fs"], wl["frames"], 32_000
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    stream = torch.cuda.current_stream(dev)
    eng = b2s.Engine(0)
    iq = synth.make_iq_int8_torch(n, frames, bench.wideband_tones(synth, n, fs, frames, bench.LEARN), seed=synth.seed_for(4, 0), quiet_frames=bench.LEARN, device=dev)
    n_samples = frames * n
    torch.cuda.synchronize()
    config4 = [b2s.get_tuned_frequency(int(mhz * 1e6), 2500) for mhz in (-12.5, -3.2, 4.7, 15.1)]

    def shifts_for(k):
        extra = [b2s.get_tuned_frequency(int(mhz * 1e6), 2500) for mhz in np.linspace(-18.0, 18.0, max(k - 4, 0) + 2)[1:-1]]
        return (config4 + extra)[:k]

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        out = fn()
        e1.record(stream)
        e1.synchronize()
        return e0.elapsed_time(e1), out

    results = []
    for k in args.ks:
        shifts = shifts_for(k)
        pool = [b2s.Recorder(eng, fs, bw, on_device=True, max_samples_per_push=n_samples) for _ in shifts]
        bank = b2s.RecorderBank(eng, fs, bw, k, on_device=True, max_samples_per_push=n_samples)
        for c, s in enumerate(shifts):
            pool[c].start(s)
            bank.start(c, s)
        ptr = iq.data_ptr()

        def run_pool():
            return [r.push(ptr, n_samples) for r in pool]

        def run_bank():
            return bank.push(ptr, 0, n_samples=n_samples)

        t_pool, t_bank = [], []
        for rep in range(args.warmup + args.reps):
            ms_a, out_a = timed(run_pool)
            ms_b, out_b = timed(run_bank)
            assert len(out_a) == len(out_b) == k
            for c in range(k):
                assert len(out_a[c]) > 0 and np.array_equal(out_a[c], out_b[c]), (k, rep, c)
            if rep >= args.warmup:
                t_pool.append(ms_a)
                t_bank.append(ms_b)
        med_a, med_b = statistics.median(t_pool), statistics.median(t_bank)
        results.append({"K": k, "shifts_hz": shifts, "pool_ms": med_a, "bank_ms": med_b, "pool_over_bank": med_a / med_b,
                        "pool_ms_range": [min(t_pool), max(t_pool)], "bank_ms_range": [min(t_bank), max(t_bank)],
                        "output_samples_per_channel": len(out_b[0]) // 2, "identical_bytes": True})
        bank.close()
        for r in pool:
            r.close()
    line = {
        "tool": "recorder_bank_bench",
        "device": bench.device_info(bench.gpu_bus_id(0), torch.cuda.get_device_name(0)),
        "input": {"sample_rate_hz": fs, "bandwidth_hz": bw, "samples_per_push": n_samples, "format": "CS8, device-resident", "stages": [list(s) for s in b2s.get_resamplers_factors(fs, bw)]},
        "reps": args.reps, "warmup": args.warmup,
        "results": results,
        "note": "(a) pool: K b2s_recorder_push calls one after another; (b) bank: one b2s_recorder_bank_push; CUDA-event medians",
    }
    print(json.dumps(line))
    eng.close()


if __name__ == "__main__":
    main()
