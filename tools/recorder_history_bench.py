#!/usr/bin/env python
"""What a recorder bank's history costs: the band's step with the history off and on, and the catch-up of b2s_band_record_from.

Input: config 4's scene (bench.py --config 4): 40 MS/s CS8 from synth (four keyed FM carriers, 32768-point frames, 2048 frames = 67.1 M
samples per step) in pinned host memory. Two synchronous bands, each with an attached bank whose first four channels record config 4's
shifts at 32 kS/s: (a) keeps no history, (b) keeps 5 s of it (b2s_recorder_bank_set_history, 200 M samples = 400 MB). After warm-up
both push every step, for --steps steps, in alternating order; each push is timed on the host clock around b2s_band_push, which
ends in the library's synchronise. Then, on (b), b2s_band_record_from starts the fifth channel 1 s and 5 s before the newest frame (a catch-up of 40 M and
200 M samples), --reps times each, timed the same way (the call is synchronous); the channel is stopped between repetitions.
Reports medians and min-max, whether the two banks' flushed chunks (bytes and times) agreed after every step, and the card's name and
power limit read in the same run, as one JSON line.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()

    import torch

    import __graft_entry__ as ge
    import bench

    b2s, synth = ge.load_b2s(), ge.load_synth()
    if not torch.cuda.is_available():
        raise SystemExit("recorder_history_bench.py needs a CUDA device: the band and the bank have no CPU fallback")
    wl = bench.WORKLOADS[4]
    n, fs, frames, bw = wl["n"], wl["fs"], wl["frames"], 32_000
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    eng = b2s.Engine(0)
    iq8 = synth.make_iq_int8_torch(n, frames, bench.wideband_tones(synth, n, fs, frames, bench.LEARN), seed=synth.seed_for(4, 0), quiet_frames=bench.LEARN, device=dev)
    host = iq8.cpu().pin_memory()
    ptr, n_samples = host.data_ptr(), frames * n
    period = synth.frame_period_ms(n, fs)
    shifts = [b2s.get_tuned_frequency(int(mhz * 1e6), 2500) for mhz in (-12.5, -3.2, 4.7, 15.1)]
    frames_per_s = math.ceil(fs / n)
    history = 5 * frames_per_s * n  # whole frames, so that a 5 s pre-roll starts at the oldest one held
    if (args.warmup + args.steps) * frames < 5 * frames_per_s:
        raise SystemExit("too few steps to fill 5 s of history")

    cfg = b2s.make_config(n, fs, learn_frames=bench.LEARN, max_frames_per_push=frames)
    bands, banks = [], []
    for keep in (0, history):
        bands.append(b2s.Band(eng, cfg))
        banks.append(b2s.RecorderBank(eng, fs, bw, len(shifts) + 1, max_samples_per_push=n_samples))
        banks[-1].set_history(keep)
        for c, s in enumerate(shifts):
            banks[-1].start(c, s)
        bands[-1].attach_recorder_bank(banks[-1])

    def flushed(bank):
        return [[(t, c.tobytes()) for t, c in bank.flush(ch, cap=1 << 16)] for ch in range(len(shifts))]

    ms = ([], [])
    agree, chunks = True, 0
    for step in range(args.warmup + args.steps):
        t0 = int(step * frames * period)
        for i in ((0, 1) if step % 2 == 0 else (1, 0)):  # alternate which band goes first
            w0 = time.perf_counter()
            bands[i].push_raw(ptr, frames, t0, period)
            w1 = time.perf_counter()
            if step >= args.warmup:
                ms[i].append((w1 - w0) * 1e3)
        fa, fb = flushed(banks[0]), flushed(banks[1])
        agree = agree and fa == fb
        chunks += sum(len(x) for x in fb)
    newest = (args.warmup + args.steps) * frames  # band frames pushed
    catch_up = {}
    for seconds in (1, 5):
        times = []
        for _ in range(args.reps):
            w0 = time.perf_counter()
            bands[1].record_from(len(shifts), shifts[0], newest - seconds * frames_per_s)
            w1 = time.perf_counter()
            times.append((w1 - w0) * 1e3)
            banks[1].stop(len(shifts))
        catch_up[seconds] = times
    for x in bands + banks:
        x.close()
    results = [{"case": case, "step_ms_median": statistics.median(ms[i]), "step_ms_range": [min(ms[i]), max(ms[i])]}
               for i, case in enumerate(("a_history_off", "b_history_5s"))]
    results.append({"bank_bytes_agree": agree, "chunks_compared": chunks})
    for seconds, times in catch_up.items():
        results.append({"case": f"record_from_preroll_{seconds}s", "catch_up_samples": seconds * frames_per_s * n, "ms_median": statistics.median(times),
                        "ms_range": [min(times), max(times)]})
    line = {
        "tool": "recorder_history_bench",
        "device": bench.device_info(bench.gpu_bus_id(0), torch.cuda.get_device_name(0)),
        "input": {"sample_rate_hz": fs, "fft_size": n, "frames_per_step": frames, "samples_per_step": n_samples, "format": "cs8", "host_memory": "pinned",
                  "bandwidth_hz": bw, "shifts_hz": shifts, "stages": [list(s) for s in b2s.get_resamplers_factors(fs, bw)], "history_samples": history},
        "steps": args.steps, "warmup": args.warmup, "reps": args.reps,
        "results": results,
        "note": "step: b2s_band_push wall time with the attached bank's history off (a) and 5 s (b), alternating; record_from: wall time of one "
                "b2s_band_record_from whose catch-up is the given pre-roll",
    }
    print(json.dumps(line))
    eng.close()


if __name__ == "__main__":
    main()
