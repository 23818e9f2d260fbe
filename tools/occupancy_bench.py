#!/usr/bin/env python
"""What spectrum occupancy (b2s_band_set_occupancy) costs per push.

Two scenes at N = 16384, 20 MS/s, T = 4096 frames per push, IQ resident on the device, asynchronous bands as bench.py runs them:
  config2       bench.py's config 2 scene (four keyed carriers): few detection entries per frame
  busy_n16384   tools/busy_track_bench.py's busy scene (three 6 MHz noise blocks, 40 carriers, levels 4 / 2 dB, detect_capacity = N):
                thousands of entries per frame
For each scene two bands, occupancy off and on, push the same IQ, alternating in one process; a push ends with b2s_band_sync.
Reported per push (medians): K1 and K2 time (b2s_profile: CUDA events on the band's stream), the wall time of push + sync on the host
clock, and the two occupancy kernels' device time from a separate torch.profiler pass (CUDA activity records, not the timed pushes).
The card's name, power limit and SM clocks are read in the same run. Prints one JSON line per scene.
Usage: python tools/occupancy_bench.py [--steps K] [--warmup W]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import __graft_entry__ as entry  # noqa: E402

b2s = entry.load_b2s()
synth = entry.load_synth()


def occupancy_kernel_ms(torch, band, iq, T, period, pushes):
    """Device time per push of k_occupancy_count and k_occupancy_max, from torch.profiler's CUDA activity records."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for p in range(pushes):
            band.push_raw(iq.data_ptr(), T, (1000 + p) * 100_000, period)
            band.sync()
        torch.cuda.synchronize()
    total = {"k_occupancy_count": 0.0, "k_occupancy_max": 0.0}
    for e in prof.events():
        for k in total:
            if k in e.name:
                total[k] += e.device_time_total / 1000.0
    return {k: v / pushes for k, v in total.items()}


def measure(torch, engine, name, cfg0, iq, T, steps, warmup):
    period = cfg0.frame_stride_samples * 1000.0 / cfg0.sample_rate_hz
    bands = {}
    for mode in ("off", "on"):
        cfg = b2s.BandConfig.from_buffer_copy(cfg0)
        cfg.flags |= b2s.FLAG_ASYNC | b2s.FLAG_IQ_ON_DEVICE
        cfg.max_frames_per_push = T
        band = b2s.Band(engine, cfg)
        band.set_occupancy(mode == "on")
        band.set_profiling(True)
        bands[mode] = band
    stats = {m: {"k1_ms": [], "k2_ms": [], "wall_ms": []} for m in bands}
    for step in range(warmup + steps):
        for m in (("off", "on") if step % 2 == 0 else ("on", "off")):
            band = bands[m]
            band.get_profile(reset=True)
            torch.cuda.synchronize()
            t = time.perf_counter()
            band.push_raw(iq.data_ptr(), T, step * 100_000, period)
            band.sync()
            wall = (time.perf_counter() - t) * 1e3
            p = band.get_profile(reset=True)
            if step >= warmup:
                stats[m]["k1_ms"].append(p.spectral_ms)
                stats[m]["k2_ms"].append(p.detect_ms)
                stats[m]["wall_ms"].append(wall)
    row = {"scene": name, "fft_size": cfg0.fft_size, "frames_per_push": T, "steps": steps}
    for m in bands:
        row[m] = {k: statistics.median(v) for k, v in stats[m].items()}
        row[m]["wall_ms_min"], row[m]["wall_ms_max"] = min(stats[m]["wall_ms"]), max(stats[m]["wall_ms"])
    bands["on"].set_profiling(False)
    row["on"].update(occupancy_kernel_ms(torch, bands["on"], iq, T, period, 3))
    occ = bands["on"].occupancy(cfg0.center_hz)
    row["on"]["entries_above_stop_per_frame"] = float(occ.above_stop.sum()) / max(occ.detect_frames, 1)
    row["psd_bytes_per_push"] = 4 * T * cfg0.fft_size
    for band in bands.values():
        band.close()
    return row


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("occupancy_bench.py needs a CUDA device: the band has no CPU fallback")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True,
                       text=True).stdout.strip()
    print(json.dumps({"device": q}))
    engine = b2s.Engine(0)
    dev = torch.device("cuda:0")
    n, fs, T = 16384, 20_000_000, 4096
    import bench
    from busy_track_bench import busy_iq_torch

    iq = synth.make_iq_int8_torch(n, T, bench.bench_tones(synth, n, T, bench.LEARN), seed=synth.seed_for(2), quiet_frames=bench.LEARN, device=dev)
    cfg = b2s.make_config(n, fs, learn_frames=bench.LEARN)
    print(json.dumps(measure(torch, engine, "config2", cfg, iq, T, args.steps, args.warmup)))
    del iq
    torch.cuda.empty_cache()
    iq = busy_iq_torch(n, fs, T, [(-9.0e6, -3.0e6, 100, 10**9, 0), (0.5e6, 6.5e6, 150, 10**9, 0), (-2.5e6, 0.0, 200, 10**9, 300)], 40, 20, 11, dev)
    cfg = b2s.make_config(n, fs, learn_frames=20, recording_bandwidth_hz=32_000, min_time_ms=12, timeout_ms=25, start_level=4.0, stop_level=2.0, detect_capacity=n)
    print(json.dumps(measure(torch, engine, "busy_n16384", cfg, iq, T, args.steps, args.warmup)))
    q = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,temperature.gpu", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"after": q}))
    engine.close()


if __name__ == "__main__":
    main()
