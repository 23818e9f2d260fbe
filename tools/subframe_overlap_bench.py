#!/usr/bin/env python
"""What overlapping sub-frames (B2S_FLAG_SUBFRAME_OVERLAP) cost per push, beside back-to-back sub-frames and no sub-frames.

Four devices, each at the library's default configuration for its sample rate (b2s_default_config: N and the decimator factor r of the
reference's 50 frames per second), plus 20 MS/s at N = 16384 with a stride of 3 N:
  2.048 MS/s (N = 8192, r = 5), 20 MS/s (N = 131072, r = 3), 40 MS/s (N = 262144, r = 3), 20 MS/s at N = 16384 (r = 3).
The same sizes as tools/subframe_bench.py. For each, five asynchronous bands with CS8 IQ resident on the device (flags off, MEAN, MAX,
MEAN + OVERLAP, MAX + OVERLAP) push the same 2 s of synthetic IQ per step, in alternating order within one process; a step ends with
b2s_band_sync. Reported per push: K1 time (spectral_ms, CUDA events; the two small lead-in copies of the overlap sit outside it), K2
time (detect_ms), wall time on the host clock around push + sync, and the sub-frame transforms per second of K1 time (r = stride / N
back to back, m = stride / (N / 2) overlapping, 1 without sub-frames). Prints the card's name, power limit and clocks read in the
same run, and one JSON line.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SECONDS_PER_STEP = 2.0


def noise_and_carrier(torch, samples, n, seed):
    """int8 IQ on the device: Gaussian noise (sigma 8 LSB) and one carrier 0.1 N above the centre at 40 LSB."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    k = torch.arange(samples, device="cuda", dtype=torch.float64)
    ph = (2 * torch.pi * (0.1 * n + 0.1) / n * k).remainder(2 * torch.pi).float()
    x = torch.randn(samples, 2, device="cuda", generator=g) * 8.0
    x[:, 0] += 40.0 * torch.cos(ph)
    x[:, 1] += 40.0 * torch.sin(ph)
    return x.round().clamp(-128, 127).to(torch.int8).reshape(-1).contiguous()


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()

    import torch

    import __graft_entry__ as ge

    b2s = ge.load_b2s()
    if not torch.cuda.is_available():
        raise SystemExit("subframe_overlap_bench.py needs a CUDA device: the band has no CPU fallback")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    print("[gpu]", gpu)
    eng = b2s.Engine(0)
    devices = [("2.048 MS/s default", 2_048_000, None), ("20 MS/s default", 20_000_000, None), ("40 MS/s default", 40_000_000, None),
               ("20 MS/s N=16384 stride 3N", 20_000_000, (16384, 3))]
    ov = b2s.FLAG_SUBFRAME_OVERLAP
    modes = [("off", 0), ("mean", b2s.FLAG_SUBFRAME_MEAN), ("max", b2s.FLAG_SUBFRAME_MAX), ("mean+ov", b2s.FLAG_SUBFRAME_MEAN | ov),
             ("max+ov", b2s.FLAG_SUBFRAME_MAX | ov)]
    out = {"gpu": gpu, "devices": []}
    for name, fs, override in devices:
        cfg0 = b2s.BandConfig()
        b2s.lib().b2s_default_config(C.byref(cfg0), fs, 100_000_000, 32_000)
        if override:
            n, r = override
            cfg0 = b2s.make_config(n, fs, decimator=r)
        n, stride = cfg0.fft_size, cfg0.frame_stride_samples
        r = stride // n
        frames = int(SECONDS_PER_STEP * fs / stride)
        period = stride * 1000.0 / fs
        iq = noise_and_carrier(torch, frames * stride, n, seed=fs)
        bands = {}
        for mname, flag in modes:
            cfg = b2s.BandConfig.from_buffer_copy(cfg0)
            cfg.flags = flag | b2s.FLAG_ASYNC | b2s.FLAG_IQ_ON_DEVICE
            cfg.max_frames_per_push = frames
            cfg.learn_frames = 40
            band = b2s.Band(eng, cfg)
            band.set_profiling(True)
            bands[mname] = band
        stats = {m: {"spectral_ms": [], "detect_ms": [], "wall_ms": []} for m, _ in modes}
        for step in range(args.warmup + args.steps):
            order = [m for m, _ in modes] if step % 2 == 0 else [m for m, _ in reversed(modes)]
            for m in order:
                band = bands[m]
                band.get_profile(reset=True)
                torch.cuda.synchronize()
                t = time.perf_counter()
                band.push_raw(iq.data_ptr(), frames, int(step * SECONDS_PER_STEP * 1000), period)
                band.sync()
                wall = (time.perf_counter() - t) * 1e3
                p = band.get_profile(reset=True)
                if step >= args.warmup:
                    stats[m]["spectral_ms"].append(p.spectral_ms)
                    stats[m]["detect_ms"].append(p.detect_ms)
                    stats[m]["wall_ms"].append(wall)
        row = {"device": name, "fft_size": n, "r": r, "frames_per_push": frames}
        for m, flag in modes:
            med = {k: statistics.median(v) for k, v in stats[m].items()}
            subs = (stride // (n // 2) if flag & ov else r) if flag else 1
            med["transforms_per_s"] = frames * subs / (med["spectral_ms"] * 1e-3)
            row[m] = med
            print(f"{name:28s} {m:7s} K1 {med['spectral_ms']:8.3f} ms  K2 {med['detect_ms']:8.3f} ms  wall {med['wall_ms']:8.2f} ms"
                  f"  {subs:2d} transforms/frame, {med['transforms_per_s'] / 1e3:8.1f} k/s")
        out["devices"].append(row)
        for band in bands.values():
            band.close()
        del iq
        torch.cuda.empty_cache()
    eng.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
