"""K4 (the device tracker) per push in busy spectrum, next to K1 + K2, with the card it ran on. Prints one JSON line per scene.

Scenes (IQ generated on the device from a seed, pushed from device memory, asynchronous bands as bench.py runs them):
  busy_n16384   N = 16384 at 20 MS/s, T = 4096: two 6 MHz noise blocks that stay on, a third that switches every 300 frames,
                40 narrow carriers; several hundred live signals (k_track_wide runs the pushes)
  busy_n1048576 N = 1048576 at 200 MS/s, T = 1024: two 8 MHz blocks and 40 carriers
  config2       bench.py's config 2 scene (four keyed carriers, N = 16384, T = 4096): k_track runs every push
For each: K4 ms per push (track_ms / pushes; track_ms spans k_track and k_track_wide), K1 and K2 ms per push, K4 / K1 (K4 runs
beside the next push's K1, on the SM K1 leaves free: a ratio below 1 means it stays hidden there), the pushes k_track_wide ran,
and event frames and getBestIndex calls per push. Usage: python tools/busy_track_bench.py [--pushes P]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import __graft_entry__ as entry  # noqa: E402

b2s = entry.load_b2s()
synth = entry.load_synth()


def busy_iq_torch(n, fs, frames, blocks, n_carriers, learn, seed, device, snr_db=22.0, sigma=8.0):
    """Like tests/test_busy_spectrum.busy_iq, on the device: blocks are (lo Hz, hi Hz, first frame, end frame, period) with
    period > 0 switching the block every `period` frames inside [first, end)."""
    import torch

    g = torch.Generator(device=device).manual_seed(seed)
    out = torch.empty((frames, n, 2), dtype=torch.int8, device=device)
    amp = sigma * (n * 10 ** (snr_db / 10)) ** 0.5
    tone = sigma * (2 * 1000 / n) ** 0.5
    rng = torch.Generator().manual_seed(seed)
    carriers = [(int(torch.randint(0, n, (1,), generator=rng)), int(torch.randint(learn, frames, (1,), generator=rng)), int(torch.randint(3, 200, (1,), generator=rng)))
                for _ in range(n_carriers)]
    t = torch.arange(n, device=device, dtype=torch.float64)
    chunk = max(1, (1 << 24) // n)
    for f0 in range(0, frames, chunk):
        f1 = min(frames, f0 + chunk)
        x = torch.complex(torch.randn((f1 - f0, n), generator=g, device=device, dtype=torch.float64), torch.randn((f1 - f0, n), generator=g, device=device, dtype=torch.float64)) * sigma
        spec = torch.zeros((f1 - f0, n), dtype=torch.complex128, device=device)
        fr = torch.arange(f0, f1, device=device)
        for lo_hz, hi_hz, a, b, period in blocks:
            lo, hi = int(n // 2 + lo_hz * n / fs), int(n // 2 + hi_hz * n / fs)
            on = (fr >= a) & (fr < b)
            if period:
                on &= ((fr - a) // period) % 2 == 0
            w = torch.complex(torch.randn((f1 - f0, hi - lo), generator=g, device=device, dtype=torch.float64), torch.randn((f1 - f0, hi - lo), generator=g, device=device, dtype=torch.float64))
            spec[:, lo:hi] += w * (amp / 2 ** 0.5) * on[:, None]
        x += torch.fft.ifft(torch.fft.ifftshift(spec, dim=1), dim=1)
        for b_, a, d in carriers:
            on = ((fr >= a) & (fr < a + d))[:, None]
            x += torch.exp(2j * torch.pi * ((b_ - n // 2) % n) * t / n)[None, :] * tone * on
        out[f0:f1, :, 0] = torch.clamp(torch.round(x.real), -127, 127).to(torch.int8)
        out[f0:f1, :, 1] = torch.clamp(torch.round(x.imag), -127, 127).to(torch.int8)
        del x, spec
    return out.reshape(-1)


def measure(engine, name, cfg, iq, T, pushes):
    """One warm-up push, then `pushes` timed ones, all of the same scene in sequence."""
    import torch

    n = cfg.fft_size
    cfg.flags |= b2s.FLAG_ASYNC | b2s.FLAG_IQ_ON_DEVICE
    cfg.max_frames_per_push = T
    band = b2s.Band(engine, cfg)
    band.push_raw(iq.data_ptr(), T, 0, 1.0)
    band.sync()
    band.set_profiling(True)
    band.get_profile(reset=True)
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for k in range(1, pushes + 1):
        band.push_raw(iq.data_ptr() + k * T * 2 * n, T, k * T, 1.0)
    res = band.sync()
    end.record()
    torch.cuda.synchronize()
    p = band.get_profile()
    live = len(band.get_signals(cap=n)[0])
    band.close()
    k1, k2, k4 = p.spectral_ms / pushes, p.detect_ms / pushes, p.track_ms / pushes
    return {"scene": name, "N": n, "T": T, "pushes": pushes, "k4_ms_per_push": round(k4, 4), "k1_ms_per_push": round(k1, 4), "k2_ms_per_push": round(k2, 4),
            "k4_over_k1": round(k4 / k1, 3), "wide_pushes": int(p.track_launches - pushes), "events_per_push": p.track_events / pushes,
            "best_index_per_push": p.track_best_index / pushes, "live_signals_after": live, "transmissions_after": res.n_transmissions_total,
            "wall_ms_per_push_profiled": round(start.elapsed_time(end) / pushes, 3)}


def main():
    import torch

    ap = argparse.ArgumentParser()
    ap.add_argument("--pushes", type=int, default=3)
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"device": q}))
    engine = b2s.Engine(0)
    dev = torch.device("cuda:0")
    P = args.pushes
    # busy, N = 16384, T = 4096
    n, fs, T = 16384, 20_000_000, 4096
    iq = busy_iq_torch(n, fs, (P + 1) * T, [(-9.0e6, -3.0e6, 100, 10**9, 0), (0.5e6, 6.5e6, 150, 10**9, 0), (-2.5e6, 0.0, 200, 10**9, 300)], 40, 20, 11, dev)
    cfg = b2s.make_config(n, fs, learn_frames=20, recording_bandwidth_hz=32_000, min_time_ms=12, timeout_ms=25, start_level=4.0, stop_level=2.0, detect_capacity=n)
    print(json.dumps(measure(engine, "busy_n16384", cfg, iq, T, P)))
    del iq
    torch.cuda.empty_cache()
    # busy, N = 1048576, T = 1024
    n, fs, T = 1048576, 200_000_000, 1024
    iq = busy_iq_torch(n, fs, (P + 1) * T, [(-60.0e6, -52.0e6, 30, 10**9, 0), (10.0e6, 18.0e6, 40, 10**9, 0)], 40, 16, 12, dev)
    cfg = b2s.make_config(n, fs, learn_frames=16, recording_bandwidth_hz=32_000, min_time_ms=12, timeout_ms=25, start_level=4.0, stop_level=2.0, detect_capacity=n)
    print(json.dumps(measure(engine, "busy_n1048576", cfg, iq, T, P)))
    del iq
    torch.cuda.empty_cache()
    # bench.py's config 2 scene
    import bench

    n, fs, T = 16384, 20_000_000, 4096
    iq = synth.make_iq_int8_torch(n, (P + 1) * T, bench.bench_tones(synth, n, (P + 1) * T, bench.LEARN), seed=synth.seed_for(2), quiet_frames=bench.LEARN, device=dev)
    cfg = b2s.make_config(n, fs, learn_frames=bench.LEARN)
    print(json.dumps(measure(engine, "config2", cfg, iq, T, P)))
    engine.close()


if __name__ == "__main__":
    main()
