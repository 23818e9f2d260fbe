#!/usr/bin/env python
"""Kernel times (CUDA events inside the library) of K1 / K2 for a sweep of FFT sizes at a constant 2^26 samples per push.
Measurement helper for DESIGN.md / profiles (not part of the product path). Usage: python tools/size_sweep.py [N ...]"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as ge  # noqa: E402


def main():
    import torch

    b2s, synth = ge.load_b2s(), ge.load_synth()
    sizes = [int(x) for x in sys.argv[1:]] or [4096, 8192, 16384, 32768, 65536, 131072, 262144, 524288, 1048576]
    eng = b2s.Engine(0)
    dev = torch.device("cuda", 0)
    out = []
    for n in sizes:
        fs = 20_000_000
        T = (1 << 26) // n
        tones = [synth.Tone(0.31 * n / 2 + 0.1, fm_dev_bins=5.0), synth.Tone(-0.62 * n / 2 + 0.1, fm_dev_bins=5.0)]
        iq = synth.make_iq_int8_torch(n, T, tones, seed=n, quiet_frames=40, device=dev)
        cfg = b2s.make_config(n, fs, learn_frames=40, max_frames_per_push=T, flags=b2s.FLAG_IQ_ON_DEVICE | b2s.FLAG_ASYNC)
        band = b2s.Band(eng, cfg)
        band.set_profiling(True)
        period = synth.frame_period_ms(n, fs)
        t = 0
        for i in range(3):
            band.push_raw(iq.data_ptr(), T, int(t), period)
            t += T * period
        band.sync()
        band.get_profile(reset=True)
        reps = 10
        for i in range(reps):
            band.push_raw(iq.data_ptr(), T, int(t), period)
            t += T * period
        band.sync()
        p = band.get_profile(reset=True)
        k1, k2 = p.spectral_ms / p.spectral_launches, p.detect_ms / p.detect_launches
        row = {"n": n, "frames": T, "k1_ms": round(k1, 4), "k2_ms": round(k2, 4), "k1_gbs": round(6 * T * n / k1 / 1e6, 1), "k2_gbs": round(4 * T * n / k2 / 1e6, 1),
               "k1_gsps": round(T * n / k1 / 1e6, 3), "k1k2_gsps": round(T * n / (k1 + k2) / 1e6, 3),
               "host_ms": round(p.tracker_host_ms / reps, 4), "k4_ms": round(p.track_ms / max(p.track_launches, 1), 4),
               "k4_evals": p.track_evals / max(p.track_launches, 1), "k4_events": p.track_events / max(p.track_launches, 1)}
        print(json.dumps(row), flush=True)
        out.append(row)
        band.close()
        del iq
    return out


if __name__ == "__main__":
    main()
