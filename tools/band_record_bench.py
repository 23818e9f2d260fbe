#!/usr/bin/env python
"""Detection and recording from one host stream: today's two calls against one push with the recorder bank attached to the band.

Input: config 4's scene (bench.py --config 4): 40 MS/s from synth (four keyed FM carriers, 32768-point frames, 2048 frames = 67.1 M
samples per step) in pinned host memory, as CS8 and as CF32. A bank of four channels records config 4's shifts at 32 kS/s. Per format,
after warm-up, the two cases alternate for --steps steps, each on its own band and bank:
  (a) b2s_band_push, then b2s_recorder_bank_push of the same buffer: the samples cross PCIe twice;
  (b) one b2s_band_push with the bank attached (b2s_band_attach_recorder_bank): the bank reads the band's copy.
Each step is timed on the host clock around calls that end in the library's synchronise (synchronous band). Reports per case the
median, min and max wall time per step and the bytes uploaded per step (the band's profiled h2d_bytes; in (a) plus the bank push's
samples times bytes per sample, computed, since the bank keeps no profile), and whether the banks' flushed chunks (bytes and times) agree
after every step. Prints one JSON line with the card's name and power limit read in the same run.
"""
from __future__ import annotations

import argparse
import json
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
    ap.add_argument("--formats", nargs="+", default=["cs8", "cf32"], choices=["cs8", "cf32"])
    args = ap.parse_args()

    import torch

    import __graft_entry__ as ge
    import bench

    b2s, synth = ge.load_b2s(), ge.load_synth()
    if not torch.cuda.is_available():
        raise SystemExit("band_record_bench.py needs a CUDA device: the band and the recorders have no CPU fallback")
    wl = bench.WORKLOADS[4]
    n, fs, frames, bw = wl["n"], wl["fs"], wl["frames"], 32_000
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    eng = b2s.Engine(0)
    iq8 = synth.make_iq_int8_torch(n, frames, bench.wideband_tones(synth, n, fs, frames, bench.LEARN), seed=synth.seed_for(4, 0), quiet_frames=bench.LEARN, device=dev)
    n_samples = frames * n
    period = synth.frame_period_ms(n, fs)
    shifts = [b2s.get_tuned_frequency(int(mhz * 1e6), 2500) for mhz in (-12.5, -3.2, 4.7, 15.1)]

    def flushed(bank):
        return [[(t, c.tobytes()) for t, c in bank.flush(ch, cap=1 << 16)] for ch in range(len(shifts))]

    results = []
    for name in args.formats:
        fmt = b2s.IQ_CS8 if name == "cs8" else b2s.IQ_CF32
        src = iq8 if fmt == b2s.IQ_CS8 else iq8.to(torch.float32) * (1.0 / 127.0)
        host = src.cpu().pin_memory()
        ptr, bps = host.data_ptr(), 2 * host.element_size()
        cfg = b2s.make_config(n, fs, iq_format=fmt, learn_frames=bench.LEARN, max_frames_per_push=frames)
        bands, banks = [], []
        for _ in range(2):
            bands.append(b2s.Band(eng, cfg))
            banks.append(b2s.RecorderBank(eng, fs, bw, len(shifts), iq_format=fmt, max_samples_per_push=n_samples))
            for c, s in enumerate(shifts):
                banks[-1].start(c, s)
        bands[1].attach_recorder_bank(banks[1])

        def step_a(t0):
            bands[0].push_raw(ptr, frames, t0, period)
            banks[0].push(ptr, t0, n_samples=n_samples)

        def step_b(t0):
            bands[1].push_raw(ptr, frames, t0, period)

        ms = ([], [])
        h2d = ([], [])
        agree, chunks = True, 0
        for step in range(args.warmup + args.steps):
            t0 = int(step * frames * period)
            for i, fn in enumerate((step_a, step_b)):
                bands[i].get_profile(reset=True)
                w0 = time.perf_counter()
                fn(t0)
                w1 = time.perf_counter()
                up = bands[i].get_profile(reset=True).h2d_bytes + (n_samples * bps if i == 0 else 0)
                if step >= args.warmup:
                    ms[i].append((w1 - w0) * 1e3)
                    h2d[i].append(up)
            fa, fb = flushed(banks[0]), flushed(banks[1])
            agree = agree and fa == fb
            chunks += sum(len(x) for x in fb)
        for x in bands + banks:
            x.close()
        for i, case in enumerate(("a_band_then_bank", "b_attached")):
            results.append({"format": name, "case": case, "step_ms_median": statistics.median(ms[i]), "step_ms_range": [min(ms[i]), max(ms[i])],
                            "h2d_bytes_per_step": statistics.median(h2d[i]), "gsamples_per_s": n_samples / statistics.median(ms[i]) / 1e6})
        results.append({"format": name, "bank_bytes_agree": agree, "chunks_compared": chunks})
    line = {
        "tool": "band_record_bench",
        "device": bench.device_info(bench.gpu_bus_id(0), torch.cuda.get_device_name(0)),
        "input": {"sample_rate_hz": fs, "fft_size": n, "frames_per_step": frames, "samples_per_step": n_samples, "bandwidth_hz": bw, "shifts_hz": shifts,
                  "host_memory": "pinned", "stages": [list(s) for s in b2s.get_resamplers_factors(fs, bw)]},
        "steps": args.steps, "warmup": args.warmup,
        "results": results,
        "note": "(a) b2s_band_push then b2s_recorder_bank_push of the same host buffer; (b) b2s_band_push with the bank attached; wall time per step; "
                "h2d_bytes_per_step is the band's profiled h2d_bytes, plus, in (a), the bank push's samples x bytes per sample (the bank keeps no profile)",
    }
    print(json.dumps(line))
    eng.close()


if __name__ == "__main__":
    main()
