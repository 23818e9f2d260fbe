#!/usr/bin/env python
"""What auto-record costs and what its batched catch-up gains.

1. Step time. Config 4's scene (bench.py --config 4): 40 MS/s CS8 from synth (four keyed FM carriers, 32768-point frames, 2048 frames =
   67.1 M samples per step) in pinned host memory. Two synchronous bands, each with an attached 8-channel bank at 32 kS/s that keeps
   5 s of history; (b) records automatically with a 1 s pre-roll, (a) does not. After warm-up both push every step, for --steps steps,
   in alternating order; each push is timed on the host clock around b2s_band_push, which ends in the library's synchronise.
2. K channels started in one decision (K = 4, 16, 64). The same rate and frame size, K FM carriers that all appear 300 frames into the
   third push of 2048 frames. Band (b) records automatically with a 1 s pre-roll, so that push ends with K catch-ups of about 1 s +
   1750 frames each, batched; its twin (a), with the event log on, pushes the same frames and then starts the same channels at the same
   frames with K sequential b2s_band_record_from calls (the one-channel path: one catch-up after another). Reported: (b)'s push minus
   (a)'s push (the decision with its batched catch-up), and the sum of (a)'s K record_from calls; whether every channel's chunks agreed.
Prints the card's name and power limit read in the same run, and one JSON line.
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

BW, PREROLL_S, HISTORY_S = 32_000, 1, 5


def flushed(bank, channels):
    return [[(t, c.tobytes()) for t, c in bank.flush(ch, cap=1 << 16)] for ch in channels]


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()

    import torch

    import __graft_entry__ as ge
    import bench

    b2s, synth = ge.load_b2s(), ge.load_synth()
    if not torch.cuda.is_available():
        raise SystemExit("auto_record_bench.py needs a CUDA device: the band and the bank have no CPU fallback")
    wl = bench.WORKLOADS[4]
    n, fs, frames = wl["n"], wl["fs"], wl["frames"]
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    eng = b2s.Engine(0)
    period = synth.frame_period_ms(n, fs)
    frames_per_s = math.ceil(fs / n)
    history = HISTORY_S * frames_per_s * n
    cfg = b2s.make_config(n, fs, learn_frames=bench.LEARN, max_frames_per_push=frames)

    def pair(n_ch, log):
        bands, banks = [], []
        for auto in (False, True):
            bands.append(b2s.Band(eng, cfg))
            banks.append(b2s.RecorderBank(eng, fs, BW, n_ch, max_samples_per_push=frames * n))
            banks[-1].set_history(history)
            bands[-1].attach_recorder_bank(banks[-1])
            if auto:
                bands[-1].set_auto_record(True, PREROLL_S * frames_per_s)
            elif log:
                bands[-1].set_event_log(True)
        return bands, banks

    # ---- 1. step time, auto-record off and on ----
    iq8 = synth.make_iq_int8_torch(n, frames, bench.wideband_tones(synth, n, fs, frames, bench.LEARN), seed=synth.seed_for(4, 0), quiet_frames=bench.LEARN, device=dev)
    host = iq8.cpu().pin_memory()
    bands, banks = pair(8, False)
    ms = ([], [])
    n_actions = 0
    for step in range(args.warmup + args.steps):
        t0 = int(step * frames * period)
        for i in ((0, 1) if step % 2 == 0 else (1, 0)):  # alternate which band goes first
            w0 = time.perf_counter()
            bands[i].push_raw(host.data_ptr(), frames, t0, period)
            w1 = time.perf_counter()
            if step >= args.warmup:
                ms[i].append((w1 - w0) * 1e3)
        n_actions += len(bands[1].auto_record_actions())
        for k in banks:
            flushed(k, range(8))
    for x in bands + banks:
        x.close()
    results = [{"case": case, "step_ms_median": statistics.median(ms[i]), "step_ms_range": [min(ms[i]), max(ms[i])]}
               for i, case in enumerate(("a_auto_record_off", "b_auto_record_on"))]
    results.append({"auto_record_actions": n_actions})
    del iq8, host

    # ---- 2. K channels started in one decision: batched against sequential ----
    onset = 2 * frames + 300
    for k in (4, 16, 64):
        tones = [synth.Tone(bin_offset=-n // 2 + n // (k + 1) * (i + 1) + 0.1, amplitude=40.0, on_frames=[(onset, 3 * frames)], fm_dev_bins=6.0) for i in range(k)]
        iq8 = synth.make_iq_int8_torch(n, 3 * frames, tones, seed=synth.seed_for(4, 1), quiet_frames=bench.LEARN, device=dev)
        host = iq8.cpu().pin_memory()
        bands, banks = pair(k, True)
        push_ms = [0.0, 0.0]
        for p in range(3):
            for i in (0, 1):
                w0 = time.perf_counter()
                bands[i].push_raw(host.data_ptr() + p * frames * n * 2, frames, int(p * frames * period), period)
                push_ms[i] = (time.perf_counter() - w0) * 1e3
        acts = [a for a in bands[1].auto_record_actions() if a[0] == b2s.REC_START]
        seq_ms = []
        for kind, ch, shift, key, frame, from_frame, t, dur in acts:
            w0 = time.perf_counter()
            if from_frame >= 0:
                bands[0].record_from(ch, shift, from_frame)
            else:
                banks[0].start(ch, shift)
            seq_ms.append((time.perf_counter() - w0) * 1e3)
        agree = flushed(banks[0], range(k)) == flushed(banks[1], range(k))
        results.append({"case": f"start_{k}_channels", "started": len(acts), "from_history": sum(1 for a in acts if a[5] >= 0),
                        "catch_up_frames_mean": statistics.mean(frame + 1 - a[5] for a in acts if a[5] >= 0) if acts else 0,
                        "batched_ms": push_ms[1] - push_ms[0], "sequential_ms": sum(seq_ms), "push_ms": {"plain": push_ms[0], "auto": push_ms[1]},
                        "chunks_agree": agree})
        for x in bands + banks:
            x.close()
        del iq8, host
    line = {
        "tool": "auto_record_bench",
        "device": bench.device_info(bench.gpu_bus_id(0), torch.cuda.get_device_name(0)),
        "input": {"sample_rate_hz": fs, "fft_size": n, "frames_per_step": frames, "format": "cs8", "host_memory": "pinned", "bandwidth_hz": BW,
                  "history_s": HISTORY_S, "preroll_s": PREROLL_S, "stages": [list(s) for s in b2s.get_resamplers_factors(fs, BW)]},
        "steps": args.steps, "warmup": args.warmup,
        "results": results,
        "note": "step: b2s_band_push wall time with auto-record off (a) and on (b), alternating; start_K: (b)'s push with K starts minus the "
                "same push on a band without auto-record, against the K sequential b2s_band_record_from calls that start the same channels",
    }
    print(json.dumps(line))
    eng.close()


if __name__ == "__main__":
    main()
