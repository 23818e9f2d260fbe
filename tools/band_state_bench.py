"""Size and cost of a band snapshot (b2s_band_save_state / b2s_band_load_state) at config 2's geometry (N = 16384, 20 MS/s) and at
N = 1048576 (200 MS/s).

For each geometry a band runs one push of T frames of a keyed scene (device IQ), so that its noise is learned, its Averager full and
signals live. Then `--reps` times each, alternating: a save into a buffer of the right size (host clock around the call, which waits
for the band and copies its state to host memory), and a load of that snapshot into a second band created with the same config. Prints
one JSON line for the card (name, power limit, maximum SM clock) and one per geometry with the snapshot size and the times in ms
(mean, min, max).
Usage: python tools/band_state_bench.py [--reps R] [--sizes 16384,1048576]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import __graft_entry__ as ge  # noqa: E402

b2s, synth = ge.load_b2s(), ge.load_synth()
GEOMETRY = {16384: (20_000_000, 4096, 300), 1048576: (200_000_000, 1024, 16)}  # N -> (sample rate, frames of the push, learn frames)


def stat(v):
    return {"mean": round(sum(v) / len(v), 3), "min": round(min(v), 3), "max": round(max(v), 3)}


def measure(engine, n, reps, dev):
    fs, T, learn = GEOMETRY[n]
    cfg = b2s.make_config(n, fs, learn_frames=learn, flags=b2s.FLAG_ASYNC | b2s.FLAG_IQ_ON_DEVICE, max_frames_per_push=T)
    iq = synth.make_iq_int8_torch(n, T, synth.standard_scene(n, T, learn), seed=synth.seed_for(2), quiet_frames=learn, device=dev)
    band, other = b2s.Band(engine, cfg), b2s.Band(engine, cfg)
    band.push_raw(iq.data_ptr(), T, 0, synth.frame_period_ms(n, fs))
    band.sync()
    live = len(band.get_signals(cap=n)[0])
    L = b2s.lib()
    written = C.c_size_t(0)
    L.b2s_band_save_state(band._h, None, 0, C.byref(written))
    buf = np.empty(written.value, np.uint8)
    save_ms, load_ms = [], []
    for _ in range(reps):
        t0 = time.perf_counter()
        rc = L.b2s_band_save_state(band._h, buf.ctypes.data, buf.size, C.byref(written))
        save_ms.append((time.perf_counter() - t0) * 1e3)
        assert rc == 0, L.b2s_last_error()
        t0 = time.perf_counter()
        rc = L.b2s_band_load_state(other._h, buf.ctypes.data, buf.size)
        load_ms.append((time.perf_counter() - t0) * 1e3)
        assert rc == 0, L.b2s_last_error()
    assert other.save_state() == buf.tobytes()
    band.close()
    other.close()
    return {"N": n, "sample_rate_hz": fs, "frames_pushed": T, "live_signals": live, "snapshot_bytes": int(buf.size), "reps": reps,
            "save_ms": stat(save_ms), "load_ms": stat(load_ms)}


def main():
    import torch

    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--sizes", default="16384,1048576")
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"device": q}), flush=True)
    engine = b2s.Engine(0)
    for n in (int(s) for s in args.sizes.split(",")):
        print(json.dumps(measure(engine, n, args.reps, torch.device("cuda:0"))), flush=True)
        torch.cuda.empty_cache()
    engine.close()


if __name__ == "__main__":
    main()
