"""What the signal event log costs: K4 time and end-to-end time per push with the log off and on, on the scenes of
tools/busy_track_bench.py (config 2's scene and the two busy scenes; device-resident IQ, asynchronous bands).

For each scene the two settings alternate, `--reps` times each, in one process. A repetition creates a band, runs one warm-up
push, then times `--pushes` pushes of the same scene: `track_ms` per push from CUDA events inside the library (it spans k_track
and k_track_wide), and wall ms per push from the host clock around the pushes and the b2s_band_sync that ends them (profiling
on, so this is a little above an unprofiled run for both settings alike). Prints one JSON line for the card and one per scene,
with the mean and the range over the repetitions.
Usage: python tools/event_log_bench.py [--pushes P] [--reps R] [--scenes config2,busy_n16384,busy_n1048576]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import busy_track_bench as btb  # noqa: E402

b2s, synth = btb.b2s, btb.synth


def one_rep(engine, cfg, iq, T, pushes, log_on):
    n = cfg.fft_size
    band = b2s.Band(engine, cfg)
    band.set_event_log(log_on)
    band.push_raw(iq.data_ptr(), T, 0, 1.0)
    band.sync()
    band.get_events()
    band.set_profiling(True)
    band.get_profile(reset=True)
    t0 = time.perf_counter()
    for k in range(1, pushes + 1):
        band.push_raw(iq.data_ptr() + k * T * 2 * n, T, k * T, 1.0)
    band.sync()
    wall = (time.perf_counter() - t0) * 1e3 / pushes
    p = band.get_profile()
    events = band.event_count()
    band.close()
    return p.track_ms / pushes, wall, events / pushes, int(p.track_launches - pushes), p.d2h_bytes / pushes


def measure(engine, name, cfg, iq, T, pushes, reps):
    cfg.flags |= b2s.FLAG_ASYNC | b2s.FLAG_IQ_ON_DEVICE
    cfg.max_frames_per_push = T
    runs = {False: [], True: []}
    for _ in range(reps):
        for log_on in (False, True):
            runs[log_on].append(one_rep(engine, cfg, iq, T, pushes, log_on))

    def stat(rows, i):
        v = [r[i] for r in rows]
        return {"mean": round(sum(v) / len(v), 4), "min": round(min(v), 4), "max": round(max(v), 4)}

    out = {"scene": name, "N": cfg.fft_size, "T": T, "pushes": pushes, "reps": reps, "wide_pushes": runs[True][0][3], "events_per_push": runs[True][0][2]}
    for log_on, key in ((False, "off"), (True, "on")):
        out[f"k4_ms_per_push_{key}"] = stat(runs[log_on], 0)
        out[f"wall_ms_per_push_{key}"] = stat(runs[log_on], 1)
        out[f"d2h_bytes_per_push_{key}"] = runs[log_on][0][4]
    assert runs[False][0][2] == 0, "a band with the log off logged events"
    return out


def main():
    import torch

    ap = argparse.ArgumentParser()
    ap.add_argument("--pushes", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--scenes", default="config2,busy_n16384,busy_n1048576")
    args = ap.parse_args()
    scenes = args.scenes.split(",")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"device": q}), flush=True)
    engine = b2s.Engine(0)
    dev = torch.device("cuda:0")
    P = args.pushes
    busy = dict(recording_bandwidth_hz=32_000, min_time_ms=12, timeout_ms=25, start_level=4.0, stop_level=2.0)
    if "config2" in scenes:
        import bench

        n, fs, T = 16384, 20_000_000, 4096
        iq = synth.make_iq_int8_torch(n, (P + 1) * T, bench.bench_tones(synth, n, (P + 1) * T, bench.LEARN), seed=synth.seed_for(2), quiet_frames=bench.LEARN, device=dev)
        print(json.dumps(measure(engine, "config2", b2s.make_config(n, fs, learn_frames=bench.LEARN), iq, T, P, args.reps)), flush=True)
        del iq
        torch.cuda.empty_cache()
    if "busy_n16384" in scenes:
        n, fs, T = 16384, 20_000_000, 4096
        iq = btb.busy_iq_torch(n, fs, (P + 1) * T, [(-9.0e6, -3.0e6, 100, 10**9, 0), (0.5e6, 6.5e6, 150, 10**9, 0), (-2.5e6, 0.0, 200, 10**9, 300)], 40, 20, 11, dev)
        print(json.dumps(measure(engine, "busy_n16384", b2s.make_config(n, fs, learn_frames=20, detect_capacity=n, **busy), iq, T, P, args.reps)), flush=True)
        del iq
        torch.cuda.empty_cache()
    if "busy_n1048576" in scenes:
        n, fs, T = 1048576, 200_000_000, 1024
        iq = btb.busy_iq_torch(n, fs, (P + 1) * T, [(-60.0e6, -52.0e6, 30, 10**9, 0), (10.0e6, 18.0e6, 40, 10**9, 0)], 40, 16, 12, dev)
        print(json.dumps(measure(engine, "busy_n1048576", b2s.make_config(n, fs, learn_frames=16, detect_capacity=n, **busy), iq, T, P, args.reps)), flush=True)
        del iq
    engine.close()


if __name__ == "__main__":
    main()
