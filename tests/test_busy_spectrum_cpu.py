"""The host tracker (tracker.h) in busy spectrum: PSD-row scenes with more than 256 live signals and frames with more than 2048
start-level candidates, the regime the device tracker hands to k_track_wide. b2s.HostTransmission, fed the oracle's NoiseLearner
and boxcar rows, must give every frame's list and total count exactly as the oracle chain does."""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as ol
from conftest import load_b2s

b2s = load_b2s()

PERIOD_MS = 100.0  # NOISE_LEARNING_TIME = 2000 ms (config.h:24) = 21 frames of this clock, as the reference objects learn
T0 = 1_700_000_000_000


def _scene(seed):
    """N = 4096 at 4.096 MS/s (1 kHz bins, group 7 bins): three blocks of 900-1800 bins that switch on and off, two of them at
    once, and dozens of narrow carriers."""
    rng = np.random.default_rng(4200 + seed)
    n, fs, frames = 4096, 4_096_000, 150
    learn = b2s.lib().b2s_learn_frames_from_ms(2000, C.c_double(PERIOD_MS))
    bw = 7 * fs // n
    cfg = b2s.make_config(n, fs, learn_frames=learn, recording_bandwidth_hz=bw, min_time_ms=300, timeout_ms=int(rng.choice([400, 900])))
    psd = (-60.0 + 1.5 * rng.standard_normal((frames, n))).astype(np.float32)
    bins = np.arange(n)
    on = int(rng.integers(learn + 5, learn + 20))
    for lo, width, a, b in ((int(rng.integers(0, 600)), int(rng.integers(1100, 1800)), on, on + 60),
                            (int(rng.integers(2200, 2500)), int(rng.integers(1100, 1500)), on, on + 45),
                            (int(rng.integers(1000, 2000)), int(rng.integers(900, 1200)), on + 75, frames)):
        psd[a:b, lo : lo + width] += (25.0 + 4.0 * rng.standard_normal((b - a, width))).astype(np.float32)
    for _ in range(40):
        c, a = float(rng.integers(0, n)), int(rng.integers(learn, frames))
        level, width = float(rng.uniform(15.0, 50.0)), float(rng.uniform(1.0, 4.0))
        for t in range(a, min(frames, a + int(rng.integers(3, 30)))):
            psd[t] += (level * np.exp(-0.5 * ((bins - c) / width) ** 2)).astype(np.float32)
    return cfg, psd, frames


def _host_push(h, box, q):
    """HostTransmission.push that also returns every frame's total count."""
    frames, n = box.shape
    count = np.zeros(frames, np.int32)
    tx = (b2s.Transmission * (frames * b2s.MAX_TX))()
    box, q = np.ascontiguousarray(box, np.float32), np.ascontiguousarray(q, np.float32)
    rc = b2s.lib().b2s_host_transmission_push(h._h, box.ctypes.data, q.ctypes.data, frames, T0, PERIOD_MS, 1, count.ctypes.data, C.cast(tx, C.c_void_p))
    assert rc == 0
    lists = [[(tx[k * b2s.MAX_TX + i].shift_hz, tx[k * b2s.MAX_TX + i].flush, tx[k * b2s.MAX_TX + i].key, np.float32(tx[k * b2s.MAX_TX + i].power))
              for i in range(min(int(count[k]), b2s.MAX_TX))] for k in range(frames)]
    return count, lists


@pytest.mark.parametrize("seed", range(3))
def test_busy_scene_host_tracker_equals_the_oracle(seed):
    cfg, psd, frames = _scene(seed)
    r = ol.OracleChain(cfg).push(psd, frames, T0, PERIOD_MS, dense=("noise_sub_db", "box_db"), psd_rows=True)
    want = [[(f, fl, k, np.float32(p)) for f, fl, k, p in fr] for fr in r.frame_tx]
    count, got = _host_push(b2s.HostTransmission(cfg), r.box_db, r.noise_sub_db)
    bad = [k for k in range(frames) if got[k] != want[k] or count[k] != r.tx_count[k]]
    assert not bad, f"seed {seed}: first differing frame {bad[0]}: count {count[bad[0]]} / {r.tx_count[bad[0]]}"
    # the scene passes both caps of k_track: > 256 live signals, and > 2048 candidates in a frame whose map changed
    cand = (r.box_db >= np.float32(cfg.start_level)).sum(axis=1)
    events = np.concatenate([[False], count[1:] != count[:-1]])
    print(f"\nseed {seed}: at most {count.max()} live signals, {cand[events].max()} candidates in an event frame")
    assert count.max() > 256 and cand[events].max() > 2048
