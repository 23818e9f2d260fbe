"""Busy spectrum through the device tracker: more than 256 live signals and event frames with more than 2048 start-level
candidates, the two caps of k_track's shared-memory tables. Such pushes run in k_track_wide; they must equal the host tracker
(tracker.h) bit for bit.

Each scene is generated from a seed: white complex noise, band-limited complex noise blocks several MHz wide switched on and
off, dozens of narrow carriers, and a start level low enough that noise peaks also start signals. Each case pushes the same IQ,
split into the same pushes, through four bands with one config:
  A  the dense path (K2's rows, fed to tests/k2_restate.py);
  B  the twin: every push host-tracked with per-frame lists;
  C  the device tracker K4, mailbox only (synchronous host IQ, or asynchronous device IQ);
  D  pushes alternating between host-tracked and device-tracked, so that the map crosses between host and device with more
     than 256 signals live.
Without tolerance: B's per-frame lists equal the host tracker run on the restated rows; after every push C and D equal B in
the complete transmission list, the signal map, n_transmissions_total and the result's embedded list. Every case shows from B
and the restated rows that its scene passes both caps, and from C's profile that k_track_wide ran."""
import ctypes as C
from dataclasses import dataclass
from typing import Optional, Sequence, Tuple

import numpy as np
import pytest

import k2_restate as k2
from conftest import load_b2s

b2s = load_b2s()
pytestmark = pytest.mark.gpu

MAX_SIGNALS, MAX_CAND = 256, 2048  # k_track's caps (csrc/track.cuh)


@dataclass
class Case:
    name: str
    n: int
    fs: int
    frames: int
    splits: Sequence[int]
    blocks: Sequence[Tuple[float, float, int, int]]  # (lo Hz, hi Hz offset from the centre, first frame, end frame)
    n_carriers: int = 40
    reset_at: Optional[int] = None  # index of the push before which every band is reset
    on_device_async: bool = False
    learn: int = 20
    start: float = 4.0  # low enough for noise peaks to start signals
    stop: float = 2.0
    block_snr_db: float = 22.0

    def config(self):
        cfg = b2s.make_config(self.n, self.fs, learn_frames=self.learn, recording_bandwidth_hz=32_000, min_time_ms=12, timeout_ms=25, start_level=self.start,
                              stop_level=self.stop, max_frames_per_push=max(self.splits), detect_capacity=self.n)
        cfg.spectrogram_interval_ms = 50
        return cfg

    def pushes(self):
        k, i = 0, 0
        while k < self.frames:
            m = min(self.splits[i % len(self.splits)], self.frames - k)
            yield i, k, m
            i += 1
            k += m


def busy_iq(case: Case, seed: int) -> np.ndarray:
    """CS8 IQ, [frames][N] complex samples interleaved. The noise has sigma 8 per component; a block has `block_snr_db` more power
    per bin than the noise, with a random complex amplitude in every bin and frame; a carrier has about 30 dB more."""
    n, rng = case.n, np.random.default_rng(seed)
    sigma = 8.0
    bins_per_hz = n / case.fs
    blocks = [(int(n // 2 + lo * bins_per_hz), int(n // 2 + hi * bins_per_hz), a, b) for lo, hi, a, b in case.blocks]
    amp = sigma * np.sqrt(n * 10 ** (case.block_snr_db / 10))
    carriers = [(int(rng.integers(0, n)), int(rng.integers(case.learn, case.frames)), int(rng.integers(3, 40))) for _ in range(case.n_carriers)]
    tone = sigma * np.sqrt(2 * 1000 / n)
    t = np.arange(n)
    out = np.empty((case.frames, n, 2), np.int8)
    for f in range(case.frames):
        x = rng.normal(0, sigma, n) + 1j * rng.normal(0, sigma, n)
        spec = np.zeros(n, np.complex128)
        for lo, hi, a, b in blocks:
            if a <= f < b:
                spec[lo:hi] += amp * (rng.normal(0, 1, hi - lo) + 1j * rng.normal(0, 1, hi - lo)) / np.sqrt(2)
        if spec.any():
            x += np.fft.ifft(np.fft.ifftshift(spec))
        for b_, a, d in carriers:
            if a <= f < a + d:
                x += tone * np.exp(2j * np.pi * ((b_ - n // 2) % n) * t / n)
        out[f, :, 0] = np.clip(np.rint(x.real), -127, 127)
        out[f, :, 1] = np.clip(np.rint(x.imag), -127, 127)
    return out.reshape(-1)


CASES = [
    # k_track<14>: N = 16384 at 20 MS/s (1221 Hz bins, group 27 bins). Two 5 MHz blocks overlap in time; a third comes later.
    # Uneven pushes and a reset in the middle; the map goes below -> above -> below the caps as the blocks time out.
    Case("n16384_sync", 16384, 20_000_000, 260, splits=(37, 64, 5, 100, 1, 53),
         blocks=((-9.5e6, -3.0e6, 40, 120), (-1.0e6, 5.5e6, 70, 150), (2.0e6, 8.0e6, 190, 240)), reset_at=4),
    Case("n16384_async_device_iq", 16384, 20_000_000, 220, splits=(64, 31, 97, 28), blocks=((-8.0e6, -2.0e6, 35, 130), (0.5e6, 7.0e6, 60, 170)),
         on_device_async=True),
    # k_track<12>: N = 1048576 at 200 MS/s (191 Hz bins, group 168 bins), at most 1024 frames per push
    Case("n1048576", 1048576, 200_000_000, 120, splits=(30, 17, 40, 33), blocks=((-60.0e6, -52.0e6, 28, 65), (10.0e6, 18.0e6, 35, 75)), learn=16),
]


def _same(a, b):
    return np.asarray(a).dtype == np.asarray(b).dtype and np.asarray(a).shape == np.asarray(b).shape and np.asarray(a).tobytes() == np.asarray(b).tobytes()


def _push_counted(band, iq, m, t0):
    """A host-tracked push that also returns every frame's total list length (frame_tx_count)."""
    res = b2s.Result()
    cnt = np.zeros(m, np.int32)
    tx = (b2s.Transmission * (m * b2s.MAX_TX))()
    res.frame_tx_count = cnt.ctypes.data_as(C.POINTER(C.c_int32))
    res.frame_tx = C.cast(tx, C.POINTER(b2s.Transmission))
    band.push_raw(iq.ctypes.data, m, t0, 1.0, res)
    lists = [[(tx[f * b2s.MAX_TX + s].shift_hz, tx[f * b2s.MAX_TX + s].flush, tx[f * b2s.MAX_TX + s].key, tx[f * b2s.MAX_TX + s].power)
              for s in range(min(int(cnt[f]), b2s.MAX_TX))] for f in range(m)]
    return res, cnt, lists


def _mailbox(res):
    return [(t.shift_hz, t.flush, t.key, t.power) for t in res.transmissions[: res.n_transmissions]]


def _candidates(cfg, box, start_ok):
    """Start-level candidates per frame (every bin of the band is in range here)."""
    return np.where(start_ok[:, None], box >= np.float32(cfg.start_level), False).sum(axis=1)


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_busy_spectrum_device_tracker_equals_the_host_tracker(engine, case):
    n = case.n
    cfg = case.config()
    iq = busy_iq(case, seed=9000 + n % 997 + len(case.name))
    band_a, band_b, band_d = b2s.Band(engine, cfg), b2s.Band(engine, cfg), b2s.Band(engine, cfg)
    ccfg = b2s.BandConfig.from_buffer_copy(cfg)
    iq_dev = None
    if case.on_device_async:
        import torch

        ccfg.flags |= b2s.FLAG_ASYNC | b2s.FLAG_IQ_ON_DEVICE
        iq_dev = torch.from_numpy(iq).cuda()
    band_c = b2s.Band(engine, ccfg)
    band_c.set_profiling(True)
    host, rest = b2s.HostTransmission(cfg), k2.K2Restatement(cfg)
    max_live, max_event_cand, pushes_c, prev_cnt = 0, 0, 0, None
    above = below_after_above = False
    for i, k, m in case.pushes():
        if i == case.reset_at:
            for x in (band_a, band_b, band_c, band_d, host, rest):
                x.reset()
            prev_cnt, above = None, False
        t0, part = 500 + k, iq[k * 2 * n : (k + m) * 2 * n]
        where = (case.name, i, k, m)
        a = band_a.push(part, m, t0, 1.0, dense=("psd_db", "noise_sub_db", "avg_db", "box_db"))
        b, cnt, b_lists = _push_counted(band_b, part, m, t0)
        if iq_dev is not None:
            band_c.push_raw(iq_dev.data_ptr() + k * 2 * n, m, t0, 1.0)
            c = band_c.sync()
        else:
            c = band_c.push_raw(part.ctypes.data, m, t0, 1.0)
        pushes_c += 1
        if i % 2 == 0:
            band_d.push(part, m, t0, 1.0, per_frame=True)
            d = band_d.sync()
        else:
            d = band_d.push_raw(part.ctypes.data, m, t0, 1.0)
        # 1. the twin against the host tracker on the restated rows
        r = rest.push(a.psd_db, t0, 1.0)
        assert _same(a.box_db, r.box) and _same(a.noise_sub_db, r.q), where
        lists = host.push(r.box, r.q, t0, 1.0)
        for f in range(m):
            assert b_lists[f] == lists[f], where + (f,)
        # 2. the device-tracked bands against the twin, complete
        want_tx = band_b.get_transmissions(cap=n)
        want_sig = band_b.get_signals(cap=n)
        assert len(want_tx) == int(cnt[-1]) == len(want_sig[0]), where
        for name, band, res in (("C", band_c, c), ("D", band_d, d)):
            assert band.get_transmissions(cap=n) == want_tx, where + (name,)
            for x, y in zip(band.get_signals(cap=n), want_sig):
                assert _same(x, y), where + (name, "signals")
            assert res.n_transmissions_total == len(want_tx) and _mailbox(res) == want_tx[: b2s.MAX_TX], where + (name,)
        # 3. the caps the scene passes, counted from the twin and the restated rows
        for v in cnt:
            above = above or v > MAX_SIGNALS
            below_after_above = below_after_above or (above and v <= MAX_SIGNALS)
        max_live = max(max_live, int(cnt.max()))
        cand = _candidates(cfg, r.box, ~np.all(r.avg == k2.NO_DATA, axis=1))
        before = np.concatenate([[prev_cnt if prev_cnt is not None else 0], cnt[:-1]])
        events = cnt != before  # a frame whose map changed replayed its candidates
        if events.any():
            max_event_cand = max(max_event_cand, int(cand[events].max()))
        prev_cnt = int(cnt[-1])
    p = band_c.get_profile()
    print(f"\n{case.name}: at most {max_live} live signals, {max_event_cand} candidates in an event frame; "
          f"K4 {p.track_launches} launches for {pushes_c} pushes, {p.track_events} events, {p.track_best_index} getBestIndex calls")
    assert max_live > MAX_SIGNALS and max_event_cand > MAX_CAND
    assert below_after_above, "the map never fell back below the cap"
    assert p.track_launches > pushes_c, "k_track_wide never ran"
    for x in (band_a, band_b, band_c, band_d, host):
        x.close()
