"""Spectrum occupancy (b2s_band_set_occupancy / b2s_band_get_occupancy) on the GPU, with no tolerance anywhere.

The reference for every count is a twin band fed the same IQ in the same pushes that returns the dense rows: above_start / above_stop
are (box_db >= level) summed over the frames past noise learning, max_db is the column maximum of psd_db over all frames (test_k2_exact.py
pins both rows bit for bit). Cases: N = 2048 (k_spectrum), 16384 and 131072 (split mode, S = 8), B2S_FLAG_SUBFRAME_MAX, synchronous
and asynchronous, host and device IQ, several pushes against one push; two hopping centres with noise learning on the frame clock;
reset and toggling; busy spectrum with a full and an overflowing detection capacity; and the band's own results unchanged.
"""
import math
from dataclasses import dataclass, field
from typing import Sequence

import numpy as np
import pytest

from conftest import load_b2s
from test_busy_spectrum import Case as BusyCase, busy_iq

from test_oracle_chain import synth

b2s = load_b2s()

pytestmark = pytest.mark.gpu


def frame_time(t0, period, k):
    return t0 + math.floor(k * period + 0.5)  # host::frame_time


class Learning:
    """Which frames of a centre's pushes are noise-learning frames: b2s_band::enqueue_chunk's rule, per centre."""

    def __init__(self, cfg):
        self.cfg, self.samples, self.ready, self.start = cfg, 0, False, None

    def mask(self, t0, period, T):
        if self.ready:
            return np.zeros(T, bool)
        if self.cfg.noise_learning_ms > 0:
            times = [frame_time(t0, period, k) for k in range(T)]
            if self.start is None:
                self.start = times[0]
            m = np.ones(T, bool)
            for k, t in enumerate(times):
                if self.start + self.cfg.noise_learning_ms <= t:
                    m[k + 1:] = False
                    self.ready = True
                    break
            return m
        m = self.samples + np.arange(T) < self.cfg.learn_frames
        self.samples += int(m.sum())
        self.ready = self.samples >= self.cfg.learn_frames
        return m


class Expected:
    """One centre's occupancy restated from the twin's dense rows."""

    def __init__(self, n):
        self.above_start = np.zeros(n, np.int64)
        self.above_stop = np.zeros(n, np.int64)
        self.max_db = np.full(n, -np.inf, np.float32)
        self.frames = self.detect_frames = self.entries = 0

    def add(self, cfg, psd, box, learning, n_entries):
        keep = ~learning
        self.above_start += (box[keep] >= np.float32(cfg.start_level)).sum(axis=0)
        self.above_stop += (box[keep] >= np.float32(cfg.stop_level)).sum(axis=0)
        if len(psd):
            self.max_db = np.maximum(self.max_db, psd.max(axis=0))
        self.frames += len(psd)
        self.detect_frames += int(keep.sum())
        self.entries += n_entries


def assert_occupancy(got, exp, what, truncated=0):
    assert got.frames == exp.frames and got.detect_frames == exp.detect_frames, (what, got.frames, exp.frames, got.detect_frames, exp.detect_frames)
    assert got.truncated == truncated, (what, got.truncated)
    np.testing.assert_array_equal(got.above_start.astype(np.int64), exp.above_start, err_msg=f"{what}: above_start")
    np.testing.assert_array_equal(got.above_stop.astype(np.int64), exp.above_stop, err_msg=f"{what}: above_stop")
    assert got.max_db.tobytes() == exp.max_db.tobytes(), f"{what}: max_db"


@dataclass
class Case:
    name: str
    n: int
    frames: int
    splits: Sequence[int]
    learn: int = 30
    flags: int = 0
    decimator: int = 1
    levels: tuple = (8.0, 5.0)
    tones: Sequence[float] = field(default_factory=lambda: (0.31, -0.62, 0.055))

    def config(self, flags=0, max_frames=None):
        fs = 20_000_000 if self.n >= 8192 else 2_048_000
        cfg = b2s.make_config(self.n, fs, learn_frames=self.learn, recording_bandwidth_hz=16 * fs // self.n, min_time_ms=20, timeout_ms=30,
                              start_level=self.levels[0], stop_level=self.levels[1], max_frames_per_push=max_frames or max(self.splits),
                              detect_capacity=self.n, decimator=self.decimator, flags=self.flags | flags)
        cfg.spectrogram_interval_ms = 23
        return cfg

    def iq(self):
        n, stride, span = self.n, self.n * self.decimator, self.frames - self.learn
        tones = [synth.Tone(f * n / 2 + 0.1, amplitude=40.0, fm_dev_bins=3.0, on_frames=[(self.learn + int(0.1 * span * (i + 1)), self.learn + int(0.2 * span * (i + 3)))], phase=float(i))
                 for i, f in enumerate(self.tones)]
        iq = synth.make_iq_int8(n * self.decimator, self.frames, [synth.Tone(t.bin_offset * self.decimator, t.amplitude, t.on_frames, t.phase, t.fm_dev_bins) for t in tones],
                                seed=n + len(self.name), quiet_frames=self.learn)
        assert iq.size == 2 * stride * self.frames
        return iq

    def pushes(self):
        k, i = 0, 0
        while k < self.frames:
            m = min(self.splits[i % len(self.splits)], self.frames - k)
            yield k, m
            i += 1
            k += m


CASES = [
    Case("n2048", 2048, 300, (64, 100, 31, 105)),
    Case("n2048_stop_above_start", 2048, 300, (150, 150), levels=(5.0, 8.0)),
    Case("n16384", 16384, 260, (96, 164)),
    Case("n16384_subframe_max", 16384, 160, (70, 90), flags=b2s.FLAG_SUBFRAME_MAX, decimator=3),
    Case("n131072_split", 131072, 48, (20, 28), learn=8),
]
MODES = ("sync_host", "sync_device", "async_host", "async_device")


def period_of(cfg):
    return cfg.frame_stride_samples * 1000.0 / cfg.sample_rate_hz


class Pusher:
    """Pushes host IQ through a band, from host or device memory, synchronously or not."""

    def __init__(self, engine, cfg, mode):
        self.on_device, self.is_async = mode.endswith("device"), mode.startswith("async")
        cfg.flags |= (b2s.FLAG_IQ_ON_DEVICE if self.on_device else 0) | (b2s.FLAG_ASYNC if self.is_async else 0)
        self.cfg, self.band, self.keep = cfg, b2s.Band(engine, cfg), []

    def push(self, iq, k, m, t0):
        stride = 2 * self.cfg.frame_stride_samples
        piece = np.ascontiguousarray(iq[k * stride:(k + m) * stride])
        if self.on_device:
            import torch
            t = torch.from_numpy(piece).cuda()
            self.keep.append(t)
            torch.cuda.synchronize()
            return self.band.push_raw(t.data_ptr(), m, t0, period_of(self.cfg))
        if self.is_async:
            return self.band.push_raw(piece.ctypes.data, m, t0, period_of(self.cfg))
        return self.band.push(piece, m, t0, period_of(self.cfg))


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_counts_match_the_dense_rows(engine, case, mode):
    if case.n == 131072 and mode in ("sync_device", "async_host"):
        pytest.skip("split mode runs sync host and async device")
    iq = case.iq()
    cfg = case.config()
    period = period_of(cfg)
    twin = b2s.Band(engine, case.config())
    band = Pusher(engine, case.config(), mode)
    band.band.set_occupancy(True)
    whole = Pusher(engine, case.config(max_frames=case.frames), mode)  # the same frames in one push
    whole.band.set_occupancy(True)
    exp, learn = Expected(case.n), Learning(cfg)
    t0 = 1000
    for k, m in case.pushes():
        out = twin.push(iq[k * 2 * cfg.frame_stride_samples:(k + m) * 2 * cfg.frame_stride_samples], m, t0 + k * 7, period, dense=("psd_db", "box_db"))
        exp.add(cfg, out.psd_db, out.box_db, learn.mask(t0 + k * 7, period, m), out.n_detect_entries)
        band.push(iq, k, m, t0 + k * 7)
    # the one-push band sees one clock: its learning frames are the same only with the frame-count rule (noise_learning_ms = 0)
    whole.push(iq, 0, case.frames, t0)
    got = band.band.occupancy(cfg.center_hz)
    assert_occupancy(got, exp, case.name)
    assert_occupancy(whole.band.occupancy(cfg.center_hz), exp, case.name + " (one push)")
    assert band.band.occupancy_centers() == [cfg.center_hz]
    assert exp.detect_frames == case.frames - case.learn and exp.above_stop.sum() > 0
    if case.levels[1] <= case.levels[0]:
        assert int(got.above_stop.sum()) == exp.entries  # every entry is a bin at or above the stop level
    else:
        assert int(got.above_start.sum()) == exp.entries
    for b in (twin, band.band, whole.band):
        b.close()


def test_hopping_centres_keep_their_own_statistics(engine):
    """Two centres alternated with set_center + reset, noise learning on the frame clock: each centre counts its own frames only."""
    n, fs = 4096, 2_048_000
    centres = (100_000_000, 101_000_000)
    def config():
        cfg = b2s.make_config(n, fs, center_hz=centres[0], learn_frames=1, noise_learning_ms=40, recording_bandwidth_hz=16 * fs // n, min_time_ms=20,
                              timeout_ms=30, max_frames_per_push=128)
        return cfg
    cfg = config()
    period = period_of(cfg)
    dwell, rounds = 60, 6
    iq = synth.make_iq_int8(n, dwell * rounds, synth.standard_scene(n, dwell * rounds, 0), seed=77)
    twin, band = b2s.Band(engine, config()), b2s.Band(engine, config())
    band.set_occupancy(True)
    exp = {c: Expected(n) for c in centres}
    learn = {c: Learning(cfg) for c in centres}
    for r in range(rounds):
        c = centres[r % 2]
        lo, hi = c - fs // 2, c + fs // 2
        for b in (twin, band):
            b.set_center(c, lo, hi)
            b.reset()
        t0 = r * 1000
        piece = iq[r * dwell * 2 * n:(r + 1) * dwell * 2 * n]
        out = twin.push(piece, dwell, t0, period, dense=("psd_db", "box_db"))
        exp[c].add(cfg, out.psd_db, out.box_db, learn[c].mask(t0, period, dwell), out.n_detect_entries)
        band.push(piece, dwell, t0, period)
    assert band.occupancy_centers() == list(centres)
    for c in centres:
        assert exp[c].frames == dwell * rounds // 2 and 0 < exp[c].detect_frames < exp[c].frames
        assert_occupancy(band.occupancy(c), exp[c], f"centre {c}")
    twin.close()
    band.close()


def test_reset_and_toggling(engine):
    """reset = 1 empties the centre's statistics after they are read; turning occupancy off and on keeps them."""
    case = Case("n2048_pushes", 2048, 320, (40,))
    iq, cfg = case.iq(), case.config()
    period = period_of(cfg)
    twin, band = b2s.Band(engine, case.config()), b2s.Band(engine, case.config())
    with pytest.raises(b2s.B2SError):
        band.occupancy(cfg.center_hz)  # no statistics yet
    band.set_occupancy(True)
    learn = Learning(cfg)
    exp = Expected(cfg.fft_size)
    for i, (k, m) in enumerate(case.pushes()):
        piece = iq[k * 2 * cfg.fft_size:(k + m) * 2 * cfg.fft_size]
        out = twin.push(piece, m, k, period, dense=("psd_db", "box_db"))
        mask = learn.mask(k, period, m)
        if i == 4:
            band.set_occupancy(False)  # this push is not counted
        elif i == 5:
            band.set_occupancy(True)
        if i != 4:
            exp.add(cfg, out.psd_db, out.box_db, mask, out.n_detect_entries)
        band.push(piece, m, k, period)
        if i == 1:
            assert_occupancy(band.occupancy(cfg.center_hz, reset=True), exp, "before the reset")
            exp = Expected(cfg.fft_size)
            cleared = band.occupancy(cfg.center_hz)
            assert cleared.frames == cleared.detect_frames == 0 and not cleared.above_start.any() and not cleared.above_stop.any()
            assert np.all(cleared.max_db == -np.inf)
        if i == 4:
            kept = band.occupancy(cfg.center_hz)
            assert_occupancy(kept, exp, "while off")
            assert kept.above_stop.any()
    assert_occupancy(band.occupancy(cfg.center_hz), exp, "after the reset")
    twin.close()
    band.close()


BUSY = BusyCase("busy_n4096", 4096, 2_048_000, frames=200, splits=(100,), blocks=[(-900_000, -100_000, 30, 200), (100_000, 900_000, 60, 160)], learn=20)


@pytest.mark.parametrize("capacity", [4096, 64])
def test_busy_spectrum(engine, capacity):
    """Entries in most bins: counts match with detect_capacity = N; a small capacity overflows and the read says so."""
    iq = busy_iq(BUSY, seed=4242)
    cfg = BUSY.config()
    cfg.detect_capacity = capacity
    period = period_of(cfg)
    twin = b2s.Band(engine, BUSY.config())
    band = b2s.Band(engine, cfg)
    band.set_occupancy(True)
    exp, learn = Expected(BUSY.n), Learning(cfg)
    overflowed = 0
    for _, k, m in BUSY.pushes():
        piece = iq[k * 2 * BUSY.n:(k + m) * 2 * BUSY.n]
        out = twin.push(piece, m, k * 5, period, dense=("psd_db", "box_db"))
        exp.add(cfg, out.psd_db, out.box_db, learn.mask(k * 5, period, m), out.n_detect_entries)
        try:
            band.push(piece, m, k * 5, period)
        except b2s.B2SError as e:
            assert "detect_capacity" in str(e)
            overflowed += 1
    got = band.occupancy(cfg.center_hz)
    if capacity == BUSY.n:
        assert overflowed == 0
        assert_occupancy(got, exp, "busy")
        assert (exp.above_stop > 0).mean() > 0.5  # entries in most bins
    else:
        assert overflowed >= 1 and got.truncated == overflowed
        assert got.frames == exp.frames and got.detect_frames == exp.detect_frames
        assert np.all(got.above_stop <= exp.above_stop) and np.all(got.above_start <= exp.above_start)  # lower bounds
        assert got.above_stop.sum() < exp.above_stop.sum()
        assert got.max_db.tobytes() == exp.max_db.tobytes()  # the max-hold does not depend on the lists
    twin.close()
    band.close()


def _state(band, bank):
    s, a, r, f = band.get_averager()
    thr, samples, ready = band.get_noise()
    keys, first, last, power = band.get_signals(cap=4096)
    times, centers, rows = band.get_spectrogram(cap=1024)
    out = [s.tobytes(), a.tobytes(), r.tobytes(), f, thr.tobytes(), samples, ready, keys.tobytes(), first.tobytes(), last.tobytes(), power.tobytes(),
           times.tobytes(), centers.tobytes(), rows.tobytes(), band.get_transmissions(), band.get_events()]
    if bank is not None:
        out += [[(t, c.tobytes()) for t, c in bank.flush(ch, cap=4096)] for ch in range(bank.n_channels)]
    return out


def _summary(out):
    """A synchronous push's mailbox and entry count, from Band.push (PushOutput) or Band.push_raw (Result)."""
    if isinstance(out, b2s.Result):
        return bytes(out)
    return out.transmissions, out.n_detect_entries


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("with_bank", [False, True], ids=["alone", "bank"])
def test_no_effect_on_results(engine, mode, with_bank):
    case = Case("n16384_effect", 16384, 260, (96, 64, 100))
    iq = case.iq()
    bands, banks = [], []
    for on in (False, True):
        p = Pusher(engine, case.config(), mode)
        p.band.set_event_log(True)
        if on:
            p.band.set_occupancy(True)
        bank = None
        if with_bank:
            bank = b2s.RecorderBank(engine, p.cfg.sample_rate_hz, 32_000, 2, on_device=p.on_device, max_samples_per_push=max(case.splits) * p.cfg.frame_stride_samples)
            p.band.attach_recorder_bank(bank)
            bank.start(0, 3_000_000)
            bank.start(1, -6_200_000)
        bands.append(p)
        banks.append(bank)
    for k, m in case.pushes():
        outs = [p.push(iq, k, m, 500 + k) for p in bands]
        if not bands[0].is_async:
            assert _summary(outs[0]) == _summary(outs[1])
        else:
            r0, r1 = bands[0].band.sync(), bands[1].band.sync()
            assert bytes(r0) == bytes(r1)
        assert _state(bands[0].band, banks[0]) == _state(bands[1].band, banks[1]), f"results differ after the push at frame {k}"
    assert bands[1].band.occupancy(bands[1].cfg.center_hz).frames == case.frames
    for p, bank in zip(bands, banks):
        p.band.close()
        if bank is not None:
            bank.close()
