"""Exact float32 restatement of K2 (k_detect, csrc/detect.cuh): NoiseLearner, Averager, the engine's frequency boxcar, the
detection entries and the spectrogram, from PSD rows on. TEST INFRASTRUCTURE ONLY.

Every operation is a vectorised numpy float32 add, subtract, multiply or divide. Those are IEEE round-to-nearest with no
contraction, so they are the kernel's __fadd_rn / __fsub_rn / __fmul_rn / __fdiv_rn, and the rows below are meant to equal
the engine's bit for bit. The state is carried across pushes the way a band carries it.
"""
from __future__ import annotations

import numpy as np

NO_DATA = np.float32(-100.0)  # kNoData
BOX_SEGMENT = 16              # kBoxSegment


def frame_stamps(t0_ms: int, period_ms: float, frames: int, first: int = 0) -> np.ndarray:
    """The frame clock: now_k = t0 + floor(k * period + 0.5), in double precision (host::frame_time)."""
    k = np.arange(first, first + frames, dtype=np.float64)
    return t0_ms + np.floor(k * float(period_ms) + 0.5).astype(np.int64)


def boxcar(avg: np.ndarray, group_x: int, segment: int | None = BOX_SEGMENT) -> np.ndarray:
    """average(avg, X) in the engine's form, row by row: over the zero-extended row, aligned segments of `segment` bins; the first
    bin of a segment is w[0] + w[1] + ... + w[2H] left to right (starting from w[0] itself), the next bins slide the sum
    (s -= leaving; s += entering); each bin is divided by its clipped window count. With X = 1 the last bin is 0.0 (the
    reference never writes it). segment=None is one segment per row: the reference's serial form."""
    rows = np.atleast_2d(np.asarray(avg, dtype=np.float32))
    t, n = rows.shape
    h = group_x // 2
    seg = n if segment is None else segment
    nseg = (n + seg - 1) // seg
    z = np.zeros((t, nseg * seg + 2 * h), np.float32)  # z[:, i] holds bin i - h
    z[:, h : h + n] = rows
    starts = np.arange(nseg) * seg
    out = np.empty((t, nseg * seg), np.float32)
    s = z[:, starts].copy()
    for i in range(1, 2 * h + 1):
        s = s + z[:, starts + i]
    out[:, starts] = s
    for k in range(1, seg):
        s = s - z[:, starts + k - 1]
        s = s + z[:, starts + k + 2 * h]
        out[:, starts + k] = s
    j = np.arange(n)
    count = (np.minimum(n - 1, j + h) - np.maximum(0, j - h) + 1).astype(np.float32)
    out = out[:, :n] / count
    if h == 0:
        out[:, n - 1] = 0.0
    return out.reshape(np.shape(avg)) if np.ndim(avg) == 1 else out


class PushRows:
    """What one push produced: noise-subtracted rows q, Averager rows avg, boxcar rows box (all [T][N] float32), the
    learning-frame mask, the detection entries per frame and the spectrogram rows [(time_ms, int8 row)] completed in it."""


class K2Restatement:
    """One band's K2 state for one centre frequency: the noise threshold (kept across reset), the Averager (cleared by reset) and
    the spectrogram accumulator (kept across reset)."""

    def __init__(self, cfg, segment: int | None = BOX_SEGMENT):
        self.n, self.x, self.y = cfg.fft_size, cfg.grouping_x, cfg.grouping_y
        self.learn_frames, self.learning_ms = cfg.learn_frames, cfg.noise_learning_ms
        self.level = np.float32(min(cfg.start_level, cfg.stop_level))
        self.spec_out, self.spec_interval = cfg.spectrogram_out_size, cfg.spectrogram_interval_ms
        self.segment = segment
        # NoiseLearner (noise_learner.cpp:16: the threshold starts at -FLT_MAX)
        self.threshold = np.full(self.n, -np.finfo(np.float32).max, np.float32)
        self.samples, self.ready = 0, False
        self.started, self.start_ms = False, 0
        # spectrogram (m_counter defined as 0; the clock starts at the first frame the centre sees)
        self.spec_sum, self.spec_counter, self.spec_last = None, 0, 0
        self.reset()

    def reset(self):
        """Transmission::resetBuffers as the engine does it: the Averager restarts from zeros; noise and spectrogram stay."""
        self.sum = np.zeros(self.n, np.float32)
        self.ring = np.zeros((self.y, self.n), np.float32)  # oldest -> newest
        self.frames = 0
        self.avg_last = np.full(self.n, NO_DATA, np.float32)

    def averager(self):
        """(m_sum, m_average after the last frame, ring oldest -> newest, m_frames): b2s_band_get_averager's order."""
        return self.sum.copy(), self.avg_last.copy(), self.ring.copy(), self.frames

    def noise(self):
        return self.threshold.copy(), self.samples, self.ready

    def _learning_frames(self, stamps: np.ndarray) -> np.ndarray:
        t = len(stamps)
        if self.ready:
            return np.zeros(t, bool)
        if self.learning_ms > 0:
            # every frame up to and including the first one stamped at or after start + noise_learning_ms learns
            if not self.started:
                self.started, self.start_ms = True, int(stamps[0])
            done = np.nonzero(self.start_ms + self.learning_ms <= stamps)[0]
            last = int(done[0]) if len(done) else -1
            learning = np.arange(t) < (last + 1 if last >= 0 else t)
            self.samples += int(learning.sum())
            self.ready = last >= 0
            return learning
        learning = self.samples + np.arange(t) < self.learn_frames
        self.samples += int(learning.sum())
        self.ready = self.samples >= self.learn_frames
        return learning

    def push(self, psd: np.ndarray, t0_ms: int, period_ms: float) -> PushRows:
        psd = np.ascontiguousarray(psd, dtype=np.float32)
        t, n, y = psd.shape[0], self.n, self.y
        stamps = frame_stamps(t0_ms, period_ms, t)
        r = PushRows()
        r.learning = self._learning_frames(stamps)
        # NoiseLearner: thr = max(thr, p) over the learning frames (a prefix of the push), then p - thr
        if r.learning.any():
            self.threshold = np.maximum(self.threshold, psd[r.learning].max(axis=0))
        r.q = np.where(r.learning[:, None], NO_DATA, psd - self.threshold).astype(np.float32)
        # Averager: m_sum = (m_sum - oldest) + newest, two roundings; m_average = m_sum / Y once Y frames were seen
        r.avg = np.empty_like(r.q)
        ring = list(self.ring)
        for k in range(t):
            self.sum = self.sum - ring.pop(0)
            self.sum = self.sum + r.q[k]
            ring.append(r.q[k])
            self.frames = min(self.frames + 1, y)
            r.avg[k] = self.sum / np.float32(y) if self.frames >= y else NO_DATA
        self.ring = np.stack(ring)
        if t:
            self.avg_last = r.avg[-1].copy()
        r.box = boxcar(r.avg, self.x, self.segment)
        r.entries = (r.box >= self.level).sum(axis=1)
        r.spectrogram = self._spectrogram(psd, stamps)
        return r

    def _spectrogram(self, psd, stamps):
        m = self.spec_out
        if m <= 0:
            return []
        d = self.n // m
        if self.spec_sum is None:
            self.spec_sum, self.spec_counter, self.spec_last = np.zeros(m, np.float32), 0, int(stamps[0])
        inv_d = np.float32(1.0 / d)
        sent = []
        for k in range(psd.shape[0]):
            if d == 1:
                v = psd[k]
            else:
                v = psd[k, 0::d].copy()  # mean of d adjacent raw bins: summed from bin 0, then multiplied by 1/d
                for i in range(1, d):
                    v = v + psd[k, i::d]
                v = v * inv_d
            self.spec_sum = self.spec_sum + v
            self.spec_counter += 1
            now = int(stamps[k])
            if self.spec_last + self.spec_interval < now:  # Spectrogram::send: float -> int truncation -> int8
                row = (self.spec_sum / np.float32(self.spec_counter)).astype(np.int32).astype(np.int8)
                sent.append((now, row))
                self.spec_sum = np.zeros(m, np.float32)
                self.spec_counter, self.spec_last = 0, now
        return sent

