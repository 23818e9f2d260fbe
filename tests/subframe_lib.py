"""Sub-frame PSD rows (B2S_FLAG_SUBFRAME_MEAN / _MAX) restated on the CPU oracle, and the scenes that show what they detect.

orc_psd_frame_subframes runs the oracle's PSD (float64 FFT rounded to fp32, oracle/scan_oracle.cpp) on each of a frame's r
sub-frames and reduces the linear rows in the order and with the fp32 operations include/b2s.h defines: MEAN adds the sub-frames
in order and divides by r once, MAX takes the per-bin maximum. numpy's float32 add, divide and maximum round like the device's
__fadd_rn, __fdiv_rn and fmaxf.
"""
from __future__ import annotations

import numpy as np

import oracle_lib as ol

MEAN, MAX = "mean", "max"


def reduce_lin(rows, mode):
    """rows: the r linear sub-frame rows [r][N] (float32) -> the frame's linear row."""
    rows = np.asarray(rows, np.float32)
    acc = rows[0].copy()
    for p in rows[1:]:
        acc = np.maximum(acc, p) if mode == MAX else np.add(acc, p, dtype=np.float32)
    if mode == MEAN:
        acc = np.divide(acc, np.float32(len(rows)), dtype=np.float32)
    return acc


def orc_psd_frame_subframes(cfg, window, iq_frame, r, mode):
    """One frame's reduced (psd_db, power_lin). iq_frame holds at least r * N samples (int8 pairs or float32 pairs per cfg)."""
    n = cfg.fft_size
    per = 2 * n  # scalars per sub-frame
    sub = [ol.oracle_psd_frame(cfg, iq_frame[j * per : (j + 1) * per], window=window, want_linear=True) for j in range(r)]
    if r == 1:  # the reduction of one row is that row: the oracle's own dB values
        return sub[0]
    p = reduce_lin([lin for _, lin in sub], mode)
    # 10 log10 in fp32 like psdDb; numpy's float32 log10 may differ from the C library's by an ulp (inside the parity criterion)
    return (np.float32(10.0) * np.log10(p)).astype(np.float32), p


def oracle_rows(cfg, iq, n_frames, mode=None):
    """dB rows of n_frames frames of `iq` (a flat int8 / float32 stream, frame k at k * frame_stride_samples) as the band computes
    them with mode (None: no sub-frames, the first N samples of each stride)."""
    n, stride = cfg.fft_size, cfg.frame_stride_samples
    r = stride // n if mode else 1
    out = np.empty((n_frames, n), np.float32)
    for k in range(n_frames):
        f = iq[2 * k * stride : 2 * k * stride + 2 * r * n]
        if mode:
            out[k] = orc_psd_frame_subframes(cfg, None, f, r, mode)[0]
        else:
            out[k] = ol.oracle_psd_frame(cfg, f)
    return out


# ---- scenes ----------------------------------------------------------------------------------------------------------------------
# N = 4096 at 2.048 MS/s with a stride of 5 N (r = 5): a frame every 10 ms. The first LEARN frames are noise only (noise learning);
# then an FM carrier (spread over ~12 bins like a voice channel, so that it moves the boxcar of dB values) is present in the
# sub-frames a scene chooses.
N, FS, R, LEARN, FRAMES = 4096, 2_048_000, 5, 40, 140
CARRIER_BIN = 0.3 * N / 2 + 0.1
CARRIER_HZ = CARRIER_BIN * FS / N


def config(b2s, mode=None, **kw):
    flags = {None: 0, MEAN: b2s.FLAG_SUBFRAME_MEAN, MAX: b2s.FLAG_SUBFRAME_MAX}[mode] | kw.pop("flags", 0)
    kw.setdefault("learn_frames", LEARN)
    kw.setdefault("spectrogram_out_size", 0)
    return b2s.make_config(N, FS, decimator=R, recording_bandwidth_hz=16 * FS // N, min_time_ms=50, timeout_ms=100, flags=flags, **kw)


def scene_iq(subframes_on, amplitude, *, frames=FRAMES, seed=1, sigma=8.0):
    """int8 IQ of `frames` strides: noise everywhere, the carrier in sub-frames `subframes_on` of every stride after LEARN."""
    stride = R * N
    rng = np.random.default_rng(seed)
    z = (rng.standard_normal((frames, stride)) + 1j * rng.standard_normal((frames, stride))) * sigma
    nn = np.arange(frames * stride, dtype=np.float64).reshape(frames, stride)
    beta = 6.0 / (3.3 / N) / N  # 6-bin deviation at 3.3 cycles per N samples
    ph = 2 * np.pi * (CARRIER_BIN / N) * nn + beta * np.sin(2 * np.pi * 3.3 * nn / N)
    on = np.zeros((frames, stride), bool)
    for j in subframes_on:
        on[LEARN:, j * N : (j + 1) * N] = True
    z += np.where(on, amplitude * np.exp(1j * ph), 0)
    q = np.empty((frames, stride, 2))
    q[..., 0], q[..., 1] = z.real, z.imag
    return np.clip(np.rint(q), -128, 127).astype(np.int8).reshape(-1)


def reported(frame_tx, hz=CARRIER_HZ, tol=FS / N * 16):
    """Whether any frame's list holds a transmission within `tol` of `hz`."""
    return any(abs(f - hz) <= tol for fr in frame_tx for f, *_ in fr)


def oracle_outcome(b2s, iq, mode, frames=FRAMES):
    """The oracle chain fed the oracle's rows for `mode`: whether it reports the carrier."""
    cfg = config(b2s, mode)
    rows = oracle_rows(cfg, iq, frames, mode)
    res = ol.OracleChain(cfg).push(rows, frames, 0, R * N * 1000.0 / FS, dense=(), psd_rows=True)
    return reported(res.frame_tx)


GAP_ON = range(1, R)          # silent in sub-frame 0 of every stride: a band without sub-frames never sees it
BURST_ON = (2,)               # one sub-frame per stride
GAP_AMP, BURST_AMP = 60.0, 60.0
WEAK_ON = range(R)            # continuous
WEAK_AMP = 6.0
