"""Overlapping sub-frames (B2S_FLAG_SUBFRAME_OVERLAP) restated on the CPU oracle, and the edge-burst scene they exist for.

A frame k of stride `stride` has m = stride / h sub-frames (h = N / 2); sub-frame j is the N samples starting at k * stride - h + j * h
(include/b2s.h). oracle_rows_overlap runs the oracle's PSD (float64 FFT rounded to fp32) on each of them and folds the linear rows
with subframe_lib.reduce_lin, the fp32 fold the device defines. A frame without a lead-in folds sub-frames 1 ... m - 1.
"""
from __future__ import annotations

import numpy as np

import oracle_lib as ol
import subframe_lib as sl

MEAN, MAX = sl.MEAN, sl.MAX


def subframe_starts(n, stride, k):
    """The first sample of each sub-frame of frame k (sample 0 = frame 0's first)."""
    h = n // 2
    return [k * stride - h + j * h for j in range(stride // h)]


def central_half(n, start):
    """The samples [lo, hi) of a sub-frame's central half."""
    return start + n // 4, start + 3 * n // 4


def overlap_config_ok(flags, n, stride, b2s):
    """include/b2s.h's rule for B2S_FLAG_SUBFRAME_OVERLAP: exactly one of MEAN / MAX, a stride >= N and a multiple of N / 2."""
    one = bool(flags & b2s.FLAG_SUBFRAME_MEAN) != bool(flags & b2s.FLAG_SUBFRAME_MAX)
    return one and stride >= n and stride % (n // 2) == 0


# (name, flags besides the overlap bit, stride) at N = sl.N
REFUSED = [
    ("no_reduction", 0, 5 * sl.N),
    ("both_reductions", 0x400 | 0x800, 5 * sl.N),
    ("stride_not_multiple_of_half", 0x400, 3 * sl.N + 1),
    ("stride_off_by_quarter", 0x800, 2 * sl.N + sl.N // 4),
]
ACCEPTED = [("mean_m2", 0x400, sl.N), ("max_m3", 0x800, 3 * sl.N // 2), ("mean_m10", 0x400, 5 * sl.N)]


def frame_row(cfg, iq, origin, k, mode, lead=True):
    """Frame k's folded (psd_db, power_lin); `iq` is a flat int8 / float32 stream whose sample `origin` is frame 0's first.
    Sub-frame 0 is dropped when lead is False."""
    n, stride = cfg.fft_size, cfg.frame_stride_samples
    starts = subframe_starts(n, stride, k)
    if not lead:
        starts = starts[1:]
    lin = []
    for s in starts:
        a = origin + s
        assert a >= 0, "sub-frame before the stream"
        lin.append(ol.oracle_psd_frame(cfg, iq[2 * a : 2 * (a + n)], want_linear=True)[1])
    p = sl.reduce_lin(lin, mode)
    return (np.float32(10.0) * np.log10(p)).astype(np.float32), p


def oracle_rows_overlap(cfg, iq, frames, mode, origin=0, no_lead=(0,), want_linear=False):
    """dB (and linear) rows of frames 0 ... frames - 1 of the stream; the frames in `no_lead` have no lead-in."""
    n = cfg.fft_size
    db, lin = np.empty((frames, n), np.float32), np.empty((frames, n), np.float32)
    for k in range(frames):
        db[k], lin[k] = frame_row(cfg, iq, origin, k, mode, lead=k not in no_lead)
    return (db, lin) if want_linear else db


# ---- the edge-burst scene -------------------------------------------------------------------------------------------------------------
# subframe_lib's band (N = 4096 at 2.048 MS/s, stride 5 N, r = 5 back to back, m = 10 overlapping). After LEARN, every stride carries
# two tone bursts of N / 16 samples: one centred on the back-to-back boundary between sub-frames 2 and 3, one centred on the frame
# boundary at the stride's start. Both sit where back-to-back Hamming windows taper to 0.08.
BURST_LEN = sl.N // 16
BURST_BIN = 0.2 * sl.N / 2 + 0.1
BURST_HZ = BURST_BIN * sl.FS / sl.N
EDGE_AMP = 40.0
EDGE_CENTRES = (0, 3 * sl.N)  # sample offsets inside a stride


def edge_burst_iq(amplitude=EDGE_AMP, *, frames=sl.FRAMES, seed=21, sigma=8.0):
    stride = sl.R * sl.N
    total = frames * stride
    rng = np.random.default_rng(seed)
    z = (rng.standard_normal(total) + 1j * rng.standard_normal(total)) * sigma
    t = np.arange(total, dtype=np.float64)
    on = np.zeros(total, bool)
    for f in range(sl.LEARN, frames):
        for c in EDGE_CENTRES:
            lo = f * stride + c - BURST_LEN // 2
            on[max(lo, 0) : lo + BURST_LEN] = True
    z += np.where(on, amplitude * np.exp(2j * np.pi * BURST_BIN / sl.N * t), 0)
    q = np.stack([z.real, z.imag], axis=-1).reshape(-1)
    return np.clip(np.rint(q), -128, 127).astype(np.int8)


def config(b2s, mode, overlap, **kw):
    flags = kw.pop("flags", 0) | (b2s.FLAG_SUBFRAME_OVERLAP if overlap else 0)
    return sl.config(b2s, mode, flags=flags, **kw)


def oracle_rows(b2s, iq, mode, overlap, frames=sl.FRAMES, **kw):
    cfg = config(b2s, mode, overlap, **kw)
    return cfg, (oracle_rows_overlap(cfg, iq, frames, mode) if overlap else sl.oracle_rows(cfg, iq, frames, mode))


def chain(cfg, rows, frames=sl.FRAMES):
    """The oracle chain fed `rows`: (its result, the chain)."""
    orc = ol.OracleChain(cfg)
    return orc.push(rows, frames, 0, sl.R * sl.N * 1000.0 / sl.FS, dense=(), psd_rows=True), orc
