"""Overlapping sub-frames without a GPU: the flag's value, the configs the flag accepts, the sub-frame layout, the oracle's fold,
and what the edge-burst and weak-carrier scenes show in the oracle chain (test_subframe_overlap.py runs them on the band)."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import oracle_lib as ol
import subframe_lib as sl
import subframe_overlap_lib as so
from conftest import ROOT, load_b2s

b2s = load_b2s()


def test_flag_value_matches_header():
    text = open(os.path.join(ROOT, "include", "b2s.h")).read()
    m = re.search(r"#define B2S_FLAG_SUBFRAME_OVERLAP\s+(0x[0-9a-fA-F]+)", text)
    assert m and int(m.group(1), 16) == b2s.FLAG_SUBFRAME_OVERLAP == 0x1000
    others = (b2s.FLAG_IQ_ON_DEVICE, b2s.FLAG_ASYNC, b2s.FLAG_SUBFRAME_MEAN, b2s.FLAG_SUBFRAME_MAX)
    assert all(b2s.FLAG_SUBFRAME_OVERLAP & f == 0 for f in others)


@pytest.mark.parametrize("case", so.REFUSED + so.ACCEPTED, ids=[c[0] for c in so.REFUSED + so.ACCEPTED])
def test_validity_rule(case):
    """The rule include/b2s.h states, on the cases test_subframe_overlap.py feeds to b2s_band_create and b2s_psd (which need a
    device before they look at the config)."""
    name, flags, stride = case
    ok = case in so.ACCEPTED
    assert so.overlap_config_ok(flags | b2s.FLAG_SUBFRAME_OVERLAP, sl.N, stride, b2s) == ok, name


def test_default_strides_qualify():
    """b2s_default_config's strides are N x decimator factor: multiples of N / 2."""
    for fs in (2_048_000, 2_400_000, 10_000_000, 20_000_000, 40_000_000, 61_440_000):
        cfg = b2s.BandConfig()
        b2s.lib().b2s_default_config(C.byref(cfg), fs, 100_000_000, 32000)
        assert cfg.frame_stride_samples >= cfg.fft_size and cfg.frame_stride_samples % (cfg.fft_size // 2) == 0


@pytest.mark.parametrize("m", [2, 3, 6])
def test_central_halves_tile_the_stream(m):
    """Sub-frame 0 straddles the previous frame, sub-frame m-1 ends with the stride, and the central halves of consecutive frames
    tile the stream: frame k owns [k * stride - N / 4, (k + 1) * stride - N / 4)."""
    n = 1024
    h, stride = n // 2, m * n // 2
    covered = []
    for k in range(4):
        starts = so.subframe_starts(n, stride, k)
        assert len(starts) == m
        assert starts[0] == k * stride - h and starts[-1] + n == (k + 1) * stride
        halves = [so.central_half(n, s) for s in starts]
        assert halves[0][0] == k * stride - n // 4 and halves[-1][1] == (k + 1) * stride - n // 4
        covered += halves
    for (lo0, hi0), (lo1, _) in zip(covered, covered[1:]):
        assert hi0 == lo1  # no gap, no overlap
    # every sample's window weight in the sub-frame whose central half holds it is at least 0.54
    w = np.hamming(n)
    assert w[n // 4 : 3 * n // 4].min() >= 0.54


def test_oracle_fold():
    """The frame row folds the oracle's float64 PSD of each sub-frame in ascending j; without a lead-in, sub-frames 1 ... m-1."""
    n, m = 1024, 3
    cfg = b2s.make_config(n, 2_048_000, flags=b2s.FLAG_SUBFRAME_MEAN | b2s.FLAG_SUBFRAME_OVERLAP)
    cfg.frame_stride_samples = m * n // 2
    rng = np.random.default_rng(8)
    origin = n // 2
    iq = np.clip(np.rint(rng.standard_normal(2 * (origin + 3 * cfg.frame_stride_samples)) * 20), -128, 127).astype(np.int8)
    for mode in (so.MEAN, so.MAX):
        for lead in (True, False):
            db, lin = so.frame_row(cfg, iq, origin, 1, mode, lead)
            starts = so.subframe_starts(n, cfg.frame_stride_samples, 1)[0 if lead else 1 :]
            rows = [ol.oracle_psd_frame(cfg, iq[2 * (origin + s) : 2 * (origin + s + n)], want_linear=True)[1] for s in starts]
            acc = rows[0]
            for p in rows[1:]:
                acc = np.maximum(acc, p) if mode == so.MAX else np.add(acc, p, dtype=np.float32)
            if mode == so.MEAN:
                acc = np.divide(acc, np.float32(len(rows)), dtype=np.float32)
            assert np.array_equal(lin, acc), (mode, lead)
    # frame 0 of a stream has no lead-in: the default restatement drops its sub-frame 0
    rows = so.oracle_rows_overlap(cfg, iq[2 * origin :], 2, so.MAX)
    assert np.array_equal(rows[0], so.frame_row(cfg, iq, origin, 0, so.MAX, lead=False)[0])


def burst_bin():
    return int(round(so.BURST_BIN + sl.N / 2))  # fftshifted


def test_edge_burst_scene_oracle():
    """Bursts of N / 16 samples on a sub-frame boundary and on a frame boundary: MAX without overlap starts nothing, MAX with
    overlap starts a transmission at the burst, and its folded row there is at least 15 dB higher."""
    iq = so.edge_burst_iq()
    cfg0, rows0 = so.oracle_rows(b2s, iq, so.MAX, False)
    cfg1, rows1 = so.oracle_rows(b2s, iq, so.MAX, True)
    res0, _ = so.chain(cfg0, rows0)
    res1, _ = so.chain(cfg1, rows1)
    assert not sl.reported(res0.frame_tx, so.BURST_HZ)
    assert sl.reported(res1.frame_tx, so.BURST_HZ)
    b = burst_bin()
    gain = np.median(rows1[sl.LEARN :, b]) - np.median(rows0[sl.LEARN :, b])
    print(f"edge burst: folded row at the burst bin {gain:.1f} dB higher with overlap")
    assert gain >= 15.0


def start_amplitude(overlap, lo=3.0, hi=7.0, step=0.25):
    """The smallest amplitude (on a `step` grid) at which MEAN starts the weak carrier, by bisection."""
    def starts(amp):
        iq = sl.scene_iq(sl.WEAK_ON, amp)
        cfg, rows = so.oracle_rows(b2s, iq, so.MEAN, overlap)
        return sl.reported(so.chain(cfg, rows)[0].frame_tx)

    assert starts(hi) and not starts(lo)
    while hi - lo > step:
        mid = round((lo + hi) / 2 / step) * step
        if mid in (lo, hi):
            break
        lo, hi = (lo, mid) if starts(mid) else (mid, hi)
    return hi


def test_weak_carrier_scene_oracle():
    """MEAN with and without overlap on subframe_lib's weak-carrier scene: the learned noise and the start amplitude, reported."""
    noise = {}
    iq = sl.scene_iq(sl.WEAK_ON, 0.0)
    for overlap in (False, True):
        cfg, rows = so.oracle_rows(b2s, iq, so.MEAN, overlap)
        noise[overlap] = so.chain(cfg, rows)[1].get_noise()[0]
    shift_mean = float(np.mean(noise[True]) - np.mean(noise[False]))
    shift_max = float(np.max(noise[True]) - np.max(noise[False]))
    amp = {ov: start_amplitude(ov) for ov in (False, True)}
    print(f"weak carrier, MEAN: learned noise shift with overlap {shift_mean:+.2f} dB (mean over bins), {shift_max:+.2f} dB (largest bin); "
          f"start amplitude {amp[False]:.2f} without, {amp[True]:.2f} with overlap ({20 * np.log10(amp[True] / amp[False]):+.2f} dB)")
    assert np.all(np.isfinite(noise[True])) and noise[True].shape == (sl.N,)
