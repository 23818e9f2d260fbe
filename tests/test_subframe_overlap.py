"""Overlapping sub-frames on the GPU (B2S_FLAG_SUBFRAME_OVERLAP, include/b2s.h): K1 folds each frame's m = stride / (N / 2)
half-overlapping sub-frames, frame 0 of a push takes its first from the band's lead-in, and the results do not depend on how the
stream is cut.

  * K1 per bin against subframe_overlap_lib's float64 restatement, with the criterion of test_subframe_psd.py: b2s_psd and a band's
    dense rows at N = 256, 2048, 4096, 16384 and 32768 (split mode), m = 2, 3, 6, MEAN and MAX, CS8 aligned and unaligned, CF32,
    host and device input.
  * the lead-in: the first push and the push after a centre change fold m - 1 sub-frames in frame 0; b2s_band_reset keeps it.
  * continuity, with no tolerance: one push equals uneven pushes in every result, sync and async, host and device IQ, pieces.
  * the chain against the oracle fed the band's own rows, and the edge-burst scene end to end.
  * an attached bank, snapshots and refusals.
"""
import ctypes as C
import struct

import numpy as np
import pytest

import oracle_lib as ol
import subframe_lib as sl
import subframe_overlap_lib as so
from conftest import load_b2s

b2s = load_b2s()
pytestmark = pytest.mark.gpu

MODES = (so.MEAN, so.MAX)
E_INVALID = -1
RED = {so.MEAN: 0x400, so.MAX: 0x800}
OVERLAP = 0x1000
PERIOD = sl.R * sl.N * 1000.0 / sl.FS


def noise_tones(n, samples, seed, fmt=0):
    """`samples` IQ samples of noise, two tones and a burst, as int8 or float32 pairs."""
    rng = np.random.default_rng(seed)
    k = np.arange(samples, dtype=np.float64)
    z = (rng.standard_normal(samples) + 1j * rng.standard_normal(samples)) * 8.0
    for b, a in ((0.31 * n / 2 + 0.1, 40.0), (-0.12 * n / 2 + 0.1, 25.0)):
        z += a * np.exp(2j * np.pi * b / n * k)
    burst = slice(samples // 3, samples // 3 + n // 8)
    z[burst] += 60.0 * np.exp(2j * np.pi * (0.05 * n / 2 + 0.1) / n * k[burst])
    inter = np.stack([z.real, z.imag], axis=-1).reshape(-1)
    if fmt == b2s.IQ_CF32:
        return (inter / 127.0).astype(np.float32)
    return np.clip(np.rint(inter), -128, 127).astype(np.int8)


def psd_cfg(n, m, mode, fmt=0, **kw):
    fs = 20_000_000 if n >= 8192 else 2_048_000
    flags = RED[mode] | OVERLAP | kw.pop("flags", 0)
    cfg = b2s.make_config(n, fs, iq_format=fmt, iq_scale=1.0 / 127.0 if fmt == 0 else 1.0, flags=flags, **kw)
    cfg.frame_stride_samples = m * n // 2
    return cfg


# ---- refusals --------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", so.REFUSED + so.ACCEPTED, ids=[c[0] for c in so.REFUSED + so.ACCEPTED])
def test_refusals(engine, case):
    name, flags, stride = case
    cfg = sl.config(b2s, None, flags=flags | OVERLAP)
    cfg.frame_stride_samples = stride
    ok = case in so.ACCEPTED
    h = C.c_void_p()
    rc = b2s.lib().b2s_band_create(engine._h, C.byref(cfg), C.byref(h))
    if h.value:
        b2s.lib().b2s_band_destroy(h)
    assert (rc == 0) == ok and (rc == E_INVALID or ok), name
    iq = np.zeros(2 * (sl.N + 2 * stride), np.int8)
    out = np.zeros(sl.N, np.float32)
    rc = b2s.lib().b2s_psd(engine._h, C.byref(cfg), iq.ctypes.data_as(C.c_void_p), 1, out.ctypes.data_as(C.c_void_p), None)
    assert (rc == 0) == ok and (rc == E_INVALID or ok), name


# ---- K1 per bin ------------------------------------------------------------------------------------------------------------------------
PSD_N = [256, 2048, 4096, 16384, 32768]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("m", [2, 3, 6])
@pytest.mark.parametrize("n", PSD_N)
def test_psd_operator_matches_oracle(engine, n, m, mode):
    """b2s_psd: `iq` starts with frame 0's lead-in, so every frame folds all m sub-frames."""
    frames = 3 if n <= 16384 else 2
    cfg = psd_cfg(n, m, mode)
    h, stride = n // 2, cfg.frame_stride_samples
    iq = noise_tones(n, h + frames * stride, seed=n + m)
    psd, lin = engine.psd(cfg, iq, frames, want_linear=True)  # exactly the documented input length
    ref, ref_lin = so.oracle_rows_overlap(cfg, iq, frames, mode, origin=h, no_lead=(), want_linear=True)
    ol.assert_db_rows_close(psd, ref, f"psd N={n} m={m} {mode}")
    assert np.array_equal(np.argmax(psd, axis=1), np.argmax(ref, axis=1))
    with pytest.raises(ValueError):
        engine.psd(cfg, iq[:-2], frames)


def band_rows(engine, cfg, iq, cuts, device=False, offset=0):
    """psd_db rows of the pushes `cuts` (frames each) of one stream; device input at `offset` bytes from a 16-byte boundary."""
    import torch

    n, stride = cfg.fft_size, cfg.frame_stride_samples
    per = 2 * stride  # scalars per frame
    band = b2s.Band(engine, cfg)
    out, f0 = [], 0
    if device:
        raw = torch.from_numpy(np.frombuffer(iq.tobytes(), np.uint8).copy())
        buf = torch.zeros(raw.numel() + 16, dtype=torch.uint8, device="cuda")
        buf[offset : offset + raw.numel()] = raw.cuda()
    for nf in cuts:
        if device:
            rows = np.zeros((nf, n), np.float32)
            r = b2s.Result()
            r.psd_db = rows.ctypes.data_as(C.POINTER(C.c_float))
            band.push_raw(buf.data_ptr() + offset + f0 * per * iq.itemsize, nf, 0, 1.0, r)
            torch.cuda.synchronize()
            out.append(rows)
        else:
            out.append(band.push(iq[f0 * per : (f0 + nf) * per], nf, 0, 1.0, per_frame=True, dense=("psd_db",)).psd_db)
        f0 += nf
    band.close()
    return np.concatenate(out)


FMTS = [(0, 0), (0, 2), (1, 0)]


@pytest.mark.parametrize("fmt,offset", FMTS, ids=["cs8", "cs8_unaligned", "cf32"])
@pytest.mark.parametrize("n", PSD_N)
@pytest.mark.parametrize("mode", MODES)
def test_band_rows(engine, n, fmt, offset, mode):
    """A band's rows over two pushes: frame 0 of the first has no lead-in (m - 1 sub-frames), the second push's frame 0 takes the
    first push's last N / 2 samples. Device input equals host input bit for bit; an offset of 2 bytes makes K1 read the int8
    frames directly instead of through the TMA staging."""
    m = 3
    frames = (3, 2) if n <= 16384 else (2, 1)
    cfg = psd_cfg(n, m, mode, fmt, learn_frames=2, spectrogram_out_size=0, max_frames_per_push=8)
    iq = noise_tones(n, sum(frames) * cfg.frame_stride_samples, seed=3 + n, fmt=fmt)
    ref = so.oracle_rows_overlap(cfg, iq, sum(frames), mode)
    host = band_rows(engine, cfg, iq, frames)
    ol.assert_db_rows_close(host, ref, f"band N={n} {mode}")
    dcfg = psd_cfg(n, m, mode, fmt, learn_frames=2, spectrogram_out_size=0, max_frames_per_push=8, flags=b2s.FLAG_IQ_ON_DEVICE)
    assert np.array_equal(band_rows(engine, dcfg, iq, frames, device=True, offset=offset), host), "device input differs from host input"


@pytest.mark.parametrize("m", [2, 6])
def test_lead_in_rules(engine, m):
    """No lead-in on the first push and after a centre change (frame 0 folds m - 1 sub-frames); set_center to the same centre and
    b2s_band_reset keep it."""
    n = 2048
    for mode in MODES:
        cfg = psd_cfg(n, m, mode, learn_frames=2, spectrogram_out_size=0)
        stride = cfg.frame_stride_samples
        cuts = (3, 2, 2, 2)
        iq = noise_tones(n, sum(cuts) * stride, seed=m)
        band = b2s.Band(engine, cfg)
        rows, f0 = [], 0
        for i, nf in enumerate(cuts):
            if i == 1:
                band.set_center(cfg.center_hz + 1_000_000, cfg.range_lo_hz, cfg.range_hi_hz)  # changes: no lead-in
            elif i == 2:
                band.set_center(cfg.center_hz + 1_000_000, cfg.range_lo_hz, cfg.range_hi_hz)  # the same centre: kept
            elif i == 3:
                band.reset()  # kept
            rows.append(band.push(iq[2 * f0 * stride : 2 * (f0 + nf) * stride], nf, 0, 1.0, per_frame=True, dense=("psd_db",)).psd_db)
            f0 += nf
        ref = so.oracle_rows_overlap(cfg, iq, sum(cuts), mode, no_lead=(0, cuts[0]))
        ol.assert_db_rows_close(np.concatenate(rows), ref, f"lead-in m={m} {mode}")


# ---- continuity ------------------------------------------------------------------------------------------------------------------------
def band_state(band, centers=()):
    s, a, ring, f = band.get_averager()
    thr, samples, ready = band.get_noise()
    occ = [tuple(np.asarray(x).tobytes() if isinstance(x, np.ndarray) else x for x in band.occupancy(c)) for c in centers]
    return dict(avg=(s, a, ring, f), noise=(thr, samples, ready), tx=band.get_transmissions(), sig=band.get_signals(),
                spec=band.get_spectrogram(), ev=band.get_events(), occ=occ)


def same(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(same(a[k], b[k]) for k in a)
    if isinstance(a, (tuple, list)):
        return len(a) == len(b) and all(same(x, y) for x, y in zip(a, b))
    if isinstance(a, np.ndarray):
        return np.array_equal(a, b)
    return a == b


def scene_cfg(mode, overlap=True, **kw):
    kw.setdefault("spectrogram_out_size", 256)
    cfg = so.config(b2s, mode, overlap, **kw)
    cfg.spectrogram_interval_ms = 50
    return cfg


def run(engine, cfg, iq, cuts, *, dense=True, src=None, bank=None):
    """Push the stream as `cuts`; with `dense`, also every frame's list and row. Returns (band, rows, lists)."""
    import torch

    band = b2s.Band(engine, cfg)
    band.set_event_log(True)
    band.set_occupancy(True)
    if bank is not None:
        band.attach_recorder_bank(bank)
    stride = cfg.frame_stride_samples
    rows, lists, f0 = [], [], 0
    for nf in cuts:
        t0 = int(round(f0 * PERIOD))
        if src is not None:
            band.push_raw(src.data_ptr() + 2 * f0 * stride, nf, t0, PERIOD)
        elif dense:
            o = band.push(iq[2 * f0 * stride : 2 * (f0 + nf) * stride], nf, t0, PERIOD, per_frame=True, dense=("psd_db",))
            rows.append(o.psd_db)
            lists += o.frame_tx
        else:
            band.push_raw(iq[2 * f0 * stride :].ctypes.data, nf, t0, PERIOD)
        f0 += nf
    if cfg.flags & b2s.FLAG_ASYNC:
        band.sync()
    torch.cuda.synchronize()
    return band, (np.concatenate(rows) if rows else None), lists


CUTS = [sl.FRAMES], [7, 33, 1, 64, 35]


@pytest.mark.parametrize("mode", MODES)
def test_cuts_do_not_show_dense(engine, mode):
    """Synchronous host pushes with pieces of 16 frames (max_frames_per_push) and spectrogram cuts: rows, per-frame lists, mailbox,
    map, events, spectrogram, Averager, noise and occupancy are the same for one push and for uneven pushes."""
    iq = so.edge_burst_iq()
    got = []
    for cuts in CUTS:
        for mfp in (0, 16):
            band, rows, lists = run(engine, scene_cfg(mode, max_frames_per_push=mfp), iq, cuts)
            got.append((rows, lists, band_state(band, [band.cfg.center_hz])))
    for g in got[1:]:
        assert np.array_equal(g[0], got[0][0]) and g[1] == got[0][1] and same(g[2], got[0][2])


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("flags", [b2s.FLAG_ASYNC, b2s.FLAG_IQ_ON_DEVICE, b2s.FLAG_ASYNC | b2s.FLAG_IQ_ON_DEVICE],
                         ids=["async_host", "sync_device", "async_device"])
def test_cuts_do_not_show(engine, mode, flags):
    """The device-tracked band (mailbox, map, events, spectrogram, Averager, noise, occupancy) in async mode and with device IQ
    equals the synchronous host band, for one push and for uneven pushes, with and without pieces."""
    import torch

    iq = so.edge_burst_iq()
    src = torch.from_numpy(iq.copy()).cuda() if flags & b2s.FLAG_IQ_ON_DEVICE else None
    ref, _, _ = run(engine, scene_cfg(mode), iq, CUTS[0], dense=False)
    want = band_state(ref, [ref.cfg.center_hz])
    for cuts in CUTS:
        for mfp in (0, 16):
            band, _, _ = run(engine, scene_cfg(mode, flags=flags, max_frames_per_push=mfp), iq, cuts, dense=False, src=src)
            assert same(band_state(band, [band.cfg.center_hz]), want), (cuts, mfp)


@pytest.mark.parametrize("mode", MODES)
def test_chain_equals_oracle_on_own_rows(engine, mode):
    """The oracle chain fed the band's own rows gives the band's per-frame lists, mailbox and noise, with no tolerance; the rows
    match the float64 restatement."""
    iq = so.edge_burst_iq()
    cfg = scene_cfg(mode)
    band, rows, lists = run(engine, cfg, iq, CUTS[1])
    orc = ol.OracleChain(cfg)
    ref = orc.push(rows, sl.FRAMES, 0, PERIOD, dense=(), psd_rows=True)
    key = lambda fr: [[(f, fl, k) for f, fl, k, _ in x] for x in fr]
    assert key(lists) == key(ref.frame_tx)
    assert key([band.get_transmissions()]) == key([orc.get_transmissions()])
    assert np.array_equal(band.get_noise()[0], orc.get_noise()[0])
    ol.assert_db_rows_close(rows[:8], so.oracle_rows_overlap(cfg, iq, 8, mode), "scene rows")


def test_edge_burst_scene(engine):
    """Bursts of N / 16 samples on sub-frame and frame edges: MAX with overlap logs a START at the burst, MAX without does not."""
    iq = so.edge_burst_iq()
    starts = {}
    for overlap in (False, True):
        band, _, lists = run(engine, scene_cfg(so.MAX, overlap), iq, [sl.FRAMES])
        ev = band.get_events()
        shift = so.BURST_HZ
        starts[overlap] = [e for e in ev if e[0] == 1 and abs(e[2] - shift) <= sl.FS / sl.N * 16]
        assert sl.reported(lists, so.BURST_HZ) == overlap
    assert starts[True] and not starts[False]


# ---- recorder bank ---------------------------------------------------------------------------------------------------------------------
def test_recorder_bank(engine):
    """An attached bank's chunks are byte-identical with the flag on and off; the band with a bank equals one without."""
    n, fs, m = 4096, 2_048_000, 6
    stride = m * n // 2
    iq = noise_tones(n, 60 * stride, seed=11)
    chunks, states = [], []
    for flags in (RED[so.MEAN], RED[so.MEAN] | OVERLAP):
        cfg = psd_cfg(n, m, so.MEAN, learn_frames=10, spectrogram_out_size=0, max_frames_per_push=32)
        cfg.flags = flags
        band = b2s.Band(engine, cfg)
        bank = b2s.RecorderBank(engine, fs, 16000, 2, max_samples_per_push=32 * stride)
        band.attach_recorder_bank(bank)
        bank.start(0, 12000)
        got, rows = [], []
        for f0, nf in ((0, 25), (25, 20), (45, 15)):
            rows.append(band.push(iq[2 * f0 * stride : 2 * (f0 + nf) * stride], nf, f0 * 6, 6.0, per_frame=True, dense=("psd_db",)).psd_db)
            got.append([[(t, c.tobytes()) for t, c in bank.flush(ch, cap=1 << 12)] for ch in (0, 1)])
        chunks.append(got)
        if flags & OVERLAP:
            plain = b2s.Band(engine, cfg)
            prow = [plain.push(iq[2 * f0 * stride : 2 * (f0 + nf) * stride], nf, f0 * 6, 6.0, per_frame=True, dense=("psd_db",)).psd_db
                    for f0, nf in ((0, 25), (25, 20), (45, 15))]
            assert np.array_equal(np.concatenate(rows), np.concatenate(prow))
            assert band.get_transmissions() == plain.get_transmissions() and same(band.get_noise(), plain.get_noise())
        band.close()
    assert chunks[0] == chunks[1]


# ---- snapshots -------------------------------------------------------------------------------------------------------------------------
def section_tags(snap):
    at, tags = 20, []
    while at < len(snap) - 8:
        tag, length = struct.unpack_from("<IQ", snap, at)
        tags.append(struct.pack("<I", tag).decode())
        at += 12 + length
    return tags


@pytest.mark.parametrize("mode", MODES)
def test_snapshots(engine, mode):
    """Save mid-stream, load into a fresh band on another engine, continue: the same as an uninterrupted band. A load is refused
    when the overlap bit differs, and changes nothing then; a snapshot without a lead-in drops frame 0's first sub-frame."""
    iq = so.edge_burst_iq()
    cfg = scene_cfg(mode)
    whole, rows, lists = run(engine, cfg, iq, [sl.FRAMES])
    a, _, _ = run(engine, cfg, iq, [60])
    snap = a.save_state()
    assert section_tags(snap)[-1] == "LEAD"
    other = b2s.Engine(0)
    try:
        b = b2s.Band(other, cfg)
        b.load_state(snap)
        stride = cfg.frame_stride_samples
        rb = b.push(iq[2 * 60 * stride :], sl.FRAMES - 60, int(round(60 * PERIOD)), PERIOD, per_frame=True, dense=("psd_db",))
        assert np.array_equal(rb.psd_db, rows[60:]) and rb.frame_tx == lists[60:]
        assert b.get_transmissions() == whole.get_transmissions() and same(b.get_signals(), whole.get_signals())
        b.close()
    finally:
        other.close()
    # refused both ways
    plain = so.config(b2s, mode, False, spectrogram_out_size=256)
    plain.spectrogram_interval_ms = 50
    c = b2s.Band(engine, plain)
    before = c.save_state()
    assert "LEAD" not in section_tags(before)
    with pytest.raises(RuntimeError):
        c.load_state(snap)
    assert c.save_state() == before
    d, _, _ = run(engine, cfg, iq, [30])
    mid = d.save_state()
    with pytest.raises(RuntimeError):
        d.load_state(before)
    assert d.save_state() == mid
    # a fresh band's snapshot holds no lead-in: after loading it, the next push's frame 0 folds m - 1 sub-frames
    fresh = b2s.Band(engine, cfg).save_state()
    d.load_state(fresh)
    stride = cfg.frame_stride_samples
    r = d.push(iq[2 * 30 * stride : 2 * 34 * stride], 4, 0, PERIOD, per_frame=True, dense=("psd_db",)).psd_db
    ol.assert_db_rows_close(r, so.oracle_rows_overlap(cfg, iq[2 * 30 * stride :], 4, mode), "after a snapshot without a lead-in")
