"""Sub-frame PSD rows on the GPU (B2S_FLAG_SUBFRAME_MEAN / _MAX, include/b2s.h): K1 folds each frame's r = floor(stride / N)
sub-frames into its row, and everything downstream sees the new rows.

  * K1 per bin against the oracle's reduced rows (subframe_lib.orc_psd_frame_subframes), the parity criterion of test_gpu_parity.py,
    through b2s_psd and a band's dense rows: every K1 family, r = 2, 3, 5 and a stride that is not a multiple of N, both reductions,
    aligned / unaligned CS8 and CF32, host and device input; peak_index / peak_value are the first maximum of the reduced row.
  * r = 1: either flag is a no-op, bit for bit.
  * the chain, with no tolerance: the oracle fed the band's own rows; the device tracker (K4) against the dense band, sync and
    async with device IQ; uneven pushes against one push.
  * the gap, burst and weak-carrier scenes of subframe_lib, whose oracle outcomes test_subframe_psd_cpu.py pins.
  * an attached recorder bank, snapshots and refusals.
"""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as ol
import subframe_lib as sl
from conftest import load_b2s

b2s = load_b2s()
pytestmark = pytest.mark.gpu

MODES = (sl.MEAN, sl.MAX)
E_INVALID = -1  # B2S_E_INVALID
FLAG = {None: 0, sl.MEAN: 0x400, sl.MAX: 0x800}


def noise_tones(n, stride, frames, seed, fmt=0):
    rng = np.random.default_rng(seed)
    k = np.arange(frames * stride, dtype=np.float64)
    z = (rng.standard_normal(k.size) + 1j * rng.standard_normal(k.size)) * 8.0
    for b, a in ((0.31 * n / 2 + 0.1, 40.0), (-0.12 * n / 2 + 0.1, 25.0)):
        z += a * np.exp(2j * np.pi * b / n * k)
    # a burst inside the last sub-frame of the first stride, so MEAN and MAX differ
    burst = slice(stride - n if stride >= 2 * n else 0, stride)
    z[burst] += 60.0 * np.exp(2j * np.pi * (0.05 * n / 2 + 0.1) / n * k[burst])
    inter = np.stack([z.real, z.imag], axis=-1).reshape(-1)
    if fmt == b2s.IQ_CF32:
        return (inter / 127.0).astype(np.float32)
    return np.clip(np.rint(inter), -128, 127).astype(np.int8)


def psd_cfg(n, stride, mode, fmt=0, **kw):
    fs = 20_000_000 if n >= 8192 else 2_048_000
    flags = FLAG[mode] | kw.pop("flags", 0)
    cfg = b2s.make_config(n, fs, iq_format=fmt, iq_scale=1.0 / 127.0 if fmt == 0 else 1.0, flags=flags, **kw)
    cfg.frame_stride_samples = stride
    return cfg


def oracle_frames(cfg, iq, frames, mode):
    n, stride = cfg.fft_size, cfg.frame_stride_samples
    r = stride // n
    db, lin = np.empty((frames, n), np.float32), np.empty((frames, n), np.float32)
    for k in range(frames):
        db[k], lin[k] = sl.orc_psd_frame_subframes(cfg, None, iq[2 * k * stride : 2 * k * stride + 2 * r * n], r, mode)
    return db, lin


def check_rows(db, ref, n, what):
    ol.assert_db_rows_close(db, ref, what)


PSD_CASES = [
    # (N, stride in units of N or absolute, frames)
    (512, 5 * 512, 4), (2048, 3 * 2048 + 100, 4), (4096, 2 * 4096, 4), (8192, 5 * 8192, 3), (16384, 3 * 16384, 3),
    (32768, 2 * 32768 + 32, 2), (1048576, 2 * 1048576, 1),
]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("n,stride,frames", PSD_CASES, ids=[f"N{c[0]}_r{c[1] // c[0]}" for c in PSD_CASES])
def test_psd_operator_matches_oracle(engine, n, stride, frames, mode):
    """b2s_psd with the flag: every K1 family (k_spectrum, k_spectrum3 direct, split), r = 2, 3, 5, strides not a multiple of N."""
    cfg = psd_cfg(n, stride, mode)
    r = stride // n
    iq = noise_tones(n, stride, frames, seed=n + r)
    need = 2 * ((frames - 1) * stride + r * n)
    psd, lin = engine.psd(cfg, iq[:need], frames, want_linear=True)  # exactly the documented input length
    ref, ref_lin = oracle_frames(cfg, iq, frames, mode)
    check_rows(psd, ref, n, f"N={n} r={r} {mode}")
    assert np.array_equal(np.argmax(psd, axis=1), np.argmax(ref, axis=1))


@pytest.mark.parametrize("fmt,unaligned", [(0, False), (0, True), (1, False)], ids=["cs8", "cs8_unaligned", "cf32"])
@pytest.mark.parametrize("n", [1024, 4096, 16384, 65536])
@pytest.mark.parametrize("mode", MODES)
def test_band_rows_and_peaks(engine, n, fmt, unaligned, mode):
    """A band's dense psd_db rows and its peaks, host and device input; an odd stride makes the CS8 frames unaligned (K1's direct
    loads instead of the TMA staging)."""
    frames = 4 if n <= 16384 else 2
    stride = 3 * n + (1 if unaligned else 0)  # one sample: frames 2 bytes off the 16-byte grid
    cfg = psd_cfg(n, stride, mode, fmt, learn_frames=2, spectrogram_out_size=0, max_frames_per_push=8)
    iq = noise_tones(n, stride, frames, seed=7 + n, fmt=fmt)
    need = 2 * ((frames - 1) * stride + 3 * n)
    ref, _ = oracle_frames(cfg, iq, frames, mode)
    got = b2s.Band(engine, cfg).push(iq[:need], frames, 0, 1.0, per_frame=True, dense=("psd_db",))
    check_rows(got.psd_db, ref, n, f"band N={n} {mode}")
    assert np.array_equal(got.peak_index, np.argmax(got.psd_db, axis=1))
    assert np.array_equal(got.peak_value, got.psd_db.max(axis=1))
    import torch

    dcfg = psd_cfg(n, stride, mode, fmt, learn_frames=2, spectrogram_out_size=0, max_frames_per_push=8, flags=b2s.FLAG_IQ_ON_DEVICE)
    dev = torch.from_numpy(iq[:need].copy()).cuda()
    res = b2s.Band(engine, dcfg)
    rows = np.zeros((frames, n), np.float32)
    r = b2s.Result()
    r.psd_db = rows.ctypes.data_as(C.POINTER(C.c_float))
    res.push_raw(dev.data_ptr(), frames, 0, 1.0, r)
    torch.cuda.synchronize()
    assert np.array_equal(rows, got.psd_db), "device input differs from host input"


# ---- the chain ---------------------------------------------------------------------------------------------------------------------
PERIOD = sl.R * sl.N * 1000.0 / sl.FS


def run_dense(engine, cfg, iq, cuts):
    band = b2s.Band(engine, cfg)
    band.set_event_log(True)
    outs, f0 = [], 0
    stride = cfg.frame_stride_samples
    for nf in cuts:
        outs.append(band.push(iq[2 * f0 * stride : 2 * (f0 + nf) * stride], nf, int(round(f0 * PERIOD)), PERIOD, per_frame=True,
                              dense=("psd_db",)))
        f0 += nf
    return band, outs


def band_state(band):
    s, a, ring, f = band.get_averager()
    thr, samples, ready = band.get_noise()
    return dict(avg=(s, a, ring, f), noise=(thr, samples, ready), tx=band.get_transmissions(), sig=band.get_signals(),
                spec=band.get_spectrogram(), ev=band.get_events())


def same(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(same(a[k], b[k]) for k in a)
    if isinstance(a, (tuple, list)):
        return len(a) == len(b) and all(same(x, y) for x, y in zip(a, b))
    if isinstance(a, np.ndarray):
        return np.array_equal(a, b)
    return a == b


@pytest.mark.parametrize("mode", MODES)
def test_r1_is_a_no_op(engine, mode):
    """stride < 2N: a band with the flag equals one without it bit for bit."""
    iq = sl.scene_iq(sl.GAP_ON, sl.GAP_AMP, frames=90)
    base = sl.config(b2s, None, spectrogram_out_size=256)
    base.frame_stride_samples = sl.N + sl.N // 2  # r = 1; the scene's strides are re-read at 1.5 N
    cfg = sl.config(b2s, mode, spectrogram_out_size=256)
    cfg.frame_stride_samples = base.frame_stride_samples
    a, oa = run_dense(engine, base, iq, [40, 50])
    b, ob = run_dense(engine, cfg, iq, [40, 50])
    for x, y in zip(oa, ob):
        assert np.array_equal(x.psd_db, y.psd_db) and x.frame_tx == y.frame_tx and np.array_equal(x.peak_index, y.peak_index)
        assert np.array_equal(x.peak_value, y.peak_value)
    assert same(band_state(a), band_state(b))


def lists(frame_tx):
    return [[(f, fl, k) for f, fl, k, _ in fr] for fr in frame_tx]


@pytest.mark.parametrize("mode", MODES)
def test_chain_equals_oracle_on_own_rows(engine, mode):
    """The oracle chain fed the band's own rows gives the band's per-frame lists, Averager, noise, spectrogram and map, with no
    tolerance; uneven pushes equal one push."""
    iq = sl.scene_iq(sl.GAP_ON, sl.GAP_AMP, seed=3)
    cfg = sl.config(b2s, mode, spectrogram_out_size=256)
    cfg.spectrogram_interval_ms = 200
    band, outs = run_dense(engine, cfg, iq, [sl.FRAMES])
    one = outs[0]
    orc = ol.OracleChain(cfg)
    ref = orc.push(one.psd_db, sl.FRAMES, 0, PERIOD, dense=(), psd_rows=True)
    # the lists' shifts, flushes and keys; a transmission's power is a float sum whose last bits the oracle does not pin (smoke())
    assert lists(one.frame_tx) == lists(ref.frame_tx) and sl.reported(one.frame_tx)
    s, a, ring, f = band.get_averager()
    rs, ra, rring, rf = orc.get_averager()
    assert np.array_equal(s, rs) and np.array_equal(a, ra) and f == rf
    thr, _, _ = band.get_noise()
    assert np.array_equal(thr, orc.get_noise()[0])
    t, c, rows = band.get_spectrogram()
    rt, rc, rrows = orc.get_spectrogram()
    assert np.array_equal(t, rt) and np.array_equal(rows, rrows) and len(t) > 0
    assert lists([band.get_transmissions()]) == lists([orc.get_transmissions()])
    uneven, uo = run_dense(engine, cfg, iq, [7, 33, 1, 64, 35])
    assert [x for o in uo for x in o.frame_tx] == one.frame_tx
    assert np.array_equal(np.concatenate([o.psd_db for o in uo]), one.psd_db)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("flags", [0, b2s.FLAG_ASYNC | b2s.FLAG_IQ_ON_DEVICE], ids=["sync", "async_device"])
def test_fast_band_equals_dense_band(engine, mode, flags):
    """The device-tracked band (K4, mailbox only) equals the dense band in mailbox, signals and events."""
    import torch

    iq = sl.scene_iq(sl.BURST_ON, sl.BURST_AMP, seed=5)
    dense, outs = run_dense(engine, sl.config(b2s, mode), iq, [sl.FRAMES])
    fast = b2s.Band(engine, sl.config(b2s, mode, flags=flags))
    fast.set_event_log(True)
    stride = sl.R * sl.N
    src = torch.from_numpy(iq.copy()).cuda() if flags & b2s.FLAG_IQ_ON_DEVICE else None
    f0 = 0
    for nf in (50, 40, 50):
        if src is not None:
            fast.push_raw(src.data_ptr() + 2 * f0 * stride, nf, int(round(f0 * PERIOD)), PERIOD)
        else:
            fast.push_raw(iq[2 * f0 * stride :].ctypes.data, nf, int(round(f0 * PERIOD)), PERIOD)
        f0 += nf
    if flags & b2s.FLAG_ASYNC:
        fast.sync()
    torch.cuda.synchronize()
    assert fast.get_transmissions() == dense.get_transmissions()
    assert same(fast.get_signals(), dense.get_signals())
    assert fast.get_events() == dense.get_events()


# ---- scenes ------------------------------------------------------------------------------------------------------------------------
def band_reports(engine, iq, mode):
    _, outs = run_dense(engine, sl.config(b2s, mode), iq, [sl.FRAMES])
    return sl.reported(outs[0].frame_tx)


def test_gap_scene(engine):
    iq = sl.scene_iq(sl.GAP_ON, sl.GAP_AMP)
    assert not band_reports(engine, iq, None)
    assert band_reports(engine, iq, sl.MEAN) and band_reports(engine, iq, sl.MAX)


def test_burst_scene(engine):
    iq = sl.scene_iq(sl.BURST_ON, sl.BURST_AMP)
    assert not band_reports(engine, iq, None)
    assert band_reports(engine, iq, sl.MAX)
    assert band_reports(engine, iq, sl.MEAN) == sl.oracle_outcome(b2s, iq, sl.MEAN)


def test_weak_carrier(engine):
    iq = sl.scene_iq(sl.WEAK_ON, sl.WEAK_AMP)
    assert not band_reports(engine, iq, None)
    assert band_reports(engine, iq, sl.MEAN)


# ---- recorder bank, snapshots, refusals ---------------------------------------------------------------------------------------------
def test_recorder_bank_input_unchanged(engine):
    """r = 3 with history: the bank's bytes equal those of a flag-off band's bank fed the same IQ; record_from maps alike."""
    n, fs, frames = 4096, 2_048_000, 60
    stride = 3 * n
    iq = noise_tones(n, stride, frames, seed=11)
    got = []
    for mode in (None, sl.MEAN):
        cfg = psd_cfg(n, stride, mode, learn_frames=10, spectrogram_out_size=0, max_frames_per_push=32)
        band = b2s.Band(engine, cfg)
        bank = b2s.RecorderBank(engine, fs, 16000, 2, max_samples_per_push=32 * stride)
        bank.set_history(8 * stride)
        band.attach_recorder_bank(bank)
        bank.start(0, 12000)
        chunks = []
        for f0, nf in ((0, 25), (25, 20), (45, 15)):
            band.push(iq[2 * f0 * stride : 2 * (f0 + nf) * stride], nf, f0 * 6, 6.0)
            if f0 == 25:
                band.record_from(1, -20000, 40)
            chunks.append([[(t, c.tobytes()) for t, c in bank.flush(ch, cap=1 << 12)] for ch in (0, 1)])
        got.append((chunks, bank.history()))
        band.close()
    assert got[0] == got[1]


@pytest.mark.parametrize("mode", MODES)
def test_snapshots(engine, mode):
    iq = sl.scene_iq(sl.GAP_ON, sl.GAP_AMP, seed=9)
    cfg = sl.config(b2s, mode)
    a, _ = run_dense(engine, cfg, iq, [60])
    snap = a.save_state()
    b = b2s.Band(engine, cfg)
    b.load_state(snap)
    stride = cfg.frame_stride_samples
    rest = iq[2 * 60 * stride :]
    ra = a.push(rest, sl.FRAMES - 60, int(round(60 * PERIOD)), PERIOD, per_frame=True, dense=("psd_db",))
    b.set_event_log(True)
    rb = b.push(rest, sl.FRAMES - 60, int(round(60 * PERIOD)), PERIOD, per_frame=True, dense=("psd_db",))
    assert ra.frame_tx == rb.frame_tx and np.array_equal(ra.psd_db, rb.psd_db)
    assert b.get_transmissions() == a.get_transmissions()
    for other in (None, sl.MAX if mode == sl.MEAN else sl.MEAN):
        c = b2s.Band(engine, sl.config(b2s, other))
        before = c.save_state()
        with pytest.raises(RuntimeError):
            c.load_state(snap)
        assert c.save_state() == before


def test_both_flags_refused(engine):
    cfg = sl.config(b2s, None, flags=b2s.FLAG_SUBFRAME_MEAN | b2s.FLAG_SUBFRAME_MAX)
    h = C.c_void_p()
    assert b2s.lib().b2s_band_create(engine._h, C.byref(cfg), C.byref(h)) == E_INVALID
    assert not h.value
    iq = np.zeros(2 * sl.R * sl.N, np.int8)
    out = np.zeros(sl.N, np.float32)
    assert b2s.lib().b2s_psd(engine._h, C.byref(cfg), iq.ctypes.data_as(C.c_void_p), 1, out.ctypes.data_as(C.c_void_p), None) == E_INVALID
