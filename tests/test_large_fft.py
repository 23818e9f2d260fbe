"""N = 524288 and 1048576: the FFT sizes b2s_default_config picks for receivers above 65.536 MS/s (getFft(fs, 250)), run as
S = 32 and 64 residue classes of K1's split mode. PSD rows against the oracle in every load mode, the packed per-frame maximum,
K2 and the trackers bit for bit against the restatement, and the reference's default configuration end to end.

Every band stays near 5 GB of device memory or below: explicit max_frames_per_push / detect_capacity, except where the default
push capacity is itself under test."""
import ctypes as C

import numpy as np
import pytest

import k2_restate as k2
import oracle_lib as ol
from conftest import load_b2s
from test_gpu_parity import _noise_tones, _tx
from test_k2_exact import DENSE, _mailbox, _same, _sm_count, k2_variant
from test_oracle_chain import synth
from test_oracle_spectrum import power_parity_stats

b2s = load_b2s()
SIZES = [524288, 1048576]


def _torch_iq(n, frames, tones, seed, quiet_frames, stride=1):
    """int8 IQ of `frames` frames of stride * n samples, generated on the GPU: synth's model with n_fft = stride * n and the tones
    rescaled, so each frame's first n samples carry the tones at their bin offsets (and FM deviations) in n-point bins."""
    tones = [synth.Tone(t.bin_offset * stride, t.amplitude, t.on_frames, t.phase, t.fm_dev_bins * stride, t.fm_rate_cycles_per_frame) for t in tones]
    return synth.make_iq_int8_torch(stride * n, frames, tones, seed=seed, quiet_frames=quiet_frames, device="cuda")


# ------------------------------------------------------------------------------------------------------------
# K1
# ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("n", SIZES)
def test_psd_rows_match_oracle(engine, n):
    """test_gpu_parity's bars, unchanged: S = 32 / 64 residue classes of 16384 points."""
    frames = 3
    cfg = b2s.make_config(n, 20_000_000)
    iq = _noise_tones(n, frames, seed=n)
    psd, lin = engine.psd(cfg, iq, frames, want_linear=True)
    ref, ref_lin = np.empty_like(psd), np.empty_like(lin)
    for k in range(frames):
        ref[k], ref_lin[k] = ol.oracle_psd_frame(cfg, iq[k * 2 * n : (k + 1) * 2 * n], want_linear=True)
    ol.assert_db_rows_close(psd, ref, f"N={n}")
    st = power_parity_stats(lin, ref_lin)
    print(f"\nN={n}: floored pass {st['pass_frac']:.5f} worst {st['worst']:.2e} strict pass {st['strict_frac']:.4f} L2rel {st['l2_rel']:.2e}")
    assert st["pass_frac"] >= 0.995 and st["worst"] <= ol.worst_tolerance(n) and st["l2_rel"] <= 1e-6, st
    assert np.array_equal(np.argmax(psd, axis=1), np.argmax(ref, axis=1))


@pytest.mark.gpu
@pytest.mark.parametrize("n", SIZES)
def test_psd_input_variants(engine, n):
    """The pre-pass in its three load modes: CS8 staged by bulk copies (aligned), CS8 loaded directly (stride N + 3), CF32; and a
    decimated stride (3N) equal to the undecimated rows.

    CF32 and CS8 round the unpack differently, so their rows are two fp32 FFTs of slightly different inputs. Each is held to the
    oracle's bars; against each other they are held to twice those bars, since each may sit at its bar on the opposite side
    (at N = 1048576 the largest main-lobe difference is about 2.2e-3 dB)."""
    fs, frames = 20_000_000, 2
    iq = _noise_tones(n, frames, seed=3)
    base = engine.psd(b2s.make_config(n, fs), iq, frames)
    ref = np.stack([ol.oracle_psd_frame(b2s.make_config(n, fs), iq[k * 2 * n : (k + 1) * 2 * n]) for k in range(frames)])
    print(f"\nN={n} cs8 vs oracle: {ol.assert_db_rows_close(base, ref, f'cs8 N={n}')}")
    f32 = (iq.astype(np.float32) * np.float32(1 / 127.0)).astype(np.float32)
    cfg_f = b2s.make_config(n, fs, iq_format=b2s.IQ_CF32)
    cf = engine.psd(cfg_f, f32, frames)
    ref_f = np.stack([ol.oracle_psd_frame(cfg_f, f32[k * 2 * n : (k + 1) * 2 * n]) for k in range(frames)])
    ol.assert_db_rows_close(cf, ref_f, f"cf32 N={n} vs oracle")
    st = ol.db_rows_stats(cf, base)
    assert st["worst"] <= 2 * ol.worst_tolerance(n) and st["pass_frac"] >= 0.995 and st["db_max_main"] <= 4e-3, ("cf32 vs cs8", st)
    del f32, cf, ref_f
    wide = np.full((frames, 3 * n * 2), 77, np.int8)
    wide[:, : 2 * n] = iq.reshape(frames, 2 * n)
    assert np.array_equal(engine.psd(b2s.make_config(n, fs, decimator=3), wide.reshape(-1), frames), base)
    del wide
    cfg = b2s.make_config(n, fs)
    cfg.frame_stride_samples = n + 3  # 2N + 6 bytes: not a multiple of 16 -> direct loads
    odd = np.zeros((frames, (n + 3) * 2), np.int8)
    odd[:, : 2 * n] = iq.reshape(frames, 2 * n)
    assert np.array_equal(engine.psd(cfg, odd.reshape(-1), frames), base)


@pytest.mark.gpu
@pytest.mark.parametrize("n", SIZES)
def test_psd_peaks_through_the_band(engine, n):
    """peak_index / peak_value: the first maximum of each row, reduced over 32 / 64 classes through the packed atomic maximum."""
    frames = 4
    cfg = b2s.make_config(n, 20_000_000, learn_frames=2, spectrogram_out_size=0, max_frames_per_push=8, detect_capacity=4096)
    iq = _noise_tones(n, frames, seed=n + 1)
    got = b2s.Band(engine, cfg).push(iq, frames, 0, 1.0, per_frame=True, dense=("psd_db",))
    assert np.array_equal(got.peak_index, np.argmax(got.psd_db, axis=1))
    assert np.array_equal(got.peak_value, got.psd_db.max(axis=1))


# ------------------------------------------------------------------------------------------------------------
# K2 and the trackers, bit for bit (test_k2_exact's method)
# ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("n,splits,reset_at", [(524288, (17, 40, 1, 62), 2), (1048576, (40, 1, 23, 56), 3)])
def test_k2_bit_exact_against_the_restatement(engine, n, splits, reset_at):
    """Dense band A, host-tracked fast band B, device-tracked band C (asynchronous with device IQ at N = 1048576): PSD rows, noise,
    Averager, entries, per-frame lists, mailbox, signal map and spectrogram without tolerance. At fs = 1000 N the spectrogram
    decimation is d = 32 / 64, so K2 takes 128-bin CTAs: k_detect<21,10,152>."""
    import torch

    frames, learn = sum(splits), 20
    cfg = b2s.make_config(n, 1000 * n, learn_frames=learn, recording_bandwidth_hz=16_000, min_time_ms=20, timeout_ms=30, max_frames_per_push=64,
                          detect_capacity=16384)
    cfg.spectrogram_interval_ms = 11
    assert n // cfg.spectrogram_out_size == n // 16384
    assert k2_variant(n, cfg.grouping_x, cfg.grouping_y, cfg.spectrogram_out_size, _sm_count()) == "<21,10,152>"
    iq_dev = _torch_iq(n, frames, synth.standard_scene(n, frames, learn), seed=synth.seed_for(7, n), quiet_frames=learn)
    iq = iq_dev.cpu().numpy()
    on_device = n == 1048576
    if not on_device:
        del iq_dev
        torch.cuda.empty_cache()
    band_a, band_b = b2s.Band(engine, cfg), b2s.Band(engine, cfg)
    ccfg = b2s.BandConfig.from_buffer_copy(cfg)
    if on_device:
        ccfg.flags |= b2s.FLAG_ASYNC | b2s.FLAG_IQ_ON_DEVICE
    band_c = b2s.Band(engine, ccfg)
    bands = (band_a, band_b, band_c)
    host, rest = b2s.HostTransmission(cfg), k2.K2Restatement(cfg)
    stop = np.float32(cfg.stop_level)
    entries = listed = below = 0
    sent = []
    k = 0
    for i, m in enumerate(splits):
        if i == reset_at:
            for x in bands + (host, rest):
                x.reset()
        t0, part = 500 + k, iq[k * 2 * n :]
        a = band_a.push(part, m, t0, 1.0, dense=DENSE)
        b = band_b.push(part, m, t0, 1.0, per_frame=True, dense=("psd_db",))
        if on_device:
            band_c.push_raw(iq_dev.data_ptr() + k * 2 * n, m, t0, 1.0)
            c = band_c.sync()
        else:
            psd_c = np.zeros((m, n), np.float32)
            c = b2s.Result()
            c.psd_db = psd_c.ctypes.data_as(C.POINTER(C.c_float))
            band_c.push_raw(part.ctypes.data, m, t0, 1.0, c)
            assert _same(psd_c, a.psd_db), (i, "psd C")
        where = (n, i, k, m)
        assert _same(a.psd_db, b.psd_db), where
        r = rest.push(a.psd_db, t0, 1.0)
        assert _same(a.noise_sub_db, r.q) and _same(a.avg_db, r.avg) and _same(a.box_db, r.box), where
        want_thr, want_samples, want_ready = rest.noise()
        for name, band in zip("ABC", bands):
            thr, samples, ready = band.get_noise()
            assert _same(thr, want_thr) and (samples, ready) == (want_samples, want_ready), where + (name, "noise")
            for got, want in zip(band.get_averager(), rest.averager()):
                assert _same(got, want), where + (name, "averager")
        want_entries = int(r.entries.sum())
        assert (a.n_detect_entries, b.n_detect_entries, c.n_detect_entries) == (want_entries,) * 3, where
        entries += want_entries
        lists = host.push(r.box, r.q, t0, 1.0)
        for f in range(m):
            assert b.frame_tx[f] == lists[f], where + (f, b.frame_tx[f], lists[f])
        listed += sum(len(x) for x in lists)
        below += sum(1 for x in lists for t in x if np.float32(t[3]) < stop)
        # at these sizes the list can outgrow the result's embedded array, which holds the MAX_TX strongest
        assert _mailbox(c) == lists[-1][: b2s.MAX_TX] and c.n_transmissions_total == len(lists[-1]), where
        sent += r.spectrogram
        k += m
    for x, y in zip(band_b.get_signals(), band_c.get_signals()):
        assert _same(x, y), n
    for name, band in zip("ABC", bands):
        times, _, rows = band.get_spectrogram(cap=4096)
        assert times.tolist() == [t for t, _ in sent], (n, name)
        assert _same(rows, np.stack([row for _, row in sent]).reshape(len(sent), -1)), (n, name)
    print(f"\nN={n}: {frames} frames, {entries} detection entries, {listed} list records, {below} below stop_level, {len(sent)} spectrogram rows")
    assert entries > 0 and listed > 0 and below > 0 and len(sent) >= 5


# ------------------------------------------------------------------------------------------------------------
# the reference's default configuration
# ------------------------------------------------------------------------------------------------------------
def _default_config(fs):
    cfg = b2s.BandConfig()
    b2s.lib().b2s_default_config(C.byref(cfg), fs, 433_000_000, 32_000)
    return cfg


@pytest.mark.gpu
@pytest.mark.parametrize("fs,n,r,d,g,cf32", [(104_857_600, 524288, 4, 32, 160, True), (200_000_000, 1048576, 3, 64, 168, False)])
def test_default_config_end_to_end(engine, fs, n, r, d, g, cf32):
    """b2s_default_config above 65.536 MS/s gives a band that works, with the default push capacity: mailbox, signal map, noise
    threshold and spectrogram rows equal the oracle chain's after every push. Only the noise-learning time and the recording
    time-outs are shortened, so that the scene fits in 160 frames."""
    import torch

    cfg = _default_config(fs)
    assert (cfg.fft_size, cfg.frame_stride_samples // cfg.fft_size, cfg.fft_size // cfg.spectrogram_out_size, cfg.group_size_bins) == (n, r, d, g)
    assert cfg.max_frames_per_push == 0 and cfg.iq_format == b2s.IQ_CS8
    period = synth.frame_period_ms(n, fs, r)
    cfg.noise_learning_ms = 400
    cfg.min_time_ms, cfg.timeout_ms = 200, 300
    learn = b2s.lib().b2s_learn_frames_from_ms(400, C.c_double(period))
    frames = 160
    iq_dev = _torch_iq(n, frames, synth.standard_scene(n, frames, learn), seed=synth.seed_for(12, r), quiet_frames=learn, stride=r)
    iq = iq_dev.cpu().numpy()
    del iq_dev
    torch.cuda.empty_cache()
    formats = [b2s.IQ_CS8] + ([b2s.IQ_CF32] if cf32 else [])
    for fmt in formats:
        c = b2s.BandConfig.from_buffer_copy(cfg)
        c.iq_format = fmt
        band, o = b2s.Band(engine, c), ol.OracleChain(c)
        k, t0, listed = 0, 1000, 0
        for m in (learn + 3, 50, 1, 160 - learn - 54):
            part = iq[k * r * 2 * n : (k + m) * r * 2 * n]
            if fmt == b2s.IQ_CF32:
                part = (part.astype(np.float32) * np.float32(1 / 127.0)).astype(np.float32)
            ts = t0 + int(np.floor(k * period + 0.5))
            res = band.push_raw(part.ctypes.data, m, ts, period)
            ref = o.push(part, m, ts, period, dense=())
            where = (n, fmt, k, m)
            assert [(f, fl, key) for f, fl, key, _ in _mailbox(res)] == _tx(ref.frame_tx)[-1], where
            for x, y in zip(band.get_signals()[:3], o.get_signals()[:3]):
                assert np.array_equal(x, y), where
            thr_g, samples_g, ready_g = band.get_noise()
            thr_o, samples_o, ready_o = o.get_noise()
            assert (samples_g, ready_g) == (samples_o, ready_o), where
            if ready_o:
                assert np.max(np.abs(thr_g - thr_o)) <= 2e-3, where
            t_g, _, rows_g = band.get_spectrogram()
            t_o, _, rows_o = o.get_spectrogram()
            assert np.array_equal(t_g, t_o) and np.max(np.abs(rows_g.astype(int) - rows_o.astype(int)), initial=0) <= 1, where
            listed += sum(len(x) for x in ref.frame_tx)
            k += m
        print(f"\nfs={fs} N={n} fmt={fmt}: {frames} frames, learn {learn}, {listed} list records")
        assert listed > 20
        band.close()


# ------------------------------------------------------------------------------------------------------------
# sizing and refusals
# ------------------------------------------------------------------------------------------------------------
def _large_config(n, max_frames):
    return b2s.make_config(n, 1000 * n, max_frames_per_push=max_frames)


def test_push_capacity_cap_is_checked_with_the_config():
    """The checks run in the config validation the host tracker shares with the band, so they hold without a GPU."""
    with pytest.raises(b2s.B2SError) as e:
        b2s.HostTransmission(_large_config(2097152, 8))
    assert "b2s error -1" in str(e.value) and "fft_size" in str(e.value)
    with pytest.raises(b2s.B2SError) as e:
        b2s.HostTransmission(_large_config(1048576, 1025))
    assert "b2s error -1" in str(e.value) and "max_frames_per_push 1025" in str(e.value) and "4 GiB" in str(e.value)
    for n, m in ((1048576, 1024), (524288, 2048), (524288, 0), (262144, 8192)):
        b2s.HostTransmission(_large_config(n, m)).close()


@pytest.mark.gpu
def test_band_refusals_and_default_capacity(engine):
    for n, m in ((2097152, 8), (1048576, 1025)):
        with pytest.raises(b2s.B2SError) as e:
            b2s.Band(engine, _large_config(n, m))
        assert "b2s error -1" in str(e.value)
    b2s.Band(engine, _large_config(524288, 0)).close()
