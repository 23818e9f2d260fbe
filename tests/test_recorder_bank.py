"""Recorder bank (b2s_recorder_bank_*): SdrDevice's pool of Recorders on one IQ stream (sdr_device.cpp:39-41,82-144), with Recorder's
timestamped flush chunks (recorder.cpp:35-39,89-97, buffer.h:22-55). Every channel must produce the bytes of a separately driven
b2s_recorder; chunks and their times follow the rule in include/b2s.h."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from conftest import ROOT, load_b2s

sys.path.insert(0, os.path.join(ROOT, "oracle"))
import recorder_oracle as ro  # noqa: E402

b2s = load_b2s()
pytestmark = pytest.mark.gpu


def _stream(fs, n, tones, seed=1, sigma=6.0):
    rng = np.random.default_rng(seed)
    t = np.arange(n, dtype=np.float64)
    x = sigma * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    for f_hz, amp in tones:
        x += amp * np.exp(2j * np.pi * (f_hz / fs) * t)
    iq = np.empty(2 * n, np.int8)
    iq[0::2] = np.clip(np.rint(x.real), -128, 127)
    iq[1::2] = np.clip(np.rint(x.imag), -128, 127)
    return iq


def _pieces(n, sizes):
    """Consecutive (start, length) pieces of a stream of n samples, cycling through `sizes`."""
    out, k, i = [], 0, 0
    while k < n:
        m = min(sizes[i % len(sizes)], n - k)
        out.append((k, m))
        k += m
        i += 1
    return out


class _Input:
    """The same stream as host arrays or as device pointers, in CS8 or CF32."""

    def __init__(self, iq8, fmt, on_device):
        self.fmt, self.on_device = fmt, on_device
        self.host = iq8 if fmt == b2s.IQ_CS8 else (iq8.astype(np.float32) * np.float32(1 / 127.0)).astype(np.float32)
        self.bytes_per_sample = 2 * self.host.itemsize
        if on_device:
            import torch

            self.dev = torch.from_numpy(self.host.copy()).cuda()
            torch.cuda.synchronize()

    def piece(self, k, m):
        """(iq argument, n_samples) for samples [k, k + m)."""
        if self.on_device:
            return self.dev.data_ptr() + k * self.bytes_per_sample, m
        return self.host[2 * k : 2 * (k + m)], None


def _push_bank(bank, inp, k, m, t0_ms=0):
    iq, n = inp.piece(k, m)
    return bank.push(iq, t0_ms, n_samples=n) if n is not None else bank.push(iq, t0_ms)


def _push_rec(rec, inp, k, m):
    iq, n = inp.piece(k, m)
    return rec.push(iq, n) if n is not None else rec.push(iq)


# ---- 1. byte equality with b2s_recorder ----
CASES = [(40_000_000, 32_000, 1 << 21), (1_024_000, 20_000, 1 << 19)]


@pytest.mark.parametrize("fs,bw,n", CASES)
@pytest.mark.parametrize("fmt", [b2s.IQ_CS8, b2s.IQ_CF32])
@pytest.mark.parametrize("on_device", [False, True])
def test_bank_channels_equal_separate_recorders(engine, fs, bw, n, fmt, on_device):
    shifts = [0, -int(0.31 * fs), int(0.12 * fs), int(0.12 * fs), -2_500 * (fs // 400_000), int(0.2 * fs)]
    tones = [(s + 1_500, 40.0) for s in shifts] + [(fs // 3, 30.0)]
    inp = _Input(_stream(fs, n, tones, seed=fs % 1000 + fmt), fmt, on_device)
    # uneven pushes: 1 sample, pieces shorter than the filters' history, large pieces
    pieces = _pieces(n, [1, 7, 301, 1000, 250_001, 17, 99_999, 3, 400_000])
    assert len(pieces) > 8
    starts = {0: [0, 1], 1: [2, 3], 3: [4, 5]}  # push index -> channels started before it
    restart_at, restart_ch, restart_shift = 6, 1, int(-0.05 * fs)  # channel 1 is stopped and restarted with a new shift before push 6
    bank = b2s.RecorderBank(engine, fs, bw, len(shifts), iq_format=fmt, on_device=on_device, max_samples_per_push=400_000)
    recs = [b2s.Recorder(engine, fs, bw, iq_format=fmt, on_device=on_device, max_samples_per_push=400_000) for _ in shifts]
    live = [False] * len(shifts)
    got = [[] for _ in shifts]
    want = [[] for _ in shifts]
    for p, (k, m) in enumerate(pieces):
        for c in starts.get(p, []):
            bank.start(c, shifts[c])
            recs[c].start(shifts[c])
            live[c] = True
        if p == restart_at:
            bank.stop(restart_ch)
            recs[restart_ch].stop()
            bank.start(restart_ch, restart_shift)
            recs[restart_ch].start(restart_shift)
            got[restart_ch], want[restart_ch] = [], []
        outs = _push_bank(bank, inp, k, m)
        for c in range(len(shifts)):
            if live[c]:
                got[c].append(outs[c])
                want[c].append(_push_rec(recs[c], inp, k, m))
            else:
                assert len(outs[c]) == 0
    for c in range(len(shifts)):
        g, w = np.concatenate(got[c]), np.concatenate(want[c])
        assert len(w) > 200 and np.array_equal(g, w), (c, len(g), len(w))
    # the two channels with the same shift and the same start produce the same bytes
    assert np.array_equal(np.concatenate(got[2]), np.concatenate(got[3]))
    assert np.abs(np.concatenate(got[0]).astype(int)).max() > 20  # the in-band tone came through
    bank.close()
    for r in recs:
        r.close()


# ---- 2. channel independence ----
def test_channel_bytes_do_not_depend_on_the_other_channels(engine):
    fs, bw, n = 40_000_000, 32_000, 1 << 21
    iq = _stream(fs, n, [(4_700_000, 50.0), (-3_200_000, 40.0)], seed=7)
    pieces = _pieces(n, [65_536, 3, 200_000, 11])
    runs = []
    for others in (False, True):
        bank = b2s.RecorderBank(engine, fs, bw, 8, max_samples_per_push=200_000)
        bank.start(5, 4_700_000)
        out = []
        for p, (k, m) in enumerate(pieces):
            if others and p == 2:
                for c, s in ((0, -3_200_000), (1, 4_700_000), (7, 0)):
                    bank.start(c, s)
            if others and p == 9:
                bank.stop(1)
            out.append(bank.push(iq[2 * k : 2 * (k + m)])[5])
        runs.append(np.concatenate(out))
        bank.close()
    assert len(runs[0]) > 1000 and np.array_equal(runs[0], runs[1])


# ---- 3. oracle ----
def test_bank_channel_matches_the_oracle(engine):
    fs, bw, shift, n = 40_000_000, 32_000, 4_700_000, 1 << 21
    iq = _stream(fs, n, [(shift + 3_000, 50.0), (shift - 6_500, 20.0), (shift + 4 * bw, 60.0)])
    bank = b2s.RecorderBank(engine, fs, bw, 3, max_samples_per_push=n)
    bank.start(0, -1_000_000)
    bank.start(2, shift)
    got = bank.push(iq)[2]
    x = (iq[0::2].astype(np.float64) + 1j * iq[1::2].astype(np.float64)) / 127.0
    want = ro.recorder_chain(x, fs, bw, shift)
    assert len(got) == len(want)
    d = np.abs(got.astype(int) - want.astype(int))
    assert d.max() <= 1 and np.mean(d == 0) >= 0.99, (d.max(), np.mean(d == 0))
    assert np.abs(want.astype(int)).max() > 30


# ---- 4. chunks ----
def _chunk_time(start_ms, j, chunk, bw):
    num = (j + 1) * chunk * 1000
    return start_ms + (2 * num + bw) // (2 * bw)


@pytest.mark.parametrize("fs,bw", [(2_048_000, 32_000), (1_024_000, 20_000)])
def test_flush_chunks_and_times(engine, fs, bw):
    n = 1 << 21
    iq = _stream(fs, n, [(1_000, 60.0)], seed=3)
    chunk = -(-(bw * 100 // 1000) // 4096) * 4096  # roundUp(bandwidth * RECORDER_FLUSH_INTERVAL / 1000, 4096), recorder.cpp:35
    assert chunk == 4096
    t_start = 1_700_000_000_000

    def t0(k):
        return t_start + (k * 1000) // fs

    results = []
    for sizes in ([131_072], [1, 4_000, 77_777, 100_000, 9]):
        bank = b2s.RecorderBank(engine, fs, bw, 2, max_samples_per_push=n)
        bank.start(1, 0)  # no rotation: the bytes do not depend on how the stream is split
        stream, chunks = [], []
        for i, (k, m) in enumerate(_pieces(n, sizes)):
            stream.append(bank.push(iq[2 * k : 2 * (k + m)], t0(k))[1])
            if i % 3 == 1:
                chunks += bank.flush(1)
        chunks += bank.flush(1)
        stream = np.concatenate(stream)
        assert len(chunks) == len(stream) // (2 * chunk) >= 8
        assert np.array_equal(np.concatenate([c for _, c in chunks]), stream[: 2 * chunk * len(chunks)])
        assert [t for t, _ in chunks] == [_chunk_time(t_start, j, chunk, bw) for j in range(len(chunks))]
        assert bank.flush(0) == []  # the idle channel holds nothing
        results.append((stream, chunks))
        bank.close()
    (s0, c0), (s1, c1) = results
    assert np.array_equal(s0, s1)
    assert [t for t, _ in c0] == [t for t, _ in c1] and all(np.array_equal(a, b) for (_, a), (_, b) in zip(c0, c1))

    # consume=0 leaves the chunks in place; stop drops everything held, including the incomplete tail
    bank = b2s.RecorderBank(engine, fs, bw, 1, max_samples_per_push=n)
    bank.start(0, 250_000)
    out = bank.push(iq[: 2 * 600_000], 5_000)[0]
    peek = bank.flush(0, consume=False)
    assert len(peek) == len(out) // (2 * chunk) >= 2
    again = bank.flush(0, cap=1)
    assert len(again) == 1 and again[0][0] == peek[0][0] and np.array_equal(again[0][1], peek[0][1])
    rest = bank.flush(0)
    assert [t for t, _ in rest] == [t for t, _ in peek[1:]] == [_chunk_time(5_000, j, chunk, bw) for j in range(1, len(peek))]
    assert len(out) % (2 * chunk) != 0  # a tail is held
    bank.stop(0)
    assert bank.flush(0) == []
    bank.start(0, 250_000)  # a new recording: chunk 0 again, stamped from its own first push
    out = bank.push(iq[2 * 600_000 : 2 * 1_200_000], 9_000)[0]
    again = bank.flush(0)
    assert len(again) == len(out) // (2 * chunk) and again[0][0] == _chunk_time(9_000, 0, chunk, bw)
    assert np.array_equal(again[0][1], out[: 2 * chunk])
    bank.close()


# ---- 5. errors ----
def _rc_push(bank, iq, cap):
    n_out = np.zeros(bank.n_channels, np.uint64)
    out = np.empty((bank.n_channels, 2 * max(cap, 1)), np.int8)
    return b2s.lib().b2s_recorder_bank_push(bank._h, iq.ctypes.data_as(C.c_void_p), iq.size // 2, 0, out.ctypes.data_as(C.c_void_p), cap, n_out.ctypes.data_as(C.c_void_p))


def test_errors_change_nothing(engine):
    fs, bw, n = 2_048_000, 32_000, 1 << 18
    iq = _stream(fs, n, [(100_000, 50.0)], seed=9)
    bank = b2s.RecorderBank(engine, fs, bw, 3, max_samples_per_push=100_000)
    twin = b2s.RecorderBank(engine, fs, bw, 3, max_samples_per_push=100_000)
    L = b2s.lib()
    h = C.c_void_p()
    for bad in (0, -1):  # n_channels <= 0
        assert L.b2s_recorder_bank_create(engine._h, fs, bw, b2s.IQ_CS8, 1 / 127.0, 0, bad, 0, C.byref(h)) == -1 and not h.value
    for k in (bank, twin):
        k.start(0, 100_000)
        k.start(2, -50_000)
    pieces = _pieces(n, [50_000, 3_001])
    for i, (k, m) in enumerate(pieces):
        x = iq[2 * k : 2 * (k + m)]
        if i == 1:
            assert L.b2s_recorder_bank_start(bank._h, 3, 0) == -1 and L.b2s_recorder_bank_start(bank._h, -1, 0) == -1  # channel out of range
            assert L.b2s_recorder_bank_stop(bank._h, 3) == -1
            assert L.b2s_recorder_bank_flush(bank._h, 7, None, None, 0, 0, None, None) == -1
            assert L.b2s_recorder_bank_start(bank._h, 0, 12_345) == -5  # already recording
            assert L.b2s_recorder_bank_stop(bank._h, 1) == -5  # idle
            assert _rc_push(bank, x, m * bw // fs - 2) == -1  # cap too small
            big = np.zeros(2 * 100_001, np.int8)
            assert _rc_push(bank, big, 100_000) == -1  # more than max_samples_per_push
        a, b = bank.push(x, 10 * i), twin.push(x, 10 * i)
        assert all(np.array_equal(u, v) for u, v in zip(a, b)), i
    assert [(t, c.tobytes()) for t, c in bank.flush(0)] == [(t, c.tobytes()) for t, c in twin.flush(0)]
    bank.close()
    twin.close()


# ---- 6. the reference's loop end to end: band -> mailbox -> scan policy -> bank ----
def test_scan_policy_drives_the_bank(engine):
    import torch

    import __graft_entry__ as ge

    synth = ge.load_synth()
    n, fs, learn, frames, per = 8192, 2_048_000, 40, 40 + 25 * 14, 25  # 25 frames = 100 ms per chunk
    step = fs / n
    tones = [
        synth.Tone(bin_offset=0.31 * n / 2 + 0.1, amplitude=60.0, on_frames=[(65, 250)], fm_dev_bins=6.0),
        synth.Tone(bin_offset=-0.62 * n / 2 + 0.1, amplitude=60.0, on_frames=[(90, 170), (240, 360)], fm_dev_bins=6.0),
        synth.Tone(bin_offset=0.055 * n / 2 + 0.1, amplitude=50.0, on_frames=[(115, 300)], phase=1.0, fm_dev_bins=5.0),
    ]
    iq = synth.make_iq_int8(n, frames, tones, seed=synth.seed_for(0, 6), quiet_frames=learn)
    dev = torch.from_numpy(iq).cuda()
    torch.cuda.synchronize()
    period = synth.frame_period_ms(n, fs)
    cfg = b2s.make_config(n, fs, learn_frames=learn, min_time_ms=100, timeout_ms=200, flags=b2s.FLAG_IQ_ON_DEVICE)
    band = b2s.Band(engine, cfg)
    n_rec = 4
    pol = b2s.ScanPolicy([(cfg.center_hz - 1_000_000, cfg.center_hz + 1_000_000)], fs, n_rec, 500)
    assert len(pol.ranges()) == 1  # one range: the scanner never retunes
    pol.begin(0)
    bank = b2s.RecorderBank(engine, fs, 32_000, n_rec, on_device=True, max_samples_per_push=per * n)
    recs = [b2s.Recorder(engine, fs, 32_000, on_device=True, max_samples_per_push=per * n) for _ in range(n_rec)]
    shift_of = [None] * n_rec
    seen = {i: [] for i in range(len(tones))}  # tone -> chunks in which a channel recorded it
    n_chunks = (frames - learn) // per
    flushed = 0
    for k in range(n_chunks - 1):
        f0 = learn + k * per if k else 0
        nf = learn + per if k == 0 else per
        t0 = int(f0 * period)
        out = band.push_raw(dev.data_ptr() + 2 * n * f0, nf, t0, period)
        mailbox = [(t.shift_hz, t.flush) for t in out.transmissions[: out.n_transmissions]]
        acts, hop = pol.notify(int((f0 + nf) * period), mailbox)
        assert hop is None
        for kind, r, shift, _ in acts:
            if kind == b2s.REC_START:
                bank.start(r, shift)
                recs[r].start(shift)
                shift_of[r] = shift
            elif kind == b2s.REC_STOP:
                bank.stop(r)
                recs[r].stop()
                shift_of[r] = None
            elif kind == b2s.REC_FLUSH:
                flushed += len(bank.flush(r))
        g0 = f0 + nf  # chunk k + 1, from the same device pointer
        outs = bank.push(dev.data_ptr() + 2 * n * g0, int(g0 * period), n_samples=per * n)
        for r in range(n_rec):
            if shift_of[r] is None:
                assert len(outs[r]) == 0
                continue
            want = recs[r].push(dev.data_ptr() + 2 * n * g0, per * n)
            assert np.array_equal(outs[r], want), (k, r)
            # a live carrier inside this channel's band: the spectrum's centre of mass sits at its residual offset from the shift
            for ti, t in enumerate(tones):
                f_hz = t.bin_offset * step
                if abs(f_hz - shift_of[r]) < 8_000 and all(synth.tone_active(t, f) for f in range(g0, g0 + per)):
                    z = outs[r][0::2].astype(np.float64) + 1j * outs[r][1::2].astype(np.float64)
                    spec = np.abs(np.fft.fftshift(np.fft.fft(z))) ** 2
                    f = np.fft.fftshift(np.fft.fftfreq(len(z), 1 / 32_000))
                    near = np.abs(f - f[np.argmax(spec)]) < 4_000
                    centroid = float(np.sum(f[near] * spec[near]) / np.sum(spec[near]))
                    assert abs(centroid - (f_hz - shift_of[r])) < 400, (k, r, centroid, f_hz - shift_of[r])
                    seen[ti].append(k)
    for ti, t in enumerate(tones):  # every carrier got a channel while it was live
        for a, b in t.on_frames:
            live_chunks = [k for k in range(n_chunks - 1) if a + 2 * per <= learn + (k + 1) * per and learn + (k + 2) * per <= b]
            assert not live_chunks or set(live_chunks) & set(seen[ti]), (ti, (a, b), seen[ti])
    assert flushed > 0
    bank.close()
    for r in recs:
        r.close()
    band.close()
