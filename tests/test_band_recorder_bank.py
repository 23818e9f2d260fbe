"""A recorder bank attached to a band (b2s_band_attach_recorder_bank): one upload of each push feeds the band and the bank.

Every comparison is byte for byte. The bank must equal a stand-alone b2s_recorder_bank fed the same samples, cut where include/b2s.h
says (each band push, and every max_frames_per_push frames within one), and the band must equal a twin band without a bank."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from conftest import ROOT, load_b2s

b2s = load_b2s()
gpu = pytest.mark.gpu

N, FS, BW, LEARN, MAX_FRAMES = 2048, 2_048_000, 32_000, 30, 600
SHIFTS = [317_500, -635_000, 55_000, -200_000]
# push index -> (channels started, channels stopped) before it: two channels record from the start, one starts and one stops later
SCHEDULE = {0: ([0, 1], []), 1: ([2], [0]), 3: ([3, 0], [])}
PATTERNS = {
    "pipelined": ([520, 40, 600], 1000),  # >= 512 frames: the synchronous host path copies the push in four pipeline chunks
    "uneven": ([1, 7, 33, 100, 3, 64, 250, 17], 1000),
    # longer than max_frames_per_push: the bank sees pieces of 600, 600 and 100 frames; channels start before pushes of 1250 and 1300
    "long": ([1300, 1250, 30, 1300], 1000),
    "emit_cut": ([200, 50], 1),  # a spectrogram row every frame or two: the band cuts the push at 16 rows
}
MODES = {  # name -> (on_device, iq_format, flags)
    "host_cs8_sync": (False, b2s.IQ_CS8, 0),
    "host_cs8_async": (False, b2s.IQ_CS8, b2s.FLAG_ASYNC),
    "host_cf32_sync": (False, b2s.IQ_CF32, 0),
    "device_cs8_sync": (True, b2s.IQ_CS8, 0),
    "device_cs8_async": (True, b2s.IQ_CS8, b2s.FLAG_ASYNC),
}


def test_binding_matches_the_header():
    """b2s.py declares b2s_band_attach_recorder_bank as include/b2s.h does: (band*, bank*) -> int."""
    header = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "b2s.h")).read(), flags=re.S)
    m = re.search(r"\bint\s+b2s_band_attach_recorder_bank\s*\(([^)]*)\)\s*;", header)
    assert m, "b2s_band_attach_recorder_bank is not declared"
    params = [p.strip() for p in m.group(1).split(",")]
    assert [re.sub(r"\s+", "", p).rsplit("*", 1)[0] + "*" for p in params] == ["b2s_band*", "b2s_recorder_bank*"]
    if not os.path.exists(b2s.LIB_PATH):
        pytest.skip("libb2s.so not built; run __graft_entry__.build()")
    f = b2s.lib().b2s_band_attach_recorder_bank
    assert f.argtypes == [C.c_void_p, C.c_void_p] and f.restype == C.c_int
    assert callable(getattr(b2s.Band, "attach_recorder_bank", None))


# ---- helpers ----
class Stream:
    """One IQ stream of whole frames (stride = N * r samples), as host arrays and, on request, on the device."""

    def __init__(self, frames, r, fmt, on_device, seed=5):
        import __graft_entry__ as ge

        synth = ge.load_synth()
        self.r, self.stride, self.fmt, self.on_device = r, N * r, fmt, on_device
        self.period = synth.frame_period_ms(N, FS, r)
        iq8 = synth.make_iq_int8(N, frames, synth.standard_scene(N, frames, LEARN), seed=seed, quiet_frames=LEARN, stride=self.stride)
        self.host = iq8 if fmt == b2s.IQ_CS8 else (iq8.astype(np.float32) * np.float32(1 / 127.0))
        self.bps = 2 * self.host.itemsize
        if on_device:
            import torch

            self.dev = torch.from_numpy(self.host.copy()).cuda()
            torch.cuda.synchronize()

    def band_ptr(self, f0):
        base = self.dev.data_ptr() if self.on_device else self.host.ctypes.data
        return base + f0 * self.stride * self.bps

    def samples(self, f0, nf):
        return self.host[2 * f0 * self.stride : 2 * (f0 + nf) * self.stride]

    def t0(self, f0):
        return 1_000 + int(f0 * self.period)


def band_config(stream, flags, interval_ms=1000):
    cfg = b2s.make_config(N, FS, decimator=stream.r, iq_format=stream.fmt, learn_frames=LEARN, min_time_ms=50, timeout_ms=100,
                          max_frames_per_push=MAX_FRAMES, flags=flags | (b2s.FLAG_IQ_ON_DEVICE if stream.on_device else 0))
    cfg.spectrogram_interval_ms = interval_ms
    return cfg


def new_bank(engine, stream, **kw):
    kw.setdefault("max_samples_per_push", MAX_FRAMES * stream.stride)
    return b2s.RecorderBank(engine, FS, BW, len(SHIFTS), iq_format=stream.fmt, **kw)


def feed_standalone(bank, stream, f0, nf):
    """What an attached bank must see of one band push: pieces of up to MAX_FRAMES frames, piece j stamped like frame j * MAX_FRAMES."""
    for j in range(0, nf, MAX_FRAMES):
        bank.push(stream.samples(f0 + j, min(MAX_FRAMES, nf - j)), stream.t0(f0) + int(np.floor(j * stream.period + 0.5)))


def flushed(bank, channel):
    return [(t, c.tobytes()) for t, c in bank.flush(channel, cap=4096)]


def start_push(band, stream, f0, nf):
    """b2s_band_push of frames [f0, f0 + nf); the result of a synchronous band, None for an asynchronous one."""
    return band.push_raw(stream.band_ptr(f0), nf, stream.t0(f0), stream.period)


def summary(band, res):
    """(mailbox, live transmissions, n_detect_entries, n_spectrogram_rows) of a push; b2s_band_sync collects an asynchronous one."""
    res = res if res is not None else band.sync()
    tx = [(t.shift_hz, t.flush, t.key, t.power) for t in res.transmissions[: res.n_transmissions]]
    return tx, res.n_transmissions_total, res.n_detect_entries, res.n_spectrogram_rows


def push_band(band, stream, f0, nf):
    return summary(band, start_push(band, stream, f0, nf))


def band_state(band):
    s, a, ring, frames = band.get_averager()
    thr, samples, ready = band.get_noise()
    times, centers, rows = band.get_spectrogram(cap=4096)
    keys, first, last, power = band.get_signals(cap=256)
    return [band.get_transmissions(), keys, first, last, power, s, a, ring, frames, thr, samples, ready, times, centers, rows]


def assert_same_band(a, b, where):
    for i, (x, y) in enumerate(zip(band_state(a), band_state(b))):
        if isinstance(x, np.ndarray):
            assert x.shape == y.shape and x.tobytes() == y.tobytes(), (where, i)
        else:
            assert x == y, (where, i)


def apply_schedule(p, banks):
    started, stopped = SCHEDULE.get(p, ([], []))
    for k in banks:
        for c in stopped:
            k.stop(c)
        for c in started:
            k.start(c, SHIFTS[c])


# ---- 1 + 2: the bank equals a stand-alone bank, the band equals its twin ----
@gpu
@pytest.mark.parametrize("pattern", sorted(PATTERNS))
@pytest.mark.parametrize("r", [1, 3])
@pytest.mark.parametrize("mode", list(MODES))
def test_attached_bank_equals_standalone_and_band_equals_twin(engine, mode, r, pattern):
    on_device, fmt, flags = MODES[mode]
    sizes, interval = PATTERNS[pattern]
    stream = Stream(sum(sizes), r, fmt, on_device)
    band, twin = b2s.Band(engine, band_config(stream, flags, interval)), b2s.Band(engine, band_config(stream, flags, interval))
    bank, alone = new_bank(engine, stream), new_bank(engine, stream, on_device=False)
    band.attach_recorder_bank(bank)
    f0, rows, total = 0, 0, 0
    for p, nf in enumerate(sizes):
        apply_schedule(p, (bank, alone))
        res = start_push(band, stream, f0, nf)
        feed_standalone(alone, stream, f0, nf)
        got = flushed(bank, 1)
        assert got == flushed(alone, 1), p  # an asynchronous band's push is settled by the next call on its bank
        total += len(got)
        got, want = summary(band, res), push_band(twin, stream, f0, nf)
        assert got == want, (p, got[1:], want[1:])
        rows += got[3]
        assert_same_band(band, twin, p)
        f0 += nf
    for c in range(len(SHIFTS)):
        got, want = flushed(bank, c), flushed(alone, c)
        assert got == want, c
        total += len(got)
    assert total > 0
    if pattern == "emit_cut":
        assert rows > 16  # the band did cut the first push at the spectrogram emission limit
    band.close()
    for x in (twin, bank, alone):
        x.close()


@gpu
def test_dense_rows_are_unchanged(engine):
    stream = Stream(560, 3, b2s.IQ_CS8, False)
    band, twin = b2s.Band(engine, band_config(stream, 0)), b2s.Band(engine, band_config(stream, 0))
    bank = new_bank(engine, stream)
    bank.start(0, SHIFTS[0])
    band.attach_recorder_bank(bank)
    f0 = 0
    for nf in (520, 40):
        x = stream.samples(f0, nf)
        a = band.push(x, nf, stream.t0(f0), stream.period, per_frame=True, dense=("psd_db",))
        b = twin.push(x, nf, stream.t0(f0), stream.period, per_frame=True, dense=("psd_db",))
        assert a.psd_db.tobytes() == b.psd_db.tobytes()
        assert a.frame_tx == b.frame_tx and a.transmissions == b.transmissions and a.n_detect_entries == b.n_detect_entries
        assert_same_band(band, twin, f0)
        f0 += nf
    assert len(flushed(bank, 0)) > 0
    band.close()
    twin.close()
    bank.close()



# ---- device input reused in the band's stream order ----
@gpu
@pytest.mark.parametrize("flags", [0, b2s.FLAG_ASYNC])
def test_device_input_rewritten_on_the_band_stream_after_each_push(engine, flags):
    """The caller writes the next push into the same device buffer on the band's stream as soon as b2s_band_push returns: the bank
    must still have read the previous samples, as K1 has."""
    import torch

    sizes = [600, 1300, 37, 600, 1250]
    stream = Stream(sum(sizes), 3, b2s.IQ_CS8, True)
    band, twin = b2s.Band(engine, band_config(stream, flags)), b2s.Band(engine, band_config(stream, flags))
    bank, alone = new_bank(engine, stream), new_bank(engine, stream)
    for k in (bank, alone):
        for c in range(len(SHIFTS)):
            k.start(c, SHIFTS[c])
    band.attach_recorder_bank(bank)
    ts = torch.cuda.Stream()
    band.set_stream(ts.cuda_stream)
    buf = torch.empty(2 * max(sizes) * stream.stride, dtype=torch.int8, device="cuda")
    f0 = 0
    with torch.cuda.stream(ts):
        for nf in sizes:
            n = 2 * nf * stream.stride
            buf[:n].copy_(stream.dev[2 * f0 * stream.stride : 2 * (f0 + nf) * stream.stride])
            band.push_raw(buf.data_ptr(), nf, stream.t0(f0), stream.period)
            buf.fill_(0)  # overwrites the push's input on the band's stream at once
            feed_standalone(alone, stream, f0, nf)
            f0 += nf
    if flags:
        band.sync()
    torch.cuda.synchronize()
    f0 = 0
    for nf in sizes:
        push_band(twin, stream, f0, nf)
        f0 += nf
    assert_same_band(band, twin, "end")
    for c in range(len(SHIFTS)):
        want = flushed(alone, c)
        assert len(want) > 3 and flushed(bank, c) == want, c
    for x in (band, twin, bank, alone):
        x.close()


@gpu
@pytest.mark.parametrize("on_device", [False, True])
def test_failed_synchronous_pushes_still_feed_the_bank_once(engine, on_device):
    """A push that overflows detect_capacity completes and then fails, leaving the bank's piece unsettled; the next push settles it
    before it launches the bank again."""
    stream = Stream(600, 1, b2s.IQ_CS8, on_device)
    cfg = [band_config(stream, 0) for _ in range(2)]
    for c in cfg:
        c.detect_capacity = 8
    band, twin = b2s.Band(engine, cfg[0]), b2s.Band(engine, cfg[1])
    bank, alone = new_bank(engine, stream), new_bank(engine, stream)
    for k in (bank, alone):
        k.start(0, SHIFTS[0])
        k.start(1, SHIFTS[1])
    band.attach_recorder_bank(bank)

    def outcome(b, f0, nf):
        try:
            b.push_raw(stream.band_ptr(f0), nf, stream.t0(f0), stream.period)
            return 0
        except b2s.B2SError as e:
            return str(e).split(":")[0]

    failed = 0
    for f0 in range(0, 600, 100):
        got = outcome(band, f0, 100)
        assert got == outcome(twin, f0, 100), f0
        failed += got != 0
        feed_standalone(alone, stream, f0, 100)
    assert failed > 0
    assert_same_band(band, twin, "end")
    for c in (0, 1):
        want = flushed(alone, c)
        assert len(want) > 3 and flushed(bank, c) == want, c
    for x in (band, twin, bank, alone):
        x.close()


# ---- 3: the closed loop mailbox -> scan policy -> bank -> next push ----
@gpu
def test_closed_loop_equals_the_two_call_recipe(engine):
    import torch

    import __graft_entry__ as ge

    synth = ge.load_synth()
    n, fs, learn, frames, per = 8192, 2_048_000, 40, 40 + 25 * 14, 25
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
    cfg = b2s.make_config(n, fs, learn_frames=learn, min_time_ms=100, timeout_ms=200, flags=b2s.FLAG_IQ_ON_DEVICE, max_frames_per_push=learn + per)
    n_rec = 4
    runs = []
    for attached in (False, True):
        band = b2s.Band(engine, cfg)
        bank = b2s.RecorderBank(engine, fs, 32_000, n_rec, on_device=True, max_samples_per_push=(learn + per) * n)
        if attached:
            band.attach_recorder_bank(bank)
        pol = b2s.ScanPolicy([(cfg.center_hz - 1_000_000, cfg.center_hz + 1_000_000)], fs, n_rec, 500)
        pol.begin(0)
        shift_of = [None] * n_rec
        log, outs = [], []
        for k in range((frames - learn) // per):
            f0 = learn + k * per if k else 0
            nf = learn + per if k == 0 else per
            t0 = int(f0 * period)
            res = band.push_raw(dev.data_ptr() + 2 * n * f0, nf, t0, period)
            if not attached:  # the recipe without the attachment: the same samples again, to the bank
                outs.append((f0, nf, list(shift_of), bank.push(dev.data_ptr() + 2 * n * f0, t0, n_samples=nf * n)))
            mailbox = [(t.shift_hz, t.flush) for t in res.transmissions[: res.n_transmissions]]
            acts, hop = pol.notify(int((f0 + nf) * period), mailbox)
            assert hop is None
            log.append(("acts", k, acts))
            for kind, r, shift, _ in acts:
                if kind == b2s.REC_START:
                    bank.start(r, shift)
                    shift_of[r] = shift
                elif kind == b2s.REC_STOP:
                    bank.stop(r)
                    shift_of[r] = None
                elif kind == b2s.REC_FLUSH:
                    log.append(("flush", k, r, flushed(bank, r)))
        log += [("end", r, flushed(bank, r)) for r in range(n_rec)]
        runs.append((log, outs))
        bank.close()
        band.close()
    (recipe, outs), (attached_log, _) = runs
    assert attached_log == recipe
    assert sum(len(e[3]) for e in recipe if e[0] == "flush") > 0
    # each live carrier lands in a channel (the recipe's bytes, which the attached bank's chunks equal)
    seen = {i: [] for i in range(len(tones))}
    for k, (f0, nf, shifts, out) in enumerate(outs):
        for r, s in enumerate(shifts):
            if s is None:
                assert len(out[r]) == 0
                continue
            for ti, t in enumerate(tones):
                f_hz = t.bin_offset * step
                if abs(f_hz - s) < 8_000 and all(synth.tone_active(t, f) for f in range(f0, f0 + nf)):
                    z = out[r][0::2].astype(np.float64) + 1j * out[r][1::2].astype(np.float64)
                    spec = np.abs(np.fft.fftshift(np.fft.fft(z))) ** 2
                    f = np.fft.fftshift(np.fft.fftfreq(len(z), 1 / 32_000))
                    near = np.abs(f - f[np.argmax(spec)]) < 4_000
                    centroid = float(np.sum(f[near] * spec[near]) / np.sum(spec[near]))
                    assert abs(centroid - (f_hz - s)) < 400, (k, r, centroid, f_hz - s)
                    seen[ti].append(k)
    n_chunks = (frames - learn) // per
    for ti, t in enumerate(tones):
        for a, b in t.on_frames:
            live = [k for k in range(1, n_chunks) if a + 2 * per <= learn + k * per and learn + (k + 1) * per <= b]
            assert not live or set(live) & set(seen[ti]), (ti, (a, b), seen[ti])


# ---- 4: one upload ----
@gpu
@pytest.mark.parametrize("mode", ["host_cs8_sync", "host_cs8_async", "host_cf32_sync"])
def test_one_upload_per_push(engine, mode):
    on_device, fmt, flags = MODES[mode]
    sizes = [520, 13, 1300]
    stream = Stream(sum(sizes), 3, fmt, on_device)
    band = b2s.Band(engine, band_config(stream, flags))
    bank = new_bank(engine, stream)
    bank.start(2, SHIFTS[2])
    band.attach_recorder_bank(bank)
    band.get_profile(reset=True)
    f0 = 0
    for nf in sizes:
        push_band(band, stream, f0, nf)
        assert band.get_profile(reset=True).h2d_bytes == nf * stream.stride * stream.bps, nf
        f0 += nf
    band.close()
    bank.close()


# ---- 5: refusals change nothing ----
@gpu
def test_refusals_change_nothing(engine):
    stream = Stream(700, 3, b2s.IQ_CS8, False)
    L = b2s.lib()
    band, twin = b2s.Band(engine, band_config(stream, 0)), b2s.Band(engine, band_config(stream, 0))
    other_band = b2s.Band(engine, band_config(stream, 0))
    other_engine = b2s.Engine(0)
    need = MAX_FRAMES * stream.stride
    refused = [
        b2s.RecorderBank(engine, FS // 2, BW, 4, max_samples_per_push=need),  # rate
        b2s.RecorderBank(engine, FS, BW, 4, iq_format=b2s.IQ_CF32, max_samples_per_push=need),  # format
        b2s.RecorderBank(engine, FS, BW, 4, iq_scale=1 / 128.0, max_samples_per_push=need),  # scale
        b2s.RecorderBank(engine, FS, BW, 4, max_samples_per_push=need - 1),  # too small for a full push
        b2s.RecorderBank(other_engine, FS, BW, 4, max_samples_per_push=need),  # another engine
    ]
    elsewhere = new_bank(engine, stream)
    other_band.attach_recorder_bank(elsewhere)
    bank, alone, second = new_bank(engine, stream), new_bank(engine, stream), new_bank(engine, stream)
    for k in refused + [elsewhere]:
        assert L.b2s_band_attach_recorder_bank(band._h, k._h) == -1
    band.attach_recorder_bank(bank)
    assert L.b2s_band_attach_recorder_bank(band._h, second._h) == -1  # a second bank
    assert L.b2s_band_attach_recorder_bank(other_band._h, bank._h) == -1  # already attached
    for k in (bank, alone, elsewhere):
        k.start(0, SHIFTS[0])
        k.start(3, SHIFTS[3])
    f0 = 0
    for nf in (300, 400):
        got = push_band(band, stream, f0, nf)
        assert got == push_band(twin, stream, f0, nf)
        push_band(other_band, stream, f0, nf)
        feed_standalone(alone, stream, f0, nf)
        assert_same_band(band, twin, f0)
        f0 += nf
    for c in (0, 3):
        want = flushed(alone, c)
        assert len(want) > 0 and flushed(bank, c) == want and flushed(elsewhere, c) == want
        assert flushed(second, c) == []
    for x in [band, twin, other_band, bank, alone, second, elsewhere] + refused:
        x.close()
    other_engine.close()


# ---- 6: lifetimes ----
@gpu
def test_destroying_the_attached_bank_leaves_the_band_as_its_twin(engine):
    stream = Stream(400, 1, b2s.IQ_CS8, False)
    for flags in (0, b2s.FLAG_ASYNC):
        band, twin = b2s.Band(engine, band_config(stream, flags)), b2s.Band(engine, band_config(stream, flags))
        bank = new_bank(engine, stream)
        bank.start(1, SHIFTS[1])
        band.attach_recorder_bank(bank)
        assert push_band(band, stream, 0, 150) == push_band(twin, stream, 0, 150)
        bank.close()
        assert band._bank is None
        for f0, nf in ((150, 120), (270, 130)):
            assert push_band(band, stream, f0, nf) == push_band(twin, stream, f0, nf)
            assert_same_band(band, twin, f0)
        band.close()
        twin.close()


@gpu
@pytest.mark.parametrize("how", ["detach", "destroy_band"])
@pytest.mark.parametrize("flags", [0, b2s.FLAG_ASYNC])
def test_recording_continues_stand_alone(engine, how, flags):
    stream = Stream(900, 3, b2s.IQ_CS8, True)
    band = b2s.Band(engine, band_config(stream, flags))
    bank, alone = new_bank(engine, stream), new_bank(engine, stream)
    for k in (bank, alone):
        k.start(0, SHIFTS[0])
        k.start(2, SHIFTS[2])
    band.attach_recorder_bank(bank)
    f0 = 0
    for nf in (333, 250):
        band.push_raw(stream.band_ptr(f0), nf, stream.t0(f0), stream.period)
        feed_standalone(alone, stream, f0, nf)
        f0 += nf
    if how == "detach":
        band.attach_recorder_bank(None)
        assert bank._band is None and band._bank is None
        push_band(band, stream, f0, 50)  # the band goes on without the bank
    else:
        band.close()
    for k in (bank, alone):
        for j in range(f0, 900, 200):
            k.push(stream.samples(j, min(200, 900 - j)), stream.t0(j))
    for c in (0, 2):
        want = flushed(alone, c)
        assert len(want) > 3 and flushed(bank, c) == want, c
    for x in (band, bank, alone):
        x.close()


@gpu
@pytest.mark.parametrize("bank_first", [False, True])
def test_python_objects_close_in_either_order(engine, bank_first):
    stream = Stream(100, 1, b2s.IQ_CS8, False)
    band, bank = b2s.Band(engine, band_config(stream, b2s.FLAG_ASYNC)), new_bank(engine, stream)
    bank.start(0, SHIFTS[0])
    band.attach_recorder_bank(bank)
    assert band._bank is bank and bank._band() is band
    band.push_raw(stream.band_ptr(0), 100, stream.t0(0), stream.period)  # left pending on the bank
    first, second = (bank, band) if bank_first else (band, bank)
    first.close()
    assert band._bank is None and bank._band is None and not first._h
    if not bank_first:
        assert bank.flush(0, consume=False) is not None  # the bank stands alone
    second.close()
    assert not band._h and not bank._h
