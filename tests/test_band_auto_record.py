"""Auto-record (b2s_band_set_auto_record): the band drives its attached bank's channels from its own detections.

An auto-recording band is compared, with no tolerance, with a twin band that a caller drives by the manual recipe of INTEGRATION.md:
collect the mailbox after every push, pass it to a b2s_scan_policy with one range and the same channel count, and for each START look
up the transmission's START event, subtract the pre-roll (never below the oldest frame the history still holds) and call
b2s_band_record_from, or b2s_recorder_bank_start when there is no usable history; STOP becomes b2s_recorder_bank_stop. After every push
the actions, every channel's flushed chunks (bytes and times) and the bands' mailboxes, maps and spectrogram rows must be equal."""
import numpy as np
import pytest

from conftest import load_b2s
from test_band_recorder_bank import MODES, band_state, flushed, summary

b2s = load_b2s()
gpu = pytest.mark.gpu
E_INVALID, E_STATE = -1, -5

N, FS, BW, LEARN = 2048, 2_048_000, 32_000, 30
CENTER = 100_000_000
FM_DEV, FM_RATE = 4.0, 3.3


class Scene:
    """Carriers (bin, amplitude, [(first frame, end frame)]) in Gaussian noise, pushed in the given sizes."""

    def __init__(self, tones, pushes, n_ch, hist_frames, sigma=8.0, max_frames=600, rec_bw=32_000, retune_after=(), n_fft=N):
        self.tones, self.pushes, self.n_ch, self.hist_frames, self.n_fft = tones, pushes, n_ch, hist_frames, n_fft
        self.sigma, self.max_frames, self.rec_bw, self.retune_after = sigma, max_frames, rec_bw, set(retune_after)
        self.frames = sum(pushes)


# Two channels for six carriers. Carrier 3 finds no free channel at first (NONE_FREE) and gets one when carrier 2 has timed out, after
# its START frame has left the 331-frame history (the fall-back). Carrier 4 starts and times out inside the push of frames 1000-1349.
# Carrier 5's catch-up straddles the ring's end (frame 4 x 331 = 1324). Carrier 6 starts in the push before the retune after frame
# 1599: an asynchronous band decides after the retune, so its START frame is refused and it falls back.
MAIN = Scene(
    tones=[(300.1, 60.0, [(60, 700)]), (-560.1, 60.0, [(80, 500)]), (50.1, 40.0, [(100, 900)]), (-200.1, 60.0, [(1010, 1050)]),
           (620.1, 60.0, [(1300, 2000)]), (-820.1, 60.0, [(1520, 2200)])],
    pushes=[150, 250, 400, 200, 350, 250, 250, 300, 250], n_ch=2, hist_frames=331, retune_after=[5])


def batch_scene(k):
    """k carriers 28 kHz apart that all start in the second push, each at its own frame, on k channels: one decision starts every
    channel, and the catch-ups (pieces of 64 frames from each channel's own start, the ring ending at frame 253) have different lengths."""
    tones = [(-1932.1 + 56 * i, 3.5, [(110 + (7 * i) % 120, 300)]) for i in range(k)]
    return Scene(tones, [100, 200], n_ch=k, hist_frames=253, sigma=2.0, max_frames=64, rec_bw=8_000, n_fft=4096)


_IQ = {}  # keyed by the Scene itself, which the key keeps alive, so that no later scene can reuse its id()


def scene_iq(scene, r, fmt):
    key = (scene, r, fmt)
    if key not in _IQ:
        n_fft = scene.n_fft
        stride = n_fft * r
        n = scene.frames * stride
        rng = np.random.default_rng(17)
        z = rng.normal(0, scene.sigma, n) + 1j * rng.normal(0, scene.sigma, n)
        for b, amp, spans in scene.tones:
            for a, e in spans:
                t = np.arange(a * stride, e * stride, dtype=np.float64)
                z[a * stride : e * stride] += amp * np.exp(1j * (2 * np.pi * b / n_fft * t + FM_DEV / FM_RATE * np.sin(2 * np.pi * FM_RATE * t / n_fft)))
        x = np.empty(2 * n, np.float64)
        x[0::2], x[1::2] = z.real, z.imag
        x8 = np.clip(np.rint(x), -127, 127).astype(np.int8)
        _IQ[key] = x8 if fmt == b2s.IQ_CS8 else x8.astype(np.float32) * np.float32(1 / 127.0)
    return _IQ[key]


class Run:
    """One scene through an auto-recording band and its manually driven twin."""

    def __init__(self, engine, scene, mode, r, preroll, history=True, auto_log=False):
        on_device, fmt, flags = MODES[mode]
        self.scene, self.r, self.preroll, self.stride = scene, r, preroll, scene.n_fft * r
        self.async_ = bool(flags & b2s.FLAG_ASYNC)
        self.period = self.stride * 1000.0 / FS
        self.host = scene_iq(scene, r, fmt)
        self.bps = 2 * self.host.itemsize
        if on_device:
            import torch

            self.dev = torch.from_numpy(self.host.copy()).cuda()
            torch.cuda.synchronize()
        self.on_device = on_device
        cfg = b2s.make_config(scene.n_fft, FS, CENTER, decimator=r, iq_format=fmt, learn_frames=LEARN, min_time_ms=50, timeout_ms=100, recording_bandwidth_hz=scene.rec_bw,
                              max_frames_per_push=scene.max_frames, detect_capacity=2048, flags=flags | (b2s.FLAG_IQ_ON_DEVICE if on_device else 0))
        self.auto, self.twin = b2s.Band(engine, cfg), b2s.Band(engine, cfg)
        self.abank, self.tbank = [b2s.RecorderBank(engine, FS, BW, scene.n_ch, iq_format=fmt, max_samples_per_push=scene.max_frames * self.stride) for _ in range(2)]
        if history:
            for k in (self.abank, self.tbank):
                k.set_history(scene.hist_frames * self.stride)
        self.history = history
        self.auto.attach_recorder_bank(self.abank)
        self.twin.attach_recorder_bank(self.tbank)
        self.auto.set_auto_record(True, preroll)
        self.auto_log = auto_log
        if auto_log:
            self.auto.set_event_log(True)
        self.twin.set_event_log(True)
        self.policy = b2s.ScanPolicy([(CENTER - 1_000_000, CENTER + 1_000_000)], FS, scene.n_ch, 500)  # one range: no hop
        self.keys = [0] * scene.n_ch
        self.starts = {}  # key -> frame of its latest START event
        self.first_mappable = 0  # frames before the last change of centre are not in the history for record_from
        self.pushes = []
        self.all_actions = []
        self.catch_ups = []  # (from_frame, end frame) of every START from history

    def t0(self, f0):
        return 1_000 + int(f0 * self.period)

    def clock(self, frame):
        for f0, nf in self.pushes:
            if f0 <= frame < f0 + nf:
                return self.t0(f0) + int(np.floor((frame - f0) * self.period + 0.5))
        raise AssertionError(frame)

    def push(self, band, f0, nf):
        base = self.dev.data_ptr() if self.on_device else self.host.ctypes.data
        return band.push_raw(base + f0 * self.stride * self.bps, nf, self.t0(f0), self.period)

    def oldest_frame(self):
        if not self.history:
            return None
        o, e = self.tbank.history()
        f = max(-(-o // self.stride), self.first_mappable)
        return f if f < e // self.stride else None

    def manual_decision(self, frame, time_ms):
        """The INTEGRATION.md recipe on the twin: what the auto-recording band must have done."""
        self.events = self.twin.get_events()
        for kind, key, _, ev_frame, _, _, _ in self.events:
            if kind == b2s.EV_START:
                self.starts[key] = ev_frame
        mailbox = self.twin.get_transmissions()
        acts, hop = self.policy.notify(time_ms, [(s, f) for s, f, _, _ in mailbox])
        assert hop is None
        out = []
        at = 0  # the actions other than STOP follow the list: each acts on the next entry with its shift (a FLUSH: with flush set)
        for kind, ch, shift, duration in acts:
            if kind == b2s.REC_STOP:
                key = self.keys[ch]
            else:
                while mailbox[at][0] != shift or (kind == b2s.REC_FLUSH and not mailbox[at][1]):
                    at += 1
                key = mailbox[at][2]
                at += 1
            from_frame, t = -1, time_ms
            if kind == b2s.REC_STOP:
                self.tbank.stop(ch)
            elif kind == b2s.REC_START:
                self.keys[ch] = key
                f, oldest = self.starts.get(key), self.oldest_frame()
                if f is not None and oldest is not None and f >= oldest:
                    from_frame = max(f - self.preroll, oldest)
                    t = self.clock(from_frame)
                    self.twin.record_from(ch, shift, from_frame)
                    self.catch_ups.append((from_frame, frame + 1))
                else:
                    self.tbank.start(ch, shift)
            out.append((kind, ch, shift, key, frame, from_frame, t, duration))
        return out

    def retune(self, f_end):
        for b in (self.auto, self.twin):
            b.set_center(CENTER + 100_000, CENTER + 100_000 - FS // 2, CENTER + 100_000 + FS // 2)
        self.first_mappable = f_end

    def check(self, f0, nf, ra, rt):
        assert summary(self.auto, ra) == summary(self.twin, rt), f0
        want = self.manual_decision(f0 + nf - 1, self.clock(f0 + nf - 1))
        assert self.auto.auto_record_actions() == want, f0
        self.all_actions += want
        for i, (a, b) in enumerate(zip(band_state(self.auto), band_state(self.twin))):
            assert (a.tobytes() == b.tobytes()) if isinstance(a, np.ndarray) else a == b, (f0, i)
        for c in range(self.scene.n_ch):
            assert flushed(self.abank, c) == flushed(self.tbank, c), (f0, c)

    def run(self):
        f0 = 0
        for i, nf in enumerate(self.scene.pushes):
            ra, rt = self.push(self.auto, f0, nf), self.push(self.twin, f0, nf)
            self.pushes.append((f0, nf))
            if self.async_ and i in self.scene.retune_after:  # the auto band decides in b2s_band_sync, after the retune
                self.retune(f0 + nf)
            self.check(f0, nf, ra, rt)
            if not self.async_ and i in self.scene.retune_after:  # the auto band decided inside its push
                self.retune(f0 + nf)
            assert self.auto.get_events() == (self.events if self.auto_log else []), f0
            f0 += nf
        return self

    def close(self):
        for x in (self.auto, self.twin, self.abank, self.tbank, self.policy):
            x.close()


def kinds(actions, kind):
    return [a for a in actions if a[0] == kind]


@gpu
@pytest.mark.parametrize("preroll", [0, 21])
@pytest.mark.parametrize("r", [1, 3])
@pytest.mark.parametrize("mode", list(MODES))
def test_auto_record_equals_the_manual_recipe(engine, mode, r, preroll):
    run = Run(engine, MAIN, mode, r, preroll).run()
    acts = run.all_actions
    starts = kinds(acts, b2s.REC_START)
    assert any(a[5] >= 0 for a in starts) and any(a[5] == -1 for a in starts), starts
    assert kinds(acts, b2s.REC_STOP) and kinds(acts, b2s.REC_NONE_FREE), acts
    ring = MAIN.hist_frames
    assert any(a // ring != (e - 1) // ring for a, e in run.catch_ups), run.catch_ups  # a catch-up read across the ring's end
    run.close()


@gpu
@pytest.mark.parametrize("mode", ["host_cs8_sync", "device_cs8_async"])
def test_without_history_it_is_the_reference(engine, mode):
    """No history, no pre-roll: every START is b2s_recorder_bank_start, what SdrDevice::updateRecordings does."""
    run = Run(engine, MAIN, mode, 1, 0, history=False).run()
    starts = kinds(run.all_actions, b2s.REC_START)
    assert len(starts) >= 4 and all(a[5] == -1 for a in starts)
    run.close()


@gpu
@pytest.mark.parametrize("k", [3, 70])
def test_one_decision_starts_many_channels_together(engine, k):
    """k channels started by one decision catch up in shared launches (70 > the 64 channels of one launch); each equals a sequential
    b2s_band_record_from on the twin's bank, pieces that straddle the ring's end included."""
    scene = batch_scene(k)
    run = Run(engine, scene, "host_cs8_sync", 1, 21).run()
    starts = kinds(run.all_actions, b2s.REC_START)
    assert len(starts) == k and len({a[4] for a in starts}) == 1, starts
    assert len({a[5] for a in starts}) > 2 and all(a[5] >= 0 for a in starts), starts
    ring = scene.hist_frames
    assert sum(1 for a, e in run.catch_ups if a // ring != (e - 1) // ring) >= k // 2
    assert len({-(-(e - a) // scene.max_frames) for a, e in run.catch_ups}) > 1  # channels with different piece counts
    run.close()


@gpu
@pytest.mark.parametrize("mode", ["host_cs8_sync", "host_cs8_async"])
def test_the_event_log_is_unchanged(engine, mode):
    """With the caller's event log on, an auto-recording band logs the same events as its twin (checked after every push)."""
    Run(engine, MAIN, mode, 1, 21, auto_log=True).run().close()


# ---- refusals and lifetimes ----
@gpu
def test_refusals_and_lifetimes(engine):
    L = b2s.lib()
    cfg = b2s.make_config(N, FS, CENTER, learn_frames=LEARN, max_frames_per_push=600)
    band = b2s.Band(engine, cfg)
    bank = b2s.RecorderBank(engine, FS, BW, 2, max_samples_per_push=600 * N)
    assert L.b2s_band_set_auto_record(band._h, 1, 0) == E_INVALID  # no bank
    assert L.b2s_band_set_auto_record(band._h, 1, -1) == E_INVALID
    assert L.b2s_band_set_auto_record(None, 1, 0) == E_INVALID
    band.attach_recorder_bank(bank)
    bank.start(1, 5_000)
    assert L.b2s_band_set_auto_record(band._h, 1, 0) == E_STATE  # a channel records
    bank.stop(1)
    bank.set_history(100 * N)
    band.set_auto_record(True, 10)
    iq = np.zeros(2 * 50 * N, np.int8)
    band.push(iq, 50, 0, 1.0)
    assert L.b2s_recorder_bank_start(bank._h, 0, 0) == E_STATE
    assert L.b2s_recorder_bank_stop(bank._h, 0) == E_STATE
    assert L.b2s_recorder_bank_start_from(bank._h, 0, 0, 0, 0) == E_STATE
    assert L.b2s_band_record_from(band._h, 0, 0, 10) == E_STATE
    assert bank.flush(0) == [] and bank.flush(1) == []
    assert band.auto_record_actions() == []
    band.set_auto_record(False)
    bank.start(0, 1_000)  # the caller drives the bank again
    bank.stop(0)
    band.set_auto_record(True)
    band.attach_recorder_bank(None)  # detaching turns auto-record off
    bank.start(0, 1_000)
    bank.stop(0)
    band.attach_recorder_bank(bank)
    band.set_auto_record(True)
    band.load_state(band.save_state())  # a load leaves it off
    bank.start(0, 1_000)
    bank.stop(0)
    band.set_auto_record(True)
    bank.close()  # destroying the bank detaches it
    band.push(iq, 50, 50, 1.0)
    assert L.b2s_band_set_auto_record(band._h, 1, 0) == E_INVALID
    other = b2s.RecorderBank(engine, FS, BW, 2, max_samples_per_push=600 * N)
    band.attach_recorder_bank(other)
    band.set_auto_record(True)
    band.close()  # destroying the band leaves the bank to its caller
    other.start(0, 1_000)
    other.push(iq[: 2 * 10 * N], 0)
    other.close()
