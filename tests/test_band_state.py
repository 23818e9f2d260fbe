"""Band and recorder bank snapshots (b2s_band_save_state / b2s_band_load_state, b2s_recorder_bank_save_state / _load_state).

Band A runs a stream without interruption. At push k its snapshot is loaded into a fresh band B, and both get the remaining pushes.
After every remaining push, and without tolerance, B equals A in everything a caller can read: the mailbox and n_transmissions_total,
the complete transmission list, the signal map, the Averager, the noise thresholds of every centre visited, the spectrogram rows, the
events and the b2s_band_sync statistics. Each read is made the same way on both bands, so reads that consume (rows, events, statistics)
consume the same on both."""
import ctypes as C
import struct

import numpy as np
import pytest

import __graft_entry__ as ge
from conftest import load_b2s
from test_busy_spectrum import Case, busy_iq

b2s = load_b2s()
synth = ge.load_synth()
pytestmark = pytest.mark.gpu

N, FS, LEARN = 2048, 2_048_000, 30
CENTERS = (100_000_000, 101_500_000)
INVALID = r"b2s error -1:"


def span(center, fs=FS):
    return center, center - fs // 2, center + fs // 2


def config(n=N, fs=FS, flags=0, **kw):
    kw.setdefault("learn_frames", LEARN)
    cfg = b2s.make_config(n, fs, min_time_ms=50, timeout_ms=100, flags=flags, **kw)
    cfg.spectrogram_interval_ms = 50  # several rows per push, and most splits fall inside an interval
    return cfg


def scene(frames, seed=11):
    return synth.make_iq_int8(N, frames, synth.standard_scene(N, frames, LEARN), seed=seed, quiet_frames=LEARN)


class Feed:
    """One CS8 stream of [frames][n] samples, on the host and, for bands with device IQ, on their device."""

    def __init__(self, iq, n=N, fs=FS):
        self.iq, self.n, self.period, self.dev = iq, n, synth.frame_period_ms(n, fs), {}

    def ptr(self, band, f0, device=0):
        if band.cfg.flags & b2s.FLAG_IQ_ON_DEVICE:
            if device not in self.dev:
                import torch

                self.dev[device] = torch.from_numpy(self.iq).to(f"cuda:{device}")
                torch.cuda.synchronize(device)
            return self.dev[device].data_ptr() + f0 * 2 * self.n
        return self.iq.ctypes.data + f0 * 2 * self.n

    def t0(self, f0):
        return 1_000 + int(np.floor(f0 * self.period + 0.5))

    def push(self, band, f0, nf, device=0, per_frame=False):
        """One push; returns whether it reported B2S_E_OVERFLOW (the push completed on truncated lists), and with per_frame (a host-IQ
        synchronous band) every frame's list."""
        try:
            if per_frame:
                out = band.push(self.iq[2 * f0 * self.n : 2 * (f0 + nf) * self.n], nf, self.t0(f0), self.period, per_frame=True)
                return False, out.frame_tx
            band.push_raw(self.ptr(band, f0, device), nf, self.t0(f0), self.period)
        except b2s.B2SError as e:
            if "b2s error -4:" not in str(e):
                raise
            return True, None
        return False, None


def state(band, centers, current):
    """Everything a caller can read of the band. The noise of each centre is read by tuning to it; the band is tuned back after."""
    n = band.cfg.fft_size
    res = band.sync()
    out = {"mailbox": [(t.shift_hz, t.flush, t.key, t.power) for t in res.transmissions[: res.n_transmissions]],
           "totals": (res.n_transmissions_total, res.n_detect_entries, res.n_spectrogram_rows),
           "tx": band.get_transmissions(cap=n),
           "signals": [x.tobytes() for x in band.get_signals(cap=n)]}
    s, a, ring, frames = band.get_averager()
    out["averager"] = (s.tobytes(), a.tobytes(), ring.tobytes(), frames)
    for c in centers:
        band.set_center(*span(c, band.cfg.sample_rate_hz))
        thr, samples, ready = band.get_noise()
        out[("noise", c)] = (thr.tobytes(), samples, ready)
    band.set_center(*current)
    times, cs, rows = band.get_spectrogram(cap=4096)
    out["rows"] = (times.tobytes(), cs.tobytes(), rows.tobytes())
    out["events"] = band.get_events()
    return out


def assert_same(a, b, centers, current, where):
    sa, sb = state(a, centers, current), state(b, centers, current)
    assert sa.keys() == sb.keys()
    for key in sa:
        assert sa[key] == sb[key], (where, key)
    return sa


def split_run(engine, cfg_a, cfg_b, feed, sizes, k, *, centers=(CENTERS[0],), engine_b=None, device_b=0, at_split=None):
    """A gets every push; B is loaded from A's snapshot before push k and gets the pushes from k on. The first push after the split is
    host-tracked (per-frame lists) on each band that takes host IQ synchronously. Returns A's states after the pushes from k on."""
    a = b2s.Band(engine, cfg_a)
    a.set_event_log(True)
    b, states, f0 = None, [], 0
    for i, nf in enumerate(sizes):
        current = span(centers[i % len(centers)], cfg_a.sample_rate_hz)
        if i == k:
            if at_split:
                at_split(a)
            blob = a.save_state()
            b = b2s.Band(engine_b or engine, cfg_b)
            b.load_state(blob)
            if cfg_a.flags == cfg_b.flags and cfg_a.detect_capacity == cfg_b.detect_capacity:
                assert b.save_state() == blob, "saving, loading and saving again changed the bytes"
        frame_lists, overflow = [], []
        for band, dev in ((a, 0), (b, device_b)):
            if band is None:
                continue
            if len(centers) > 1:
                band.set_center(*current)
            per_frame = i == k and not band.cfg.flags & (b2s.FLAG_ASYNC | b2s.FLAG_IQ_ON_DEVICE)
            o, lists = feed.push(band, f0, nf, dev, per_frame)
            overflow.append(o)
            if lists is not None:
                frame_lists.append(lists)
        if b is not None:
            assert overflow[0] == overflow[1], (i, overflow)
            if len(frame_lists) == 2:
                assert frame_lists[0] == frame_lists[1], i
            states.append(assert_same(a, b, centers, current, i))
        f0 += nf
    for x in (a, b):
        x.close()
    return states


MODES = {  # A -> B
    "sync": (0, 0),
    "sync_to_async_device": (0, b2s.FLAG_ASYNC | b2s.FLAG_IQ_ON_DEVICE),
    "async_device_to_sync": (b2s.FLAG_ASYNC | b2s.FLAG_IQ_ON_DEVICE, 0),
}


@pytest.mark.parametrize("mode", list(MODES))
def test_split_during_noise_learning_and_averager_warm_up(engine, mode):
    """noise_learning_ms: the split falls after 5 frames, with the centre's learning started but not finished and the Averager warming
    up, inside a spectrogram interval."""
    fa, fb = MODES[mode]
    sizes = [5, 10, 7, 60, 100, 33, 185]
    seen = {}

    def check(a):
        _, samples, ready = a.get_noise()
        seen["noise"] = (samples, ready, a.get_averager()[3])

    split_run(engine, config(flags=fa, noise_learning_ms=40), config(flags=fb, noise_learning_ms=40), Feed(scene(sum(sizes))), sizes, 1, at_split=check)
    samples, ready, frames = seen["noise"]
    assert 0 < samples and not ready and 0 < frames < 21, seen


@pytest.mark.parametrize("mode", list(MODES))
def test_split_with_live_signals_that_time_out_later(engine, mode):
    fa, fb = MODES[mode]
    sizes = [50, 90, 13, 100, 147]
    live = {}
    states = split_run(engine, config(flags=fa), config(flags=fb), Feed(scene(sum(sizes))), sizes, 2,
                       at_split=lambda a: live.setdefault("keys", set(a.get_signals(cap=N)[0].tolist())))
    stopped = {e[1] for s in states for e in s["events"] if e[0] == b2s.EV_STOP}
    assert live["keys"] and live["keys"] & stopped, (live, stopped)


@pytest.mark.parametrize("mode", ["sync", "sync_to_async_device"])
def test_split_under_a_hop_schedule(engine, mode):
    """Two centres alternate every push: the noise and spectrogram maps hold a slot for each, one of them still learning."""
    fa, fb = MODES[mode]
    sizes = [20] * 24
    states = split_run(engine, config(flags=fa, noise_learning_ms=90), config(flags=fb, noise_learning_ms=90), Feed(scene(sum(sizes))), sizes, 5,
                       centers=CENTERS)
    first = states[0]
    assert all(first[("noise", c)][1] > 0 for c in CENTERS)
    assert any(c == CENTERS[1] for c in np.frombuffer(first["rows"][1], np.int32))


def test_split_on_a_second_engine_of_the_same_device(engine):
    sizes = [50, 90, 13, 100, 147]
    other = b2s.Engine(0)
    split_run(engine, config(), config(), Feed(scene(sum(sizes))), sizes, 2, engine_b=other)
    other.close()


def test_split_onto_another_gpu(engine):
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU: the move to another device was not run")
    sizes = [50, 90, 13, 100, 147]
    other = b2s.Engine(1)
    split_run(engine, config(), config(flags=b2s.FLAG_IQ_ON_DEVICE), Feed(scene(sum(sizes))), sizes, 2, engine_b=other, device_b=1)
    other.close()


BUSY = Case("busy_n16384", 16384, 20_000_000, 200, splits=(37, 64, 5, 100), blocks=((-9.5e6, -3.0e6, 30, 120), (-1.0e6, 5.5e6, 50, 150)))


def test_split_with_more_than_256_live_signals(engine):
    """The split falls where A's map holds more than 256 signals, so that B's next push runs k_track_wide from the restored map."""
    case = BUSY
    iq = busy_iq(case, seed=4242)
    feed = Feed(iq, case.n, case.fs)
    sizes = [m for _, _, m in case.pushes()]
    probe, f0, k = b2s.Band(engine, case.config()), 0, None
    for i, nf in enumerate(sizes):  # the first push after which more than 256 signals are live
        feed.push(probe, f0, nf)
        f0 += nf
        if len(probe.get_signals(cap=case.n)[0]) > 256:
            k = i + 1
            break
    probe.close()
    assert k is not None and k < len(sizes), "the scene never had more than 256 live signals"
    cfg_b = case.config()
    cfg_b.flags = b2s.FLAG_ASYNC | b2s.FLAG_IQ_ON_DEVICE
    cfg_b.detect_capacity = 0
    split_run(engine, case.config(), cfg_b, feed, sizes, k, centers=(case.config().center_hz,))


def test_split_after_the_detection_capacity_grew(engine):
    """A overflows its small per-frame capacity and grows it; B, created with the default capacity, takes the grown one."""
    case = Case("capacity", N, FS, 200, splits=(40,), blocks=((-0.5e6, 0.4e6, 30, 190),), learn=20)
    cfg_a, cfg_b = case.config(), case.config()
    cfg_a.detect_capacity, cfg_b.detect_capacity = 64, 0  # B's default is 256 at N = 2048; the block alone is about 900 bins wide
    feed = Feed(busy_iq(case, seed=77))
    a = b2s.Band(engine, cfg_a)
    assert any(feed.push(a, f0, 40)[0] for f0 in (0, 40)), "A never overflowed"
    a.close()
    sizes = [40] * 5
    split_run(engine, cfg_a, cfg_b, feed, sizes, 2, centers=(cfg_a.center_hz,))


def test_split_at_n_1048576(engine):
    case = Case("n1048576", 1048576, 200_000_000, 80, splits=(30, 17, 33), blocks=((-60.0e6, -52.0e6, 20, 60), (10.0e6, 18.0e6, 25, 75)), learn=16)
    cfg_b = case.config()
    cfg_b.flags = b2s.FLAG_ASYNC | b2s.FLAG_IQ_ON_DEVICE
    feed = Feed(busy_iq(case, seed=1048), case.n, case.fs)
    split_run(engine, case.config(), cfg_b, feed, [30, 17, 33], 1, centers=(case.config().center_hz,))


# ---- an attached recorder bank saved and restored with its band ----
BW, MAX_FRAMES = 32_000, 600


def flushed(bank, channel):
    return [(t, c.tobytes()) for t, c in bank.flush(channel, cap=4096)]


@pytest.mark.parametrize("r,flags", [(1, 0), (3, 0), (3, b2s.FLAG_ASYNC | b2s.FLAG_IQ_ON_DEVICE)], ids=["r1_sync", "r3_sync", "r3_async_device"])
def test_attached_bank_restored_with_its_band(engine, r, flags):
    stride = N * r
    sizes = [100, 37, 250, 64, 120]
    iq = synth.make_iq_int8(N, sum(sizes), synth.standard_scene(N, sum(sizes), LEARN), seed=5, quiet_frames=LEARN, stride=stride)
    period = synth.frame_period_ms(N, FS, r)

    def new_band():
        cfg = config(flags=flags, decimator=r, max_frames_per_push=MAX_FRAMES)
        return b2s.Band(engine, cfg)

    def new_bank():
        return b2s.RecorderBank(engine, FS, BW, 3, max_samples_per_push=MAX_FRAMES * stride)

    dev = None
    if flags & b2s.FLAG_IQ_ON_DEVICE:
        import torch

        dev = torch.from_numpy(iq).cuda()
        torch.cuda.synchronize()

    def push(band, f0, nf):
        base = dev.data_ptr() if dev is not None else iq.ctypes.data
        band.push_raw(base + f0 * stride * 2, nf, 1_000 + int(np.floor(f0 * period + 0.5)), period)

    a, bank_a = new_band(), new_bank()
    a.attach_recorder_bank(bank_a)
    bank_a.start(0, 317_500)  # rotated
    bank_a.start(1, 0)
    b = bank_b = None
    f0, total = 0, 0
    for i, nf in enumerate(sizes):
        if i == 2:
            blob, kblob = a.save_state(), bank_a.save_state()  # an asynchronous band leaves its last piece pending: the save settles it
            b, bank_b = new_band(), new_bank()
            b.load_state(blob)
            bank_b.load_state(kblob)
            assert bank_b.save_state() == kblob
            b.attach_recorder_bank(bank_b)
        if i == 3:
            for k in (bank_a, bank_b):
                k.start(2, -200_000)
                k.stop(1)
        for band in (a, b):
            if band is not None:
                push(band, f0, nf)
        if b is not None:
            for c in range(3):
                got, want = flushed(bank_b, c), flushed(bank_a, c)
                assert got == want, (i, c)
                total += len(got)
            assert_same(a, b, (CENTERS[0],), span(CENTERS[0]), i)
        f0 += nf
    assert total > 0
    for x in (a, b, bank_a, bank_b):
        x.close()


# ---- saving changes nothing ----
@pytest.mark.parametrize("flags", [0, b2s.FLAG_ASYNC | b2s.FLAG_IQ_ON_DEVICE], ids=["sync", "async_device"])
def test_saving_does_not_perturb(engine, flags):
    sizes = [5, 40, 60, 100, 33, 120]
    feed = Feed(scene(sum(sizes)))
    a, twin = b2s.Band(engine, config(flags=flags)), b2s.Band(engine, config(flags=flags))
    for x in (a, twin):
        x.set_event_log(True)
    f0, blobs = 0, []
    for i, nf in enumerate(sizes):
        for x in (a, twin):
            feed.push(x, f0, nf)
        blobs.append(a.save_state())  # before the sync of an asynchronous push: the save finishes it but collects nothing
        assert_same(a, twin, (CENTERS[0],), span(CENTERS[0]), i)
        f0 += nf
    assert len(set(blobs)) == len(blobs)
    for x in (a, twin):
        x.close()


# ---- refusals ----
def fnv1a64(data):
    h = 0xCBF29CE484222325
    for x in data:
        h = ((h ^ x) * 0x100000001B3) & 0xFFFFFFFFFFFFFFFF
    return h


def resealed(body):
    """`body` (a snapshot without its checksum) with a correct checksum, so that the check that refuses it is not the checksum's."""
    return body + struct.pack("<Q", fnv1a64(body))


def assert_refused(engine, cfg, blob, feed, f0=0, nf=60):
    """A band refuses the snapshot with B2S_E_INVALID and then equals a twin that never saw it, after another push."""
    band, twin = b2s.Band(engine, cfg), b2s.Band(engine, cfg)
    for x in (band, twin):
        feed.push(x, f0, nf)
    with pytest.raises(b2s.B2SError, match=INVALID):
        band.load_state(blob)
    for x in (band, twin):
        feed.push(x, f0 + nf, nf)
    assert_same(band, twin, (cfg.center_hz,), span(cfg.center_hz, cfg.sample_rate_hz), "after the refusal")
    band.close()
    twin.close()


def test_damaged_and_foreign_snapshots_are_refused(engine):
    feed = Feed(scene(400))
    a = b2s.Band(engine, config())
    a.set_event_log(True)
    for f0, nf in ((0, 60), (60, 120)):
        feed.push(a, f0, nf)
    blob = a.save_state()
    a.close()
    assert fnv1a64(blob[:-8]) == struct.unpack("<Q", blob[-8:])[0]
    bad = [blob[:n] for n in (0, 10, 20, 27, len(blob) // 2, len(blob) - 9, len(blob) - 1)]
    flipped = bytearray(blob)
    flipped[len(blob) // 2] ^= 0x10
    bad.append(bytes(flipped))
    bad.append(resealed(b"XXXX" + blob[4:-8]))  # magic
    bad.append(resealed(blob[:4] + struct.pack("<I", 2) + blob[8:-8]))  # version
    bad.append(resealed(blob[:8] + struct.pack("<I", 2) + blob[12:-8]))  # kind: a bank
    for x in bad:
        assert_refused(engine, config(), x, feed, 180)

    bank = b2s.RecorderBank(engine, FS, BW, 2)
    bank.start(0, 1000)
    bank.push(feed.iq[: 2 * 8192])
    kblob = bank.save_state()
    with pytest.raises(b2s.B2SError, match=INVALID):
        bank.load_state(blob)  # a band snapshot into a bank
    assert_refused(engine, config(), kblob, feed, 180)  # and the reverse
    other = b2s.RecorderBank(engine, FS, BW, 3)
    with pytest.raises(b2s.B2SError, match=INVALID):
        other.load_state(kblob)  # another channel count
    assert bank.save_state() == kblob
    bank.close()
    other.close()


@pytest.mark.parametrize("field,value", [("fft_size", 4096), ("start_level", 7.0), ("grouping_x", 19)])
def test_snapshot_of_another_config_is_refused(engine, field, value):
    feed = Feed(scene(300))
    a = b2s.Band(engine, config())
    feed.push(a, 0, 100)
    blob = a.save_state()
    a.close()
    cfg = config()
    setattr(cfg, field, value)
    if field == "fft_size":
        cfg = config(n=value)
        feed = Feed(synth.make_iq_int8(value, 200, synth.standard_scene(value, 200, LEARN), seed=3, quiet_frames=LEARN), value)
    assert_refused(engine, cfg, blob, feed)


def test_snapshot_with_other_user_window_taps_is_refused(engine):
    feed = Feed(scene(300))
    taps = np.hamming(N).astype(np.float32)
    other = taps.copy()
    other[N // 3] = np.nextafter(other[N // 3], np.float32(2))

    def user_config(w):
        cfg = config()
        cfg.window_kind = 1
        cfg.window_taps = w.ctypes.data_as(C.POINTER(C.c_float))
        return cfg

    a = b2s.Band(engine, user_config(taps))
    feed.push(a, 0, 100)
    blob = a.save_state()
    a.close()
    assert_refused(engine, user_config(other), blob, feed)
    taps_again = taps.copy()  # the config holds a raw pointer: the array must live until the band is created
    same = b2s.Band(engine, user_config(taps_again))
    same.load_state(blob)  # equal taps from another array are accepted
    assert same.save_state() == blob
    same.close()


# ---- every section cut short, and every list count forged ----
def sections(blob):
    """[(tag, start of the payload, payload length)] of a snapshot, found from the framing alone (u32 tag, u64 length)."""
    out, at, end = [], 20, len(blob) - 8
    while at < end:
        tag, n = struct.unpack_from("<4sQ", blob, at)
        out.append((tag.decode(), at + 12, n))
        at += 12 + n
    assert at == end
    return out


def variants(blob, counts):
    """(what, snapshot): each section's payload cut by one byte, and each list count that `counts(tag, payload)` locates as
    (offset, struct format) raised to count + 1 and to 2^32 - 1; the section length, the total length and the checksum fixed up."""
    for tag, start, n in sections(blob):
        payload = blob[start : start + n]
        changed = [(f"{tag} cut by one byte", payload[:-1])]
        for off, fmt in counts(tag, payload):
            for v in (struct.unpack_from(fmt, payload, off)[0] + 1, 2**32 - 1):
                p = bytearray(payload)
                struct.pack_into(fmt, p, off, v)
                changed.append((f"{tag} count at {off} set to {v}", bytes(p)))
        for what, p in changed:
            body = blob[: start - 8] + struct.pack("<Q", len(p)) + p + blob[start + n : -8]
            yield what, resealed(body[:12] + struct.pack("<Q", len(body) + 8) + body[20:])


def test_every_section_cut_or_with_a_forged_count_is_refused(engine):
    feed = Feed(scene(400))
    a = b2s.Band(engine, config())
    a.set_event_log(True)
    for f0, nf in ((0, 60), (60, 120)):
        feed.push(a, f0, nf)
    blob = a.save_state()
    a.close()
    assert [t for t, _, _ in sections(blob)] == ["CONF", "SCAL", "NOIS", "SPEC", "AVGR", "SMAP", "MBOX", "EVNT", "ROWS"]
    band_counts = {"NOIS": "<I", "SPEC": "<I", "SMAP": "<I", "MBOX": "<I", "EVNT": "<Q", "ROWS": "<Q"}  # each at the payload's start
    for what, x in variants(blob, lambda tag, payload: [(0, band_counts[tag])] if tag in band_counts else []):
        try:
            assert_refused(engine, config(), x, feed, 180)
        except BaseException as e:
            raise AssertionError(what) from e

    bank = b2s.RecorderBank(engine, FS, BW, 3)
    bank.start(0, 317_500)
    bank.start(1, 0)  # channel 2 stays idle
    bank.push(feed.iq)
    kblob = bank.save_state()
    chunk_bytes = len(bank.flush(0, cap=1, consume=False)[0][1])
    chan = [(start, n) for t, start, n in sections(kblob) if t == "CHAN"]
    assert [t for t, _, _ in sections(kblob)] == ["CONF", "RAWC"] + ["CHAN"] * 3
    carry = chan[2][1] - 50  # the idle channel: 2 bool bytes, 4 x 8 bytes, its carries, a chunk count of 0 and a tail of 0 (u64 each)

    def chan_counts(tag, payload):
        if tag != "CHAN":
            return []
        at = 34 + carry
        n = struct.unpack_from("<Q", payload, at)[0]
        return [(at, "<Q"), (at + 8 + n * chunk_bytes, "<Q")]  # the complete chunks, the tail's bytes

    assert struct.unpack_from("<Q", kblob, chan[0][0] + 34 + carry)[0] > 0, "channel 0 holds no complete chunk"
    for what, x in variants(kblob, chan_counts):
        try:
            with pytest.raises(b2s.B2SError, match=INVALID):
                bank.load_state(x)
            assert bank.save_state() == kblob
        except BaseException as e:
            raise AssertionError(what) from e
    bank.close()
