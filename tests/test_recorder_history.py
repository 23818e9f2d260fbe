"""A recorder bank's history (b2s_recorder_bank_set_history): a recording that starts at a sample already pushed.

Every comparison is byte for byte, chunk times included. A channel started from the history must equal a channel of a fresh
stand-alone bank started with the same shift and pushed the history's samples from that position, cut every max_samples_per_push
samples (the first push at the given start time), then the same later pushes (include/b2s.h). The other channels, and a band the
bank is attached to, must equal twins that keep no history."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from conftest import ROOT, load_b2s
from test_band_recorder_bank import MAX_FRAMES, MODES, Stream, band_config, band_state, feed_standalone, flushed, new_bank, start_push, summary

b2s = load_b2s()
gpu = pytest.mark.gpu
E_INVALID, E_STATE = -1, -5
PRE_ROLL = 21  # the Averager's Y: a carrier crosses the start level up to Y frames after it appeared


def test_binding_matches_the_header():
    """b2s.py declares the four history functions as include/b2s.h does."""
    header = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "b2s.h")).read(), flags=re.S)
    want = {
        "b2s_recorder_bank_set_history": (["b2s_recorder_bank*", "size_t"], [C.c_void_p, C.c_size_t]),
        "b2s_recorder_bank_history": (["b2s_recorder_bank*", "int64_t*", "int64_t*"], [C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
        "b2s_recorder_bank_start_from": (["b2s_recorder_bank*", "int", "int32_t", "int64_t", "int64_t"], [C.c_void_p, C.c_int, C.c_int32, C.c_int64, C.c_int64]),
        "b2s_band_record_from": (["b2s_band*", "int", "int32_t", "int64_t"], [C.c_void_p, C.c_int, C.c_int32, C.c_int64]),
    }
    for name, (c_types, _) in want.items():
        m = re.search(r"\bint\s+" + name + r"\s*\(([^)]*)\)\s*;", header)
        assert m, f"{name} is not declared"
        assert [re.sub(r"\s+", "", re.sub(r"\w+\s*$", "", p)) for p in m.group(1).split(",")] == c_types, name  # types without names
    if not os.path.exists(b2s.LIB_PATH):
        pytest.skip("libb2s.so not built; run __graft_entry__.build()")
    for name, (_, argtypes) in want.items():
        f = getattr(b2s.lib(), name)
        assert f.argtypes == argtypes and f.restype == C.c_int, name
    assert all(callable(getattr(b2s.RecorderBank, m, None)) for m in ("set_history", "history", "start_from"))
    assert callable(getattr(b2s.Band, "record_from", None))


# ---- a stand-alone bank: 1.024 MS/s to 8 kS/s (two decimating stages) ----
FS, BW = 1_024_000, 8_000
M = 300_000  # max_samples_per_push
H = 1_000_003  # history: the ring ends at multiples of H, away from every push boundary
SIZES = [250_000, 300_000, 123_457, 300_000, 300_000, 300_000, 226_543, 300_000]  # 2.1 M samples: the ring has wrapped
LATER = [300_000, 300_000, 100_000]
TWIN_SHIFTS = [55_000, -200_000]  # channels 0 and 1 record from the start, in the bank and its twin
HIST_SHIFTS = [0, 137_000, -301_500]  # channels 2, 3 and 4 start from the history
START_MS = 77_777


def positions():
    end = sum(SIZES)
    boundary = sum(SIZES[:5])
    return {"boundary": boundary, "mid_push": boundary + 126_544, "oldest": end - H, "end": end}


def stream_iq(fmt, n, seed=11):
    rng = np.random.default_rng(seed)
    t = np.arange(n)
    z = 40 * np.exp(2j * np.pi * (140_000 / FS) * t) + 30 * np.exp(-2j * np.pi * (290_000 / FS) * t) + rng.normal(0, 12, n) + 1j * rng.normal(0, 12, n)
    x = np.empty(2 * n, np.float64)
    x[0::2], x[1::2] = z.real, z.imag
    x8 = np.clip(np.rint(x), -127, 127).astype(np.int8)
    return x8 if fmt == b2s.IQ_CS8 else x8.astype(np.float32) * np.float32(1 / 127.0)


def test_the_stand_alone_scene_wraps_and_straddles():
    """The scene covers what the stand-alone test is for: two stages, a wrapped ring, a catch-up longer than two pushes with a piece
    that straddles the ring's end (or whose carry does), for every position but `end`."""
    end = sum(SIZES)
    assert end > H
    for name, p in positions().items():
        assert end - H <= p <= end, name
        if name == "end":
            continue
        assert end - p > 2 * M, name
        cuts = list(range(p, end, M))
        assert any(s // H != (min(s + M, end) - 1) // H for s in cuts), name
    if os.path.exists(b2s.LIB_PATH):
        assert len(b2s.get_resamplers_factors(FS, BW)) == 2


class Input:
    def __init__(self, fmt, on_device):
        self.fmt, self.on_device = fmt, on_device
        self.host = stream_iq(fmt, sum(SIZES) + sum(LATER))
        self.bps = 2 * self.host.itemsize
        if on_device:
            import torch

            self.dev = torch.from_numpy(self.host.copy()).cuda()
            torch.cuda.synchronize()

    def samples(self, a, b):
        return self.host[2 * a : 2 * b]

    def push(self, bank, a, b, t0):
        if self.on_device:
            return bank.push(self.dev.data_ptr() + a * self.bps, t0, n_samples=b - a)
        return bank.push(self.samples(a, b), t0)


def t0_of(pos):
    return 5_000 + pos * 1000 // FS


def chunks(bank, channel):
    return [(t, c.tobytes()) for t, c in bank.flush(channel, cap=4096)]


@gpu
@pytest.mark.parametrize("where", ["boundary", "mid_push", "oldest", "end"])
@pytest.mark.parametrize("fmt,on_device", [(b2s.IQ_CS8, False), (b2s.IQ_CS8, True), (b2s.IQ_CF32, False), (b2s.IQ_CF32, True)])
def test_start_from_equals_a_fresh_bank_fed_the_same_cuts(engine, fmt, on_device, where):
    x = Input(fmt, on_device)
    n_ch = len(TWIN_SHIFTS) + len(HIST_SHIFTS)
    bank = b2s.RecorderBank(engine, FS, BW, n_ch, iq_format=fmt, on_device=on_device, max_samples_per_push=M)
    twin = b2s.RecorderBank(engine, FS, BW, n_ch, iq_format=fmt, on_device=on_device, max_samples_per_push=M)
    fresh = b2s.RecorderBank(engine, FS, BW, n_ch, iq_format=fmt, max_samples_per_push=M)
    bank.set_history(H)
    for k in (bank, twin):
        for c, s in enumerate(TWIN_SHIFTS):
            k.start(c, s)
    pos = 0
    for n in SIZES:
        for k in (bank, twin):
            x.push(k, pos, pos + n, t0_of(pos))
        pos += n
    end = pos
    assert bank.history() == (end - H, end)
    position = positions()[where]
    for i, s in enumerate(HIST_SHIFTS):
        bank.start_from(len(TWIN_SHIFTS) + i, s, position, START_MS)
        fresh.start(len(TWIN_SHIFTS) + i, s)
    assert bank.history() == (end - H, end)  # a catch-up appends nothing
    for j, a in enumerate(range(position, end, M)):
        fresh.push(x.samples(a, min(a + M, end)), START_MS if j == 0 else 0)
    for n in LATER:
        for k in (bank, twin):
            x.push(k, pos, pos + n, t0_of(pos))
        fresh.push(x.samples(pos, pos + n), t0_of(pos))
        pos += n
    assert bank.history() == (pos - H, pos)
    for c in range(len(TWIN_SHIFTS)):
        want = chunks(twin, c)
        assert len(want) > 3 and chunks(bank, c) == want, c
    for c in range(len(TWIN_SHIFTS), n_ch):
        want = chunks(fresh, c)
        assert len(want) >= (1 if where == "end" else 2) and chunks(bank, c) == want, c
        assert chunks(twin, c) == []
    for k in (bank, twin, fresh):
        k.close()


# ---- the band path: record_from(START frame - 21) on the modes of test_band_recorder_bank ----
BAND_SIZES = [130, 520, 700, 150]  # pipelined host copies, and a push the bank sees as pieces of 600 and 100 frames


def frame_clock(stream, pushes, frame):
    for f0, nf in pushes:
        if f0 <= frame < f0 + nf:
            return stream.t0(f0) + int(np.floor((frame - f0) * stream.period + 0.5))
    raise AssertionError(frame)


@gpu
@pytest.mark.parametrize("r", [1, 3])
@pytest.mark.parametrize("mode", list(MODES))
def test_record_from_a_start_event(engine, mode, r):
    on_device, fmt, flags = MODES[mode]
    stream = Stream(sum(BAND_SIZES), r, fmt, on_device)
    band, twin = b2s.Band(engine, band_config(stream, flags)), b2s.Band(engine, band_config(stream, flags))
    bank, twin_bank = new_bank(engine, stream), new_bank(engine, stream)
    bank.set_history(sum(BAND_SIZES) * stream.stride)
    for b, k in ((band, bank), (twin, twin_bank)):
        b.set_event_log(True)
        k.start(2, 317_500)  # records from the start in both
        b.attach_recorder_bank(k)
    alone = {}  # channel -> (stand-alone bank, its first chunk time)
    pushes, f0 = [], 0
    for nf in BAND_SIZES:
        want = summary(twin, start_push(twin, stream, f0, nf))
        events = twin.get_events()
        res = start_push(band, stream, f0, nf)  # an asynchronous band's push is still running during the catch-up
        pushes.append((f0, nf))
        for c in alone:
            feed_standalone(alone[c][0], stream, f0, nf)
        for kind, _, shift, frame, time_ms, _, _ in events:
            c = len(alone)
            if kind != b2s.EV_START or c >= 2:
                continue
            first = frame - PRE_ROLL
            assert first >= 0 and time_ms == frame_clock(stream, pushes, frame)
            band.record_from(c, shift, first)
            start_ms = frame_clock(stream, pushes, first)
            k = new_bank(engine, stream, on_device=False)
            k.start(c, shift)
            for j, a in enumerate(range(first, f0 + nf, MAX_FRAMES)):
                k.push(stream.samples(a, min(MAX_FRAMES, f0 + nf - a)), start_ms if j == 0 else 0)
            alone[c] = (k, start_ms)
        assert summary(band, res) == want, f0
        assert band.get_events() == events, f0
        got, ref = band_state(band), band_state(twin)
        for i, (a, b) in enumerate(zip(got, ref)):
            assert (a.tobytes() == b.tobytes()) if isinstance(a, np.ndarray) else a == b, (f0, i)
        f0 += nf
    assert len(alone) > 0
    chunk_ms = lambda j: int(np.floor((j + 1) * 4096 * 1000 / 32_000 + 0.5))  # chunk_samples = 4096 at 32 kS/s
    for c, (k, start_ms) in alone.items():
        want = flushed(k, c)
        assert len(want) > 0 and want[0][0] == start_ms + chunk_ms(0), c
        assert flushed(bank, c) == want, c
        k.close()
    assert flushed(bank, 2) == flushed(twin_bank, 2) and len(flushed(twin_bank, 3)) == 0
    band.close()
    twin.close()
    bank.close()
    twin_bank.close()


# ---- refusals change nothing ----
@gpu
def test_refusals_change_nothing(engine):
    stream = Stream(900, 1, b2s.IQ_CS8, False)
    L = b2s.lib()
    band, twin = b2s.Band(engine, band_config(stream, 0)), b2s.Band(engine, band_config(stream, 0))
    bank, twin_bank = new_bank(engine, stream), new_bank(engine, stream)
    for k in (bank, twin_bank):
        k.start(1, -635_000)
    f0 = 0

    def push(nf):
        nonlocal f0
        for b in (band, twin):
            summary(b, start_push(b, stream, f0, nf))
        f0 += nf

    def same():
        assert bank.history() == twin_bank.history()
        for c in range(4):
            assert [(t, x.tobytes()) for t, x in bank.flush(c, consume=False)] == [(t, x.tobytes()) for t, x in twin_bank.flush(c, consume=False)], c
        for i, (a, b) in enumerate(zip(band_state(band), band_state(twin))):
            assert (a.tobytes() == b.tobytes()) if isinstance(a, np.ndarray) else a == b, i

    def refused(rc_want, frame=None, channel=0, position=None):
        if position is None:
            rc = L.b2s_band_record_from(band._h, channel, 0, frame)
        else:
            rc = L.b2s_recorder_bank_start_from(bank._h, channel, 0, position, 0)
        assert rc == rc_want, (frame, position, rc)
        same()

    push(100)  # frames 0-99: no bank attached
    refused(E_INVALID, 50)
    for b, k in ((band, bank), (twin, twin_bank)):
        b.attach_recorder_bank(k)
    push(100)  # frames 100-199: the bank keeps no history
    refused(E_INVALID, 150)
    refused(E_INVALID, position=0)
    keep = 150 * stream.stride
    for k in (bank, twin_bank):
        k.set_history(keep)
    push(200)  # frames 200-399: the history holds frames 250-399
    assert bank.history() == (200 * stream.stride - keep, 200 * stream.stride)
    for frame in (50, 150, 249, 400, 10_000, -1):  # before attach, before set_history, no longer held, not yet pushed
        refused(E_INVALID, frame)
    oldest, end = bank.history()
    refused(E_INVALID, position=oldest - 1)
    refused(E_INVALID, position=end + 1)
    refused(E_INVALID, 300, channel=4)
    refused(E_STATE, 300, channel=1)
    refused(E_STATE, channel=1, position=end)
    lo, hi = band.cfg.range_lo_hz, band.cfg.range_hi_hz
    for b in (band, twin):
        b.set_center(band.cfg.center_hz, lo, hi)  # the same centre: frames stay usable
    push(50)  # frames 400-449
    for b in (band, twin):
        b.reset()  # does not limit record_from
    for b in (band, twin):
        b.record_from(2, 250_000, 300)
    same()
    for b in (band, twin):
        b.set_center(band.cfg.center_hz + 100_000, lo + 100_000, hi + 100_000)
    push(50)  # frames 450-499
    refused(E_INVALID, 449)
    for b in (band, twin):
        b.record_from(3, -55_000, 460)
    same()
    for b in (band, twin):
        b.load_state(b.save_state())
    refused(E_INVALID, 470)
    push(100)
    refused(E_INVALID, 499)
    for b in (band, twin):
        b.record_from(0, 0, 520)
    push(300)
    same()
    for c in range(4):
        want = flushed(twin_bank, c)
        assert len(want) > 0 and flushed(bank, c) == want, c
    for x in (band, twin, bank, twin_bank):
        x.close()


# ---- lifetimes and snapshots ----
@gpu
def test_lifetimes_and_snapshots(engine):
    stream = Stream(700, 1, b2s.IQ_CS8, False)
    s = stream.stride
    band = b2s.Band(engine, band_config(stream, 0))
    bank, plain = new_bank(engine, stream), new_bank(engine, stream)
    assert bank.history() == (0, 0)
    bank.set_history(100 * s)
    for k in (bank, plain):
        k.start(0, 317_500)
    band.attach_recorder_bank(bank)
    summary(band, start_push(band, stream, 0, 150))
    plain.push(stream.samples(0, 150), stream.t0(0))
    assert bank.history() == (50 * s, 150 * s)
    bank.set_history(0)
    assert bank.history() == (0, 0)
    summary(band, start_push(band, stream, 150, 50))
    plain.push(stream.samples(150, 50), stream.t0(150))
    assert bank.history() == (50 * s, 50 * s)  # positions count on, nothing is held
    bank.set_history(120 * s)  # a resize empties the history
    assert bank.history() == (0, 0)
    summary(band, start_push(band, stream, 200, 100))
    plain.push(stream.samples(200, 100), stream.t0(200))
    band.attach_recorder_bank(None)  # detaching keeps the history; stand-alone pushes append to it
    assert bank.history() == (0, 100 * s)
    for k in (bank, plain):
        k.push(stream.samples(300, 100), stream.t0(300))
    assert bank.history() == (80 * s, 200 * s)
    assert bank.save_state() == plain.save_state()  # the history is not in a snapshot
    start_ms = 12_345
    bank.start_from(1, -55_000, 130 * s, start_ms)  # frame 330: positions count from the resize at frame 200
    fresh = new_bank(engine, stream, on_device=False)
    fresh.start(1, -55_000)
    fresh.push(stream.samples(330, 70), start_ms)
    snap = bank.save_state()
    other = new_bank(engine, stream)
    other.set_history(50 * s)
    other.load_state(snap)
    assert other.history() == (0, 0)
    for k in (bank, other, fresh):
        k.push(stream.samples(400, 300), stream.t0(400))
    for c in (0, 1):
        want = flushed(bank, c)
        assert len(want) > 0 and flushed(other, c) == want, c
        if c == 1:
            assert flushed(fresh, c) == want
    for x in (band, bank, plain, fresh, other):
        x.close()
