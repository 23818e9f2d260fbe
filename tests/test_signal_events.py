"""The signal event log of the device tracker (K4: k_track / k_track_wide appending START and STOP records) against a host-tracked
twin fed the same IQ. The twin's per-frame lists give the expected events (signal_events.py), the twin's own log (tracker.h) must
equal them, and the device-tracked band's log must equal the twin's record for record. No tolerance anywhere."""
import numpy as np
import pytest

import signal_events as se
from conftest import load_b2s
from test_busy_spectrum import CASES as BUSY_CASES
from test_busy_spectrum import MAX_CAND, MAX_SIGNALS, Case, busy_iq

b2s = load_b2s()
pytestmark = pytest.mark.gpu


def _load_synth():
    import __graft_entry__ as g

    return g.load_synth()


def _spans(lengths):
    k = 0
    for m in lengths:
        yield k, m
        k += m


def _keys(res):
    return {t.key for t in res.transmissions[: res.n_transmissions]}


def _twin(engine, cfg, iq, lengths, t0, period, reset_before=None, dense=()):
    """Host-tracked pushes with every frame's list. Returns the expected changes, the twin's log and, per push, the outputs."""
    n = cfg.fft_size
    band = b2s.Band(engine, cfg)
    band.set_event_log(True)
    exp, want, outs = se.Expected(), [], []
    for i, (k, m) in enumerate(_spans(lengths)):
        if i == reset_before:
            band.reset()
            exp.reset()
        out = band.push(iq[k * 2 * n : (k + m) * 2 * n], m, t0 + int(k * period), period, per_frame=True, dense=dense)
        want += exp.feed(out.frame_tx)
        outs.append(out)
    log = band.get_events()
    band.close()
    return want, log, outs


def _device(engine, cfg, iq, lengths, t0, period, reset_before=None, async_device=False, log=True):
    """Device-tracked pushes. Returns the log, and per push the result (synchronous bands) and K4's launches."""
    n = cfg.fft_size
    cfg = b2s.BandConfig.from_buffer_copy(cfg)
    src = iq
    if async_device:
        import torch

        cfg.flags |= b2s.FLAG_ASYNC | b2s.FLAG_IQ_ON_DEVICE
        src = torch.from_numpy(iq).cuda()
    band = b2s.Band(engine, cfg)
    if log:
        band.set_event_log(True)
    band.set_profiling(True)
    results, launches = [], []
    for i, (k, m) in enumerate(_spans(lengths)):
        if i == reset_before:
            band.reset()
        ptr = src.data_ptr() + k * 2 * n if async_device else iq[k * 2 * n :].ctypes.data
        results.append(band.push_raw(ptr, m, t0 + int(k * period), period))
        if not async_device:
            launches.append(band.get_profile().track_launches)
    if async_device:
        band.sync()
    return band, band.get_events() if log else None, results, launches


# ---------------------------------------------------------------------------------------------------------------
# keyed carriers: N = 4096 at 2.048 MS/s, 2 ms per frame
# ---------------------------------------------------------------------------------------------------------------
N, FS, FRAMES, LEARN, T0, PERIOD = 4096, 2_048_000, 1200, 40, 1000, 2.0
PUSHES = (300, 500, 400)
TIMEOUT, MAX_TIME = 30, 500


def _keyed_config(**kw):
    return b2s.make_config(N, FS, learn_frames=LEARN, recording_bandwidth_hz=16 * FS // N, min_time_ms=20, timeout_ms=TIMEOUT, max_time_ms=MAX_TIME,
                           max_frames_per_push=512, **kw)


@pytest.fixture(scope="module")
def keyed():
    synth = _load_synth()
    T = synth.Tone
    tones = [
        T(bin_offset=635.1, amplitude=60.0, on_frames=[(340, 420)], fm_dev_bins=6.0),              # starts and times out inside the second push
        T(bin_offset=-1269.9, amplitude=60.0, on_frames=[(100, 500)], fm_dev_bins=6.0),            # first push -> second (longer than max_time)
        T(bin_offset=112.7, amplitude=60.0, on_frames=[(700, 1100)], phase=1.0, fm_dev_bins=5.0),  # second push -> third
        T(bin_offset=-400.1, amplitude=60.0, fm_dev_bins=6.0),                                     # always on: max_time stops it again and again
    ]
    return synth.make_iq_int8(N, FRAMES, tones, seed=synth.seed_for(7), quiet_frames=LEARN)


def _frame_time(f):
    return T0 + 2 * f


def test_a_transmission_inside_one_push_is_logged(engine, keyed):
    cfg = _keyed_config()
    want, twin_log, _ = _twin(engine, cfg, keyed, PUSHES, T0, PERIOD)
    se.assert_log_equals(twin_log, want, "twin")
    se.assert_times(twin_log, TIMEOUT, MAX_TIME, _frame_time)
    band, log, results, launches = _device(engine, cfg, keyed, PUSHES, T0, PERIOD)
    band.close()
    assert log == twin_log
    assert launches == [1, 1, 1], "k_track ran every push"
    # the case the log exists for: a key inserted and erased inside the second push, in no mailbox around it
    lo, hi = PUSHES[0], PUSHES[0] + PUSHES[1]
    started = {}
    inside = set()
    for kind, key, _, frame, *_ in log:
        if kind == se.START:
            started[key] = frame
        elif lo <= started[key] and frame < hi:
            inside.add(key)
    unseen = inside - _keys(results[0]) - _keys(results[1])
    assert unseen, (inside, [_keys(r) for r in results])
    # carriers that start in one push and stop in a later one, and both kinds of stop
    crossing = [e for e in log if e[0] == se.STOP and any(e[5] < _frame_time(b) <= e[4] for b in (lo, hi))]
    assert crossing
    by_max_time = [e for e in log if e[0] == se.STOP and e[5] + MAX_TIME <= e[4] and not e[6] + TIMEOUT <= e[4]]
    by_timeout = [e for e in log if e[0] == se.STOP and e[6] + TIMEOUT <= e[4] and not e[5] + MAX_TIME <= e[4]]
    assert by_max_time and by_timeout


@pytest.mark.parametrize("reset_before", [None, 2], ids=["no_reset", "reset"])
def test_the_log_does_not_depend_on_how_the_stream_is_pushed(engine, keyed, reset_before):
    cfg = _keyed_config()
    # the reset falls on frame 370 in every split
    splits = {
        "sync": ((37, 333, 1, 700, 129), 2),          # 700 frames exceed max_frames_per_push: two K4 launches
        "one_or_two": ((370, 830), 1),
        "async_device": ((369, 1, 31, 799), 2),
    }
    twin_lengths = (370, 830)
    want, twin_log, _ = _twin(engine, cfg, keyed, twin_lengths, T0, PERIOD, reset_before=1 if reset_before else None)
    se.assert_log_equals(twin_log, want, "twin")
    assert twin_log[-1][3] > 900, "frames go on counting"
    if reset_before:
        _, plain, _ = _twin(engine, cfg, keyed, twin_lengths, T0, PERIOD)
        assert plain != twin_log and [e for e in twin_log if e[3] < 370] == [e for e in plain if e[3] < 370], "a reset logs nothing"
    for name, (lengths, at) in splits.items():
        band, log, _, _ = _device(engine, cfg, keyed, lengths, T0, PERIOD, reset_before=at if reset_before else None, async_device=name == "async_device")
        band.close()
        assert log == twin_log, name
    if not reset_before:
        band, log, _, _ = _device(engine, cfg, keyed, (FRAMES,), T0, PERIOD)
        band.close()
        assert log == twin_log, "one push"


def test_log_off_is_the_default_and_changes_nothing(engine, keyed):
    cfg = _keyed_config()
    on, log, res_on, _ = _device(engine, cfg, keyed, PUSHES, T0, PERIOD)
    off, none, res_off, _ = _device(engine, cfg, keyed, PUSHES, T0, PERIOD, log=False)
    assert log and off.get_events() == [] and off.event_count() == 0
    for a, b in zip(res_on, res_off):
        assert bytes(a) == bytes(b)
    assert on.get_transmissions() == off.get_transmissions()
    for x, y in zip(on.get_signals(), off.get_signals()):
        assert x.tobytes() == y.tobytes()
    for x, y in zip(on.get_averager()[:3], off.get_averager()[:3]):
        assert x.tobytes() == y.tobytes()
    for x, y in zip(on.get_spectrogram(), off.get_spectrogram()):
        assert len(x) > 0 and x.tobytes() == y.tobytes()
    # turning the log off keeps what it holds; the pushes after it add nothing
    on.set_event_log(True)
    on.push_raw(keyed.ctypes.data, 100, T0 + 2 * FRAMES, PERIOD)
    on.set_event_log(False)
    kept = on.get_events(consume=False)
    on.push_raw(keyed.ctypes.data, 300, T0 + 2 * (FRAMES + 100), PERIOD)
    assert on.get_events(consume=False) == kept
    on.close()
    off.close()


def test_consume(engine, keyed):
    band, _, _, _ = _device(engine, _keyed_config(), keyed, PUSHES, T0, PERIOD)
    # (_device has consumed the log: push the scene's start again, with a later clock)
    band.push_raw(keyed.ctypes.data, 512, T0 + 2 * FRAMES, PERIOD)
    total = band.event_count()
    assert total >= 4
    all_ev = band.get_events(consume=False)
    assert len(all_ev) == total == band.event_count()
    assert band.get_events(cap=3, consume=False) == all_ev[:3] and band.event_count() == total
    assert band.get_events(cap=3) == all_ev[:3] and band.event_count() == total - 3, "drops only what it copied"
    assert band.get_events(cap=0) == [] and band.event_count() == total - 3
    assert band.get_events() == all_ev[3:] and band.event_count() == 0
    band.close()


# ---------------------------------------------------------------------------------------------------------------
# overflow of the device log: N = 256 records per K4 launch
# ---------------------------------------------------------------------------------------------------------------
def test_a_full_device_log_reports_what_it_lost(engine):
    synth = _load_synth()
    n, learn, lengths = 256, 20, (40, 400, 50)
    cfg = b2s.make_config(n, FS, learn_frames=learn, recording_bandwidth_hz=16 * FS // n, min_time_ms=0, timeout_ms=0, max_frames_per_push=400)
    # timeout 0: every frame inserts the steady carrier's key and erases it again, two events per frame
    iq = synth.make_iq_int8(n, sum(lengths), [synth.Tone(bin_offset=40.1, amplitude=60.0, fm_dev_bins=3.0)], seed=synth.seed_for(8), quiet_frames=learn)
    want, twin_log, _ = _twin(engine, cfg, iq, lengths, T0, 1.0)
    assert want == [], "a key erased in the frame that inserted it is in no frame's list"
    for start, stop in zip(twin_log[0::2], twin_log[1::2]):  # the log alone shows it: its START, then its STOP
        assert (start[0], stop[0]) == (se.START, se.STOP) and start[1:6] == stop[1:6] and stop[6] == stop[4]
    band, log, _, launches = _device(engine, cfg, iq, lengths, T0, 1.0)
    band.close()
    assert launches == [1, 1, 1]
    per_push = [[e for e in twin_log if k <= e[3] < k + m] for k, m in _spans(lengths)]
    assert len(per_push[0]) <= n and len(per_push[1]) >= 2 * 390 and 0 < len(per_push[2]) <= n
    kept = per_push[1][:n]
    lost = (se.LOST, len(per_push[1]) - n, 0, kept[-1][3], kept[-1][4], 0, 0)
    assert log == per_push[0] + kept + [lost] + per_push[2]


# ---------------------------------------------------------------------------------------------------------------
# busy spectrum: pushes k_track runs, pushes it leaves to k_track_wide, and one it leaves after it has appended records
# ---------------------------------------------------------------------------------------------------------------
def test_busy_spectrum_across_the_hand_off(engine):
    case = Case("events_n16384", 16384, 20_000_000, 260, splits=(45, 70, 33, 1, 51, 30, 30), blocks=((-9.5e6, -3.0e6, 60, 130), (-1.0e6, 5.5e6, 90, 160), (6.0e6, 6.3e6, 205, 260)),
                n_carriers=120)  # two wide blocks take the map from 0 to several hundred keys and back; a narrow one follows, within k_track's caps
    n, cfg = case.n, case.config()
    iq = busy_iq(case, seed=4242)
    lengths = [m for _, _, m in case.pushes()]
    want, twin_log, outs = _twin(engine, cfg, iq, lengths, 500, 1.0, dense=("box_db", "avg_db"))
    band, log, _, launches = _device(engine, cfg, iq, lengths, 500, 1.0)
    band.close()
    assert log == twin_log
    assert all(e[0] in (se.START, se.STOP) for e in log)
    # (the per-frame lists are cut at MAX_TX entries, so here the twin's log is the yardstick, not the lists)
    # what each push met, from the twin: the live count before every frame's clearSignals, and the start-level candidates
    live, at = 0, 0
    abandoned, wide_from_start, small_after_wide, met = [], [], [], []
    seen_wide = False
    for i, ((k, m), out) in enumerate(zip(_spans(lengths), outs)):
        live_before = live
        first_over = None  # first frame of the push that k_track cannot finish
        first_event = None
        cand = (out.box_db >= np.float32(cfg.start_level)).sum(axis=1)
        cand[np.all(out.avg_db == np.float32(-1e30), axis=1) | np.all(np.isinf(out.avg_db), axis=1)] = 0
        for f in range(k, k + m):
            starts = stops = 0
            while at < len(log) and log[at][3] == f:
                starts += log[at][0] == se.START
                stops += log[at][0] == se.STOP
                at += 1
            if (starts or stops) and first_event is None:
                first_event = f
            if first_over is None and (live + starts > MAX_SIGNALS or cand[f - k] > MAX_CAND):
                first_over = f
            live += starts - stops
        met.append((k, live_before, first_event, first_over))
        if launches[i] == 2:
            seen_wide = True
            if live_before > MAX_SIGNALS:
                wide_from_start.append(i)
            elif first_event is not None and first_over is not None and first_event < first_over:
                abandoned.append(i)  # k_track had appended the records of first_event when it reached first_over
        elif seen_wide and first_event is not None:
            small_after_wide.append(i)
    print(f"\nlaunches per push {launches}; wide from the start {wide_from_start}, handed off after appending {abandoned}, k_track again {small_after_wide}")
    print("per push (first frame, live before, first event frame, first frame past k_track's caps):", met)
    assert launches[0] == 1 and wide_from_start and abandoned and small_after_wide, (launches, met)


def test_busy_spectrum_at_n1048576(engine):
    case = BUSY_CASES[2]
    assert case.n == 1048576
    cfg = case.config()
    iq = busy_iq(case, seed=777)
    lengths = [m for _, _, m in case.pushes()]
    _, twin_log, _ = _twin(engine, cfg, iq, lengths, 500, 1.0)
    band, log, _, launches = _device(engine, cfg, iq, lengths, 500, 1.0)
    band.close()
    assert log == twin_log and len(log) > 2 * MAX_SIGNALS
    assert 1 in launches and 2 in launches, launches  # k_track<12> and k_track_wide<12> both logged
