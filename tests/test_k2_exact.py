"""K2 (k_detect) bit for bit against tests/k2_restate.py at every launch variant, dense path and fast path alike.

Each case pushes the same IQ, split into the same pushes, through three bands with one config:
  A  the dense path: K2's noise, Averager and boxcar rows requested (every tile takes the generic march, levels on quotients);
  B  the fast path with host-tracked per-frame lists (only psd_db requested: steady tiles and sum thresholds stay on);
  C  the fast path with the device tracker K4, mailbox only (one case runs C with B2S_FLAG_ASYNC | B2S_FLAG_IQ_ON_DEVICE).
Every assertion compares two values computed from identical inputs, without tolerance: K1's PSD rows are the only input, and
the restatement is fed A's. The case matrix reaches every k_detect instantiation band.cuh can launch on a 132-SM H100; the
variant a case expects follows from the CTA-width rule of b2s_band::init, restated in k2_variant()."""
import ctypes as C
from dataclasses import dataclass
from typing import Optional, Sequence, Tuple

import numpy as np
import pytest

import k2_restate as k2
from conftest import load_b2s
from test_oracle_chain import synth

b2s = load_b2s()
pytestmark = pytest.mark.gpu

DENSE = ("psd_db", "noise_sub_db", "avg_db", "box_db")
SUM_THREADS = 160  # kSumThreads: the columns of a K2 CTA (bins + both halos)
INSTANTIATIONS = {"<21,10,152>", "<21,10,136>", "<21,10,56>", "<21,10>", "<0,-1>"}


def k2_variant(n: int, group_x: int, group_y: int, spec_out: int, sm_count: int) -> str:
    """The k_detect instantiation a band launches: b2s_band::init's CTA width, then band.cuh's dispatch on (X/2, Y, width)."""
    d = n // spec_out if spec_out > 0 else 1
    hp = (group_x // 2 + 3) & ~3
    fits = lambda b: b % d == 0 and b + 2 * hp <= SUM_THREADS
    waves = lambda b: (-(-n // b) + sm_count - 1) // sm_count
    bins = 0
    if n >= 8192:
        bins = next((b for b in (112, 128, 96, 64) if fits(b)), 0)
        if bins == 112 and fits(128) and waves(128) < waves(112):
            bins = 128
    else:
        bins = next((b for b in range(16, 129, 16) if fits(b) and -(-n // b) <= sm_count), 0)
        if not bins and fits(112):
            bins = 112
    assert bins, "no K2 CTA width fits this config"
    width = bins + 2 * hp
    if group_x // 2 == 10 and group_y == 21:
        return f"<21,10,{width}>" if width in (152, 136, 56) else "<21,10>"
    return "<0,-1>"


@dataclass
class Case:
    name: str
    n: int
    x: int = 21
    y: int = 21
    frames: int = 300
    learn: int = 40
    splits: Sequence[int] = (64, 100, 31, 32, 33, 97)
    levels: Optional[Tuple[float, float]] = None  # (start, stop); None: the reference's (8, 5)
    quantiles: Optional[Tuple[float, float]] = None  # (start, stop) as quantiles of the box values the restatement attains
    spec_out: int = 0  # 0: make_config's default (no decimation at fs = 1000 N)
    reset_at: Optional[int] = None  # index of the push before which every band is reset
    learning_ms: int = 0
    on_device_async: bool = False

    def config(self):
        n = self.n
        start, stop = self.levels or (8.0, 5.0)
        cfg = b2s.make_config(n, 1000 * n, learn_frames=self.learn, recording_bandwidth_hz=16_000, min_time_ms=20, timeout_ms=30, start_level=start,
                              stop_level=stop, spectrogram_out_size=self.spec_out or None, max_frames_per_push=512, detect_capacity=n,
                              noise_learning_ms=self.learning_ms)
        cfg.grouping_x, cfg.grouping_y = self.x, self.y
        cfg.spectrogram_interval_ms = 23
        return cfg

    def pushes(self):
        k, i = 0, 0
        while k < self.frames:
            m = min(self.splits[i % len(self.splits)], self.frames - k)
            yield i, k, m
            i += 1
            k += m


CASES = [
    # <21,10> with the runtime CTA width: 16-bin CTAs, and 64-bin CTAs with SPEC warps (d = 64)
    Case("n256", 256, splits=(1, 5, 31, 32, 33, 97)),
    Case("n1024_reset", 1024, splits=(97, 33, 32, 31, 5, 1, 101), reset_at=3),
    Case("n2048", 2048, splits=(32, 150, 118)),
    Case("n4096_d64", 4096, spec_out=64, splits=(70, 130, 100)),
    Case("x20_n1024", 1024, x=20, splits=(33, 97, 64, 106)),
    # <21,10,56>
    Case("n4096_learning_ms", 4096, learning_ms=45, splits=(32, 97, 171)),
    Case("x20_n4096_negative_stop", 4096, x=20, levels=(8.0, -1.0), splits=(64, 236)),
    # <21,10,136>: 74 CTAs, the last one owns 16 bins
    Case("n8192", 8192, splits=(31, 128, 141)),
    Case("x20_n8192", 8192, x=20, splits=(96, 204)),
    # <21,10,152>
    Case("n16384_async", 16384, splits=(64, 128, 108), on_device_async=True),
    Case("n16384_d128", 16384, spec_out=128, splits=(100, 200)),
    Case("n32768_two_waves", 32768, frames=260, splits=(96, 164)),
    Case("x20_n16384", 16384, x=20, splits=(33, 167, 100)),
    # levels on values the restated boxcar attains: real bins sit exactly on the >= boundary
    Case("levels_start_above_stop", 1024, quantiles=(0.995, 0.99), splits=(64, 236)),
    Case("levels_start_below_stop", 2048, quantiles=(0.99, 0.995), splits=(128, 172)),
    # <0,-1>: runtime X and Y
    Case("g1x1", 1024, x=1, y=1, splits=(5, 95, 200)),
    Case("g2x21", 4096, x=2, y=21, splits=(64, 236)),
    Case("g9x7", 1024, x=9, y=7, splits=(1, 31, 32, 33, 97, 106)),
    Case("g33x40", 4096, x=33, y=40, splits=(100, 200)),
    Case("g64x21", 1024, x=64, y=21, quantiles=(0.995, 0.99), splits=(64, 236)),
    Case("g65x3", 4096, x=65, y=3, levels=(5.0, 3.0), splits=(32, 268)),
    Case("g9x32_n16384", 16384, x=9, y=32, splits=(128, 172)),
    Case("y256_short_pushes", 1024, y=256, frames=480, splits=(100, 50, 200, 130)),
]


def _sm_count():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def _quantile_levels(engine, case, cfg, iq):
    """(start, stop) at quantiles of the non-warm-up box values the restatement computes from a probe band's PSD rows."""
    probe = b2s.Band(engine, cfg)
    rest, values = k2.K2Restatement(cfg), []
    for i, k, m in case.pushes():
        if i == case.reset_at:
            rest.reset()
        r = rest.push(probe.push(iq[k * 2 * case.n :], m, 500 + k, 1.0, dense=("psd_db",)).psd_db, 500 + k, 1.0)
        values.append(r.box[~np.all(r.avg == k2.NO_DATA, axis=1)].ravel())
    values = np.concatenate(values)
    return tuple(float(np.quantile(values, q, method="lower")) for q in case.quantiles)


def _mailbox(res):
    return [(t.shift_hz, t.flush, t.key, t.power) for t in res.transmissions[: res.n_transmissions]]


def _same(a, b):
    return np.asarray(a).dtype == np.asarray(b).dtype and np.asarray(a).shape == np.asarray(b).shape and np.asarray(a).tobytes() == np.asarray(b).tobytes()


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_k2_bit_exact_against_the_restatement(engine, case):
    sm = _sm_count()
    cfg = case.config()
    variant = k2_variant(case.n, case.x, case.y, cfg.spectrogram_out_size, sm)
    n = case.n
    iq = synth.make_iq_int8(n, case.frames, synth.standard_scene(n, case.frames, case.learn), seed=synth.seed_for(7, n + case.x), quiet_frames=case.learn)
    if case.quantiles:
        cfg.start_level, cfg.stop_level = _quantile_levels(engine, case, cfg, iq)
    print(f"\n{case.name}: k_detect{variant} on {sm} SMs, levels ({cfg.start_level:.9g}, {cfg.stop_level:.9g})")
    band_a, band_b = b2s.Band(engine, cfg), b2s.Band(engine, cfg)
    ccfg = b2s.BandConfig.from_buffer_copy(cfg)
    iq_dev = None
    if case.on_device_async:
        import torch

        ccfg.flags |= b2s.FLAG_ASYNC | b2s.FLAG_IQ_ON_DEVICE
        iq_dev = torch.from_numpy(iq).cuda()
    band_c = b2s.Band(engine, ccfg)
    bands = (band_a, band_b, band_c)
    host, rest = b2s.HostTransmission(cfg), k2.K2Restatement(cfg)
    stop = np.float32(cfg.stop_level)
    entries = below = listed = 0
    sent = []
    for i, k, m in case.pushes():
        if i == case.reset_at:
            for x in bands + (host, rest):
                x.reset()
        t0, part = 500 + k, iq[k * 2 * n :]
        a = band_a.push(part, m, t0, 1.0, dense=DENSE)
        b = band_b.push(part, m, t0, 1.0, per_frame=True, dense=("psd_db",))
        if iq_dev is not None:
            band_c.push_raw(iq_dev.data_ptr() + k * 2 * n, m, t0, 1.0)
            c = band_c.sync()
        else:
            psd_c = np.zeros((m, n), np.float32)
            c = b2s.Result()
            c.psd_db = psd_c.ctypes.data_as(C.POINTER(C.c_float))
            band_c.push_raw(part.ctypes.data, m, t0, 1.0, c)
            assert _same(psd_c, a.psd_db), (i, "psd C")
        where = (case.name, i, k, m)
        # 1. one input for everything below
        assert _same(a.psd_db, b.psd_db), where
        # 2. the dense rows
        r = rest.push(a.psd_db, t0, 1.0)
        assert _same(a.noise_sub_db, r.q), where
        assert _same(a.avg_db, r.avg), where
        assert _same(a.box_db, r.box), where
        # 3. noise and Averager state of every band
        want_thr, want_samples, want_ready = rest.noise()
        for name, band in zip("ABC", bands):
            thr, samples, ready = band.get_noise()
            assert _same(thr, want_thr) and (samples, ready) == (want_samples, want_ready), where + (name, "noise")
            for got, want in zip(band.get_averager(), rest.averager()):
                assert _same(got, want), where + (name, "averager")
        # 4. detection entries
        want_entries = int(r.entries.sum())
        assert (a.n_detect_entries, b.n_detect_entries, c.n_detect_entries) == (want_entries,) * 3, where
        entries += want_entries
        # 5. the fast path's per-frame lists against the host tracker on the restated rows
        lists = host.push(r.box, r.q, t0, 1.0)
        for f in range(m):
            assert b.frame_tx[f] == lists[f], where + (f, b.frame_tx[f], lists[f])
        listed += sum(len(x) for x in lists)
        below += sum(1 for x in lists for t in x if np.float32(t[3]) < stop)
        # 6. the device tracker's mailbox after the push
        assert _mailbox(c) == lists[-1], where
        sent += r.spectrogram
    for x, y in zip(band_b.get_signals(), band_c.get_signals()):
        assert _same(x, y), case.name
    # 7. spectrogram rows and times
    for name, band in zip("ABC", bands):
        times, _, rows = band.get_spectrogram(cap=4096)
        assert times.tolist() == [t for t, _ in sent], (case.name, name)
        assert _same(rows, np.stack([row for _, row in sent]).reshape(len(sent), -1)), (case.name, name)
    print(f"  {case.frames} frames: {entries} detection entries, {listed} list records, {below} below stop_level, {len(sent)} spectrogram rows")
    assert entries > 0 and listed > 0 and len(sent) >= 5
    assert below > 0, "the scene never shows a live signal below stop_level"


def test_the_case_matrix_reaches_every_k_detect_instantiation():
    """N = 16384 launches <21,10,152> only where 128-bin CTAs need fewer waves than 112-bin ones (>= 128 SMs)."""
    sm = _sm_count()
    if sm < 128:
        pytest.skip(f"{sm} SMs: N = 16384 takes 112-bin CTAs here, so k_detect<21,10,152> is never launched")
    reached = {}
    for case in CASES:
        v = k2_variant(case.n, case.x, case.y, case.config().spectrogram_out_size, sm)
        reached.setdefault(v, []).append(case.name)
    for v in sorted(reached):
        print(f"\nk_detect{v}: {', '.join(reached[v])}")
    assert set(reached) == INSTANTIATIONS


@pytest.mark.parametrize("size", [9, 100, 4097])
@pytest.mark.parametrize("group", [1, 2, 9, 20, 21, 33, 64, 65])
def test_device_average_equals_the_engine_form(engine, group, size):
    """b2s_average(exact=0) is the engine's boxcar (k_boxcar, boxcar_value): bit for bit the restated form."""
    x = (np.random.default_rng(31 * group + size).standard_normal((3, size)) * 20 - 7).astype(np.float32)
    assert _same(engine.average(x, group, exact=False), k2.boxcar(x, group))
    assert _same(engine.average(x, group, exact=True), k2.boxcar(x, group, segment=None))
