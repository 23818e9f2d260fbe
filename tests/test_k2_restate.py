"""CPU self-tests of tests/k2_restate.py, the exact float32 restatement of K2 that tests/test_k2_exact.py holds the engine to.

The restatement is pinned from two sides: with one segment per row its boxcar is the reference's serial average() bit for bit
(ol.cpu_average, itself pinned to the compiled reference and its golden record), and fed the oracle's own PSD rows its
NoiseLearner, Averager, serial boxcar and spectrogram equal the oracle chain's bit for bit."""
import numpy as np
import pytest

import k2_restate as k2
import oracle_lib as ol
from conftest import load_b2s
from test_gpu_parity import _window_mean64
from test_oracle_chain import scene

b2s = load_b2s()

GROUPS = [1, 2, 9, 20, 21, 33, 64, 65]
SIZES = [9, 100, 4097]


def _rows(size, seed):
    return (np.random.default_rng(seed).standard_normal((3, size)) * 20 - 7).astype(np.float32)


@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("group", GROUPS)
def test_one_segment_per_row_is_the_serial_reference_form(group, size):
    x = _rows(size, 100 * group + size)
    want = np.stack([ol.cpu_average(r, group) for r in x])
    assert k2.boxcar(x, group, segment=None).tobytes() == want.tobytes()
    assert k2.boxcar(x[0], group, segment=None).tobytes() == want[0].tobytes()


@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("group", GROUPS)
def test_engine_form_stays_within_the_design_bars(group, size):
    """16-bin segments change the rounding only: within 1e-3 of the serial form and 2e-5 of the float64 window mean."""
    x = _rows(size, 7 * group + size)
    got = k2.boxcar(x, group)
    assert np.max(np.abs(got - np.stack([ol.cpu_average(r, group) for r in x]))) <= 1e-3
    assert np.max(np.abs(got - np.stack([_window_mean64(r, group) for r in x]))) <= 2e-5


def test_engine_form_restarts_at_every_aligned_segment():
    """The first bin of each 16-bin segment is summed afresh: the same window values give the same bits whatever precedes them."""
    rng = np.random.default_rng(5)
    x = (rng.standard_normal(160) * 30).astype(np.float32)
    y = x.copy()
    y[:40] = (rng.standard_normal(40) * 1e4).astype(np.float32)  # bins 0..39 differ: segments from 64 on see windows >= 54
    a, b = k2.boxcar(x, 21), k2.boxcar(y, 21)
    assert a[64:].tobytes() == b[64:].tobytes()
    assert k2.boxcar(x, 21, segment=None)[64:].tobytes() != k2.boxcar(y, 21, segment=None)[64:].tobytes()


@pytest.mark.parametrize("learning_ms", [0, 30])
def test_restatement_equals_the_oracle_chain_on_its_own_psd_rows(learning_ms):
    """A scene with noise learning (by frame count or by noise_learning_ms), Averager warm-up, a reset between pushes and a
    decimating spectrogram, pushed in pieces: q, Averager rows and state, serial boxcar rows and spectrogram rows equal the oracle's."""
    n, frames = 256, 300
    cfg, tones, iq, period = scene(n=n, fs=1000 * n, frames=frames, learn=40)
    cfg.noise_learning_ms = learning_ms
    cfg.spectrogram_out_size, cfg.spectrogram_interval_ms = 64, 9
    o = ol.OracleChain(cfg)
    r = k2.K2Restatement(cfg, segment=None)
    k, sent = 0, []
    for i, m in enumerate([1, 5, 31, 32, 33, 97, 101]):
        if i == 5:
            o.reset(), r.reset()
        want = o.push(iq[k * 2 * n :], m, 500 + k, period)
        got = r.push(want.psd_db, 500 + k, period)
        assert got.q.tobytes() == want.noise_sub_db.tobytes(), (i, m)
        assert got.avg.tobytes() == want.avg_db.tobytes(), (i, m)
        assert got.box.tobytes() == want.box_db.tobytes(), (i, m)
        for a, b in zip(r.averager(), o.get_averager()):
            assert np.array_equal(a, b) and np.asarray(a).tobytes() == np.asarray(b).tobytes(), (i, m)
        thr, samples, ready = o.get_noise()
        assert r.noise()[0].tobytes() == thr.tobytes() and r.noise()[1:] == (samples, ready), (i, m)
        sent += got.spectrogram
        k += m
    assert r.ready
    t_o, _, rows_o = o.get_spectrogram(cap=256)
    assert len(sent) == len(t_o) >= 10
    assert [t for t, _ in sent] == t_o.tolist()
    assert np.stack([row for _, row in sent]).tobytes() == rows_o.tobytes()


def test_learning_and_warm_up_rows():
    """The rows a band reports while learning and while the Averager warms up, and the threshold it learns."""
    n = 64
    cfg = b2s.make_config(n, 1000 * n, learn_frames=3, spectrogram_out_size=0)
    cfg.grouping_y = 5
    psd = (np.random.default_rng(2).standard_normal((20, n)) * 3 - 60).astype(np.float32)
    r = k2.K2Restatement(cfg)
    a = r.push(psd[:2], 0, 1.0)
    assert r.noise()[1:] == (2, False)
    b = r.push(psd[2:], 2, 1.0)
    assert r.noise()[1:] == (3, True) and np.array_equal(r.threshold, psd[:3].max(axis=0))
    q = np.concatenate([a.q, b.q])
    assert np.all(q[:3] == -100.0) and q[3:].tobytes() == (psd[3:] - psd[:3].max(axis=0)).tobytes()
    avg = np.concatenate([a.avg, b.avg])
    assert np.all(avg[:4] == -100.0) and not np.any(avg[4:] == -100.0)
    assert avg[4].tobytes() == ((((np.float32(-300.0) + q[3]) + q[4]) / np.float32(5))).astype(np.float32).tobytes()
    assert np.array_equal(np.concatenate([a.entries, b.entries]), (k2.boxcar(avg, 21) >= 5.0).sum(axis=1))
