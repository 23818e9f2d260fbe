"""Sub-frame PSD rows without a GPU: the flags' values, the oracle's reduction at r = 1, and the scene properties that
test_subframe_psd.py relies on (so that its scene tests would fail on a band that ignores the flags)."""
import os
import re

import numpy as np

import oracle_lib as ol
import subframe_lib as sl
from conftest import ROOT, load_b2s

b2s = load_b2s()


def test_flag_values_match_header():
    text = open(os.path.join(ROOT, "include", "b2s.h")).read()
    for name in ("SUBFRAME_MEAN", "SUBFRAME_MAX", "ASYNC", "IQ_ON_DEVICE"):
        m = re.search(rf"#define B2S_FLAG_{name}\s+(0x[0-9a-fA-F]+)", text)
        assert m and int(m.group(1), 16) == getattr(b2s, f"FLAG_{name}"), name
    assert b2s.FLAG_SUBFRAME_MEAN & b2s.FLAG_SUBFRAME_MAX == 0


def test_reduction_order_and_r1():
    rng = np.random.default_rng(4)
    n = 1024
    cfg = b2s.make_config(n, 2_048_000)
    iq = np.clip(np.rint(rng.standard_normal(2 * n) * 20), -128, 127).astype(np.int8)
    ref_db, ref_lin = ol.oracle_psd_frame(cfg, iq, want_linear=True)
    for mode in (sl.MEAN, sl.MAX):
        db, lin = sl.orc_psd_frame_subframes(cfg, None, iq, 1, mode)
        assert np.array_equal(lin, ref_lin) and np.array_equal(db, ref_db), mode
    rows = rng.random((5, 64), dtype=np.float32)
    acc = rows[0]
    for p in rows[1:]:
        acc = (acc + p).astype(np.float32)
    assert np.array_equal(sl.reduce_lin(rows, sl.MEAN), (acc / np.float32(5)).astype(np.float32))
    assert np.array_equal(sl.reduce_lin(rows, sl.MAX), rows.max(axis=0))


def test_gap_scene_oracle():
    """A carrier silent in sub-frame 0 of every stride: only the sub-frame rows see it."""
    iq = sl.scene_iq(sl.GAP_ON, sl.GAP_AMP)
    assert [sl.oracle_outcome(b2s, iq, m) for m in (None, sl.MEAN, sl.MAX)] == [False, True, True]


def test_burst_scene_oracle():
    """A burst filling one sub-frame per stride: MAX reports it, the default chain does not."""
    iq = sl.scene_iq(sl.BURST_ON, sl.BURST_AMP)
    assert not sl.oracle_outcome(b2s, iq, None)
    assert sl.oracle_outcome(b2s, iq, sl.MAX)


def test_weak_carrier_oracle():
    """A continuous carrier below the default chain's start level and above MEAN's."""
    iq = sl.scene_iq(sl.WEAK_ON, sl.WEAK_AMP)
    assert not sl.oracle_outcome(b2s, iq, None)
    assert sl.oracle_outcome(b2s, iq, sl.MEAN)
