"""The signal event log without a GPU: the ABI surface, and the host tracker's log (b2s_host_transmission_get_events) against the
events derived from the oracle's per-frame lists on the fuzz scenes of test_host_tracker_fuzz.py."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

import oracle_lib as ol
import signal_events as se
from conftest import ROOT, load_b2s
from test_host_tracker_fuzz import _scene

b2s = load_b2s()


def test_the_mirror_matches_the_header():
    src = r"""
#include <stdio.h>
#include <stddef.h>
#include "b2s.h"
int main(void){
  printf("%zu %zu %zu %zu %d %d %d\n", sizeof(b2s_signal_event), offsetof(b2s_signal_event, frame), offsetof(b2s_signal_event, first_ms),
         offsetof(b2s_signal_event, last_ms), B2S_EV_START, B2S_EV_STOP, B2S_EV_LOST);
  return 0; }
"""
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "p.c"), "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", os.path.join(d, "p"), os.path.join(d, "p.c")])
        got = [int(x) for x in subprocess.check_output([os.path.join(d, "p")]).split()]
    E = b2s.SignalEvent
    assert got == [C.sizeof(E), E.frame.offset, E.first_ms.offset, E.last_ms.offset, b2s.EV_START, b2s.EV_STOP, b2s.EV_LOST]
    assert C.sizeof(E) == 48
    assert (se.START, se.STOP, se.LOST) == (b2s.EV_START, b2s.EV_STOP, b2s.EV_LOST)
    lib = C.CDLL(b2s.LIB_PATH)
    for name in ("b2s_band_set_event_log", "b2s_band_get_events", "b2s_host_transmission_get_events"):
        assert hasattr(lib, name), name


@pytest.mark.parametrize("seed", range(24))
def test_host_tracker_log_equals_the_oracle_lists(seed):
    cfg, psd, frames, period = _scene(seed)
    r = ol.OracleChain(cfg).push(psd, frames, 0, period, dense=("noise_sub_db", "box_db"), psd_rows=True)
    want = se.Expected().feed(r.frame_tx)
    _CHANGES.append(sum(len(a) + len(b) for _, a, b in want))
    logs = []
    for use_watch in (False, True):
        h = b2s.HostTransmission(cfg)
        h.push(r.box_db, r.noise_sub_db, 0, period, use_watch=use_watch)
        logs.append(h.get_events())
    h = b2s.HostTransmission(cfg)  # in chunks: `frame` goes on counting, the log is one sequence
    for a in range(0, frames, 37):
        b = min(frames, a + 37)
        h.push(r.box_db[a:b], r.noise_sub_db[a:b], int(a * period), period, use_watch=True)
    logs.append(h.get_events())
    for ev in logs:
        se.assert_log_equals(ev, want, f"seed {seed}")
        left = se.assert_times(ev, cfg.timeout_ms, cfg.max_time_ms, lambda f: int(np.floor(f * period + 0.5)))
        assert sorted(left) == sorted(se_keys(r.frame_tx[-1])), "the signals never stopped are the last frame's list"
    assert logs[0] == logs[1] == logs[2]
    assert h.get_events() == [], "consumed"


def se_keys(frame_list):
    return [k for _, _, k, _ in frame_list]


_CHANGES = []


def test_consume_and_reset():
    cfg, psd, frames, period = _scene(3)
    r = ol.OracleChain(cfg).push(psd, frames, 0, period, dense=("noise_sub_db", "box_db"), psd_rows=True)
    h = b2s.HostTransmission(cfg)
    h.push(r.box_db, r.noise_sub_db, 0, period)
    all_ev = h.get_events(consume=False)
    assert len(all_ev) >= 4 and h.get_events(consume=False) == all_ev
    assert h.get_events(cap=3) == all_ev[:3]            # drops only what it copied
    assert h.get_events(cap=0) == [] and h.get_events(consume=False) == all_ev[3:]
    h.reset()                                           # resetBuffers is silent and does not restart `frame`
    assert h.get_events() == all_ev[3:]
    h.push(r.box_db, r.noise_sub_db, 0, period)
    again = h.get_events()
    assert [(e[0], e[1], e[2], e[3] - frames) + e[4:] for e in again] == all_ev


def test_the_scenes_changed_their_maps():
    """Runs after the parametrised cases (file order)."""
    assert len(_CHANGES) == 24 and sum(1 for x in _CHANGES if x >= 6) >= 16, _CHANGES
