"""Auto-record without a GPU: the ctypes declarations follow include/b2s.h, NULL and bad arguments are refused before any CUDA call, and
the recorder assignment the band runs (ScanPolicy::update_recordings, through b2s_scan_policy_notify) gives the reference's actions, with
the map key the band reports for each, on the host tracker's lists of the fuzz scenes."""
import ctypes as C
import os
import re

import pytest

from conftest import ROOT, load_b2s
from test_host_tracker_fuzz import _scene

b2s = load_b2s()
import oracle_lib as ol  # noqa: E402


def declared(name):
    header = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "b2s.h")).read(), flags=re.S)
    m = re.search(r"\bint\s+" + name + r"\s*\(([^)]*)\)\s*;", header)
    assert m, f"{name} is not declared"
    return [re.sub(r"\s+", "", re.sub(r"\w+$", "", p.strip())) for p in m.group(1).split(",")]


def lib_or_skip():
    if not os.path.exists(b2s.LIB_PATH):
        pytest.skip("libb2s.so not built; run __graft_entry__.build()")
    return b2s.lib()


def test_bindings_match_the_header():
    assert declared("b2s_band_set_auto_record") == ["b2s_band*", "int", "int32_t"]
    assert declared("b2s_band_get_auto_record_actions") == ["b2s_band*", "b2s_auto_record_action*", "int", "int", "int*"]
    header = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "b2s.h")).read(), flags=re.S)
    body = re.search(r"typedef struct b2s_auto_record_action \{(.*?)\} b2s_auto_record_action;", header, re.S).group(1)
    fields = [tuple(f.split()) for f in body.replace("\n", " ").split(";") if f.strip()]
    sizes = {"int32_t": 4, "int64_t": 8}
    off = 0
    for (ctype, name), (py_name, py_type) in zip(fields, b2s.AutoRecordAction._fields_):
        assert name == py_name and C.sizeof(py_type) == sizes[ctype], name
        assert getattr(b2s.AutoRecordAction, name).offset == off, name
        off += sizes[ctype]
    assert len(fields) == len(b2s.AutoRecordAction._fields_) and C.sizeof(b2s.AutoRecordAction) == off == 48
    L = lib_or_skip()
    assert L.b2s_band_set_auto_record.argtypes == [C.c_void_p, C.c_int, C.c_int32] and L.b2s_band_set_auto_record.restype == C.c_int
    f = L.b2s_band_get_auto_record_actions
    assert f.argtypes == [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_int)] and f.restype == C.c_int
    assert callable(getattr(b2s.Band, "set_auto_record", None)) and callable(getattr(b2s.Band, "auto_record_actions", None))


def test_null_and_bad_arguments_are_refused():
    L = lib_or_skip()
    count = C.c_int(7)
    acts = (b2s.AutoRecordAction * 4)()
    assert L.b2s_band_set_auto_record(None, 1, 0) == -1
    assert L.b2s_band_set_auto_record(None, 0, 0) == -1
    assert L.b2s_band_set_auto_record(None, 1, -5) == -1
    assert L.b2s_band_get_auto_record_actions(None, C.cast(acts, C.c_void_p), 4, 1, C.byref(count)) == -1
    assert L.b2s_band_get_auto_record_actions(None, None, 0, 0, None) == -1
    assert count.value == 7


def reference_update_recordings(recorders, ignored, keys, now, mailbox):
    """SdrDevice::updateRecordings (sdr_device.cpp:82-144) restated, with the key the band reports: that of the list entry acted on,
    or for a STOP the key its recorder was started for. recorders[i] = [shift or None, first, last]."""
    out = []
    shifts = [s for s, _, _ in mailbox]
    for r, rec in enumerate(recorders):
        if rec[0] is not None and rec[0] not in shifts:
            out.append((b2s.REC_STOP, r, rec[0], keys[r], rec[2] - rec[1]))
            recorders[r] = [None, 0, 0]
    for shift, flush, key in mailbox:
        r = next((i for i, rec in enumerate(recorders) if rec[0] == shift), None)
        if r is not None:
            if flush:
                recorders[r][2] = now
                out.append((b2s.REC_FLUSH, r, shift, key, 0))
            continue
        f = next((i for i, rec in enumerate(recorders) if rec[0] is None), None)
        if f is not None:
            recorders[f] = [shift, now, now]
            keys[f] = key
            out.append((b2s.REC_START, f, shift, key, 0))
        elif shift not in ignored:
            ignored.add(shift)
            out.append((b2s.REC_NONE_FREE, -1, shift, key, 0))
    ignored.intersection_update(shifts)
    return out


@pytest.mark.parametrize("seed", range(0, 24, 3))
@pytest.mark.parametrize("n_rec", [1, 3])
def test_actions_on_the_fuzz_mailboxes(seed, n_rec):
    lib_or_skip()
    cfg, psd, frames, period = _scene(seed)
    r = ol.OracleChain(cfg).push(psd, frames, 0, period, dense=("noise_sub_db", "box_db"), psd_rows=True)
    lists = b2s.HostTransmission(cfg).push(r.box_db, r.noise_sub_db, 0, period, use_watch=True)
    pol = b2s.ScanPolicy([(cfg.range_lo_hz, cfg.range_hi_hz)], cfg.sample_rate_hz, n_rec, 500)
    recorders, ignored, keys = [[None, 0, 0] for _ in range(n_rec)], set(), [0] * n_rec
    seen = 0
    for k in range(0, frames, 5):  # one notification per push of 5 frames: the list after its last frame
        now = int((k + 4) * period)
        mailbox = [(s, f, key) for s, f, key, _ in lists[min(k + 4, frames - 1)]]
        acts, _ = pol.notify(now, [(s, f) for s, f, _ in mailbox])
        want = reference_update_recordings(recorders, ignored, keys, now, mailbox)
        assert [(a[0], a[1], a[2], a[4]) for a in want] == acts, (seed, k)
        seen += len(acts)
    assert seen > 0
