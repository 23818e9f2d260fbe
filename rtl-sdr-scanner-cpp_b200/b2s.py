"""ctypes binding of the b2s C-ABI (include/b2s.h) — the Python face of the drop-in boundary.

Mirrors the reference's operator surface for the hot path (Averager, average(), the Decimator..Transmission chain of
sources/radio/sdr_device.cpp:161-171) so that parity tests read like the reference's own unit tests
(tests/test_averager.cpp, tests/test_utils.cpp). There is NO fallback here: if the CUDA library is missing or no
H100 is visible, loading / engine creation raises.
"""
from __future__ import annotations

import ctypes as C
import os
import weakref
from typing import NamedTuple, Optional

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("B2S_LIB") or os.path.join(_HERE, "lib", "libb2s.so")  # B2S_LIB: an A/B build of the same ABI (measurements)

MAX_IGNORED = 16
MAX_TX = 64
IQ_CS8, IQ_CF32 = 0, 1
FLAG_IQ_ON_DEVICE = 0x100
FLAG_ASYNC = 0x200
FLAG_SUBFRAME_MEAN = 0x400  # a frame's PSD row is the mean of its stride's floor(stride / N) sub-frame periodograms (include/b2s.h)
FLAG_SUBFRAME_MAX = 0x800   # ... or their per-bin maximum; make_config(flags=...) and Engine.psd pass them through
FLAG_SUBFRAME_OVERLAP = 0x1000  # with MEAN or MAX: stride / (N / 2) sub-frames overlapping by half; Engine.psd then reads a lead-in


class BandConfig(C.Structure):
    """b2s_band_config (also layout-compatible with the oracle's orc_config prefix)."""

    _fields_ = [
        ("fft_size", C.c_int32),
        ("sample_rate_hz", C.c_int32),
        ("frame_stride_samples", C.c_int32),
        ("iq_format", C.c_int32),
        ("iq_scale", C.c_float),
        ("window_kind", C.c_int32),
        ("window_taps", C.POINTER(C.c_float)),
        ("grouping_x", C.c_int32),
        ("grouping_y", C.c_int32),
        ("group_size_bins", C.c_int32),
        ("start_level", C.c_float),
        ("stop_level", C.c_float),
        ("learn_frames", C.c_int32),
        ("center_hz", C.c_int32),
        ("range_lo_hz", C.c_int32),
        ("range_hi_hz", C.c_int32),
        ("n_ignored", C.c_int32),
        ("ignored_lo_hz", C.c_int32 * MAX_IGNORED),
        ("ignored_hi_hz", C.c_int32 * MAX_IGNORED),
        ("tuning_step_hz", C.c_int32),
        ("min_time_ms", C.c_int64),
        ("timeout_ms", C.c_int64),
        ("max_time_ms", C.c_int64),
        ("spectrogram_out_size", C.c_int32),
        ("spectrogram_interval_ms", C.c_int64),
        ("flags", C.c_int32),
        ("max_frames_per_push", C.c_int32),
        ("detect_capacity", C.c_int32),
        ("noise_learning_ms", C.c_int64),
    ]


class Transmission(C.Structure):
    _fields_ = [("shift_hz", C.c_int32), ("flush", C.c_int32), ("key", C.c_int32), ("power", C.c_float)]


EV_START, EV_STOP, EV_LOST = 1, 2, 3


class SignalEvent(C.Structure):
    """b2s_signal_event: one change of the signal map (for EV_LOST, `key` events that did not fit the device log)."""

    _fields_ = [("kind", C.c_int32), ("key", C.c_int32), ("shift_hz", C.c_int32), ("reserved", C.c_int32), ("frame", C.c_int64), ("time_ms", C.c_int64),
                ("first_ms", C.c_int64), ("last_ms", C.c_int64)]

    def astuple(self):
        return (self.kind, self.key, self.shift_hz, self.frame, self.time_ms, self.first_ms, self.last_ms)


class AutoRecordAction(C.Structure):
    """b2s_auto_record_action: what an auto-recording band did to its bank after one push (kind: REC_START / STOP / FLUSH / NONE_FREE)."""

    _fields_ = [("kind", C.c_int32), ("channel", C.c_int32), ("shift_hz", C.c_int32), ("key", C.c_int32), ("frame", C.c_int64), ("from_frame", C.c_int64),
                ("time_ms", C.c_int64), ("duration_ms", C.c_int64)]

    def astuple(self):
        return (self.kind, self.channel, self.shift_hz, self.key, self.frame, self.from_frame, self.time_ms, self.duration_ms)


class Result(C.Structure):
    _fields_ = [
        ("n_transmissions", C.c_int32),
        ("transmissions", Transmission * MAX_TX),
        ("frame_tx_count", C.POINTER(C.c_int32)),
        ("frame_tx", C.POINTER(Transmission)),
        ("peak_index", C.POINTER(C.c_int32)),
        ("peak_value", C.POINTER(C.c_float)),
        ("psd_db", C.POINTER(C.c_float)),
        ("noise_sub_db", C.POINTER(C.c_float)),
        ("avg_db", C.POINTER(C.c_float)),
        ("box_db", C.POINTER(C.c_float)),
        ("n_detect_entries", C.c_int32),
        ("n_spectrogram_rows", C.c_int32),
        ("n_transmissions_total", C.c_int32),
    ]


class Profile(C.Structure):
    _fields_ = [
        ("spectral_ms", C.c_double),
        ("detect_ms", C.c_double),
        ("window_ms", C.c_double),
        ("tracker_host_ms", C.c_double),
        ("spectral_launches", C.c_int64),
        ("detect_launches", C.c_int64),
        ("window_launches", C.c_int64),
        ("pushes", C.c_int64),
        ("frames", C.c_int64),
        ("h2d_bytes", C.c_int64),
        ("d2h_bytes", C.c_int64),
        ("detect_cta_median_ms", C.c_double),
        ("detect_cta_max_ms", C.c_double),
        ("track_ms", C.c_double),
        ("track_launches", C.c_int64),
        ("track_evals", C.c_int64),
        ("track_events", C.c_int64),
        ("track_best_index", C.c_int64),
    ]


def make_config(
    fft_size: int,
    sample_rate_hz: int,
    center_hz: int = 100_000_000,
    *,
    decimator: int = 1,
    iq_format: int = IQ_CS8,
    iq_scale: float = 1.0 / 127.0,
    recording_bandwidth_hz: int = 32000,
    group_size_bins: Optional[int] = None,
    start_level: float = 8.0,
    stop_level: float = 5.0,
    learn_frames: int = 100,
    tuning_step_hz: int = 2500,
    min_time_ms: int = 2000,
    timeout_ms: int = 2000,
    max_time_ms: int = 600_000,
    spectrogram_out_size: Optional[int] = None,
    ignored=(),
    range_hz=None,
    max_frames_per_push: int = 0,
    detect_capacity: int = 0,
    flags: int = 0,
    noise_learning_ms: int = 0,
) -> BandConfig:
    """Reference defaults (config.h:24-38, config.example.json:9-13, sdr_device.cpp:148-152) for an explicit N."""
    import math

    cfg = BandConfig()
    cfg.fft_size = fft_size
    cfg.sample_rate_hz = sample_rate_hz
    cfg.frame_stride_samples = fft_size * decimator
    cfg.iq_format = iq_format
    cfg.iq_scale = iq_scale
    cfg.window_kind = 0
    cfg.grouping_x = 21
    cfg.grouping_y = 21
    step = sample_rate_hz / fft_size
    cfg.group_size_bins = group_size_bins if group_size_bins is not None else int(math.ceil(recording_bandwidth_hz / step))
    cfg.start_level = start_level
    cfg.stop_level = stop_level
    cfg.learn_frames = learn_frames
    cfg.center_hz = center_hz
    lo, hi = range_hz if range_hz is not None else (center_hz - sample_rate_hz // 2, center_hz + sample_rate_hz // 2)
    cfg.range_lo_hz, cfg.range_hi_hz = lo, hi
    cfg.n_ignored = len(ignored)
    for i, (a, b) in enumerate(ignored):
        cfg.ignored_lo_hz[i], cfg.ignored_hi_hz[i] = a, b
    cfg.tuning_step_hz = tuning_step_hz
    cfg.min_time_ms, cfg.timeout_ms, cfg.max_time_ms = min_time_ms, timeout_ms, max_time_ms
    if spectrogram_out_size is None:
        n = 1
        while 1000 < sample_rate_hz / n:  # getFft(fs, SPECTROGRAM_PREFERRED_MAX_STEP), radio_utils.cpp:98-104
            n <<= 1
        spectrogram_out_size = min(16384, n, fft_size)
    cfg.spectrogram_out_size = spectrogram_out_size
    cfg.spectrogram_interval_ms = 1000
    cfg.flags = flags
    cfg.max_frames_per_push = max_frames_per_push
    cfg.detect_capacity = detect_capacity
    cfg.noise_learning_ms = noise_learning_ms  # 0: learn_frames frames per centre; > 0: the reference's wall-clock rule (noise_learner.cpp:23)
    return cfg


class B2SError(RuntimeError):
    pass


_lib = None


def lib():
    """Load libb2s.so (built by __graft_entry__.build()); fails loudly when it is absent."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise B2SError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` (no CPU fallback exists)")
        L = C.CDLL(LIB_PATH)
        L.b2s_last_error.restype = C.c_char_p
        L.b2s_get_tuned_frequency.restype = C.c_int32
        L.b2s_band_push.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int64, C.c_double, C.POINTER(Result)]
        L.b2s_engine_create.argtypes = [C.c_int, C.POINTER(C.c_void_p)]
        L.b2s_engine_destroy.argtypes = [C.c_void_p]
        L.b2s_engine_device_name.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t]
        L.b2s_band_create.argtypes = [C.c_void_p, C.POINTER(BandConfig), C.POINTER(C.c_void_p)]
        L.b2s_band_destroy.argtypes = [C.c_void_p]
        L.b2s_band_set_stream.argtypes = [C.c_void_p, C.c_void_p]
        L.b2s_band_attach_recorder_bank.argtypes = [C.c_void_p, C.c_void_p]
        L.b2s_band_attach_recorder_bank.restype = C.c_int
        L.b2s_band_reset.argtypes = [C.c_void_p]
        L.b2s_band_sync.argtypes = [C.c_void_p, C.POINTER(Result)]
        L.b2s_band_set_profiling.argtypes = [C.c_void_p, C.c_int]
        L.b2s_band_get_profile.argtypes = [C.c_void_p, C.POINTER(Profile), C.c_int]
        L.b2s_band_set_center.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32]
        L.b2s_band_get_averager.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int32)]
        L.b2s_band_get_noise.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
        L.b2s_band_get_spectrogram.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_int)]
        L.b2s_band_get_transmissions.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.POINTER(C.c_int)]
        L.b2s_band_get_signals.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.POINTER(C.c_int)]
        L.b2s_band_set_event_log.argtypes = [C.c_void_p, C.c_int]
        L.b2s_recorder_bank_set_history.argtypes = [C.c_void_p, C.c_size_t]
        L.b2s_recorder_bank_history.argtypes = [C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
        L.b2s_recorder_bank_start_from.argtypes = [C.c_void_p, C.c_int, C.c_int32, C.c_int64, C.c_int64]
        L.b2s_band_record_from.argtypes = [C.c_void_p, C.c_int, C.c_int32, C.c_int64]
        L.b2s_band_set_auto_record.argtypes = [C.c_void_p, C.c_int, C.c_int32]
        L.b2s_band_get_auto_record_actions.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_int)]
        L.b2s_band_set_occupancy.argtypes = [C.c_void_p, C.c_int]
        L.b2s_band_occupancy_centers.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.POINTER(C.c_int)]
        L.b2s_band_get_occupancy.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64),
                                             C.POINTER(C.c_int64), C.c_int]
        for f in ("b2s_recorder_bank_set_history", "b2s_recorder_bank_history", "b2s_recorder_bank_start_from", "b2s_band_record_from",
                  "b2s_band_set_auto_record", "b2s_band_get_auto_record_actions", "b2s_band_set_occupancy", "b2s_band_occupancy_centers",
                  "b2s_band_get_occupancy"):
            getattr(L, f).restype = C.c_int
        for f in ("b2s_band", "b2s_recorder_bank"):
            getattr(L, f + "_save_state").argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
            getattr(L, f + "_save_state").restype = C.c_int
            getattr(L, f + "_load_state").argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
            getattr(L, f + "_load_state").restype = C.c_int
        for f in ("b2s_band_get_events", "b2s_host_transmission_get_events"):
            getattr(L, f).argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_int)]
        L.b2s_averager_create.argtypes = [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_void_p)]
        L.b2s_averager_destroy.argtypes = [C.c_void_p]
        L.b2s_averager_push.argtypes = [C.c_void_p, C.c_void_p]
        L.b2s_averager_push_many.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        L.b2s_averager_reset.argtypes = [C.c_void_p]
        L.b2s_averager_average.argtypes = [C.c_void_p, C.c_void_p]
        L.b2s_averager_data.argtypes = [C.c_void_p, C.c_void_p]
        L.b2s_averager_sum.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_int32)]
        L.b2s_average.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int]
        L.b2s_psd.argtypes = [C.c_void_p, C.POINTER(BandConfig), C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
        L.b2s_get_max_index.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int]
        L.b2s_contains_with_margin.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int)]
        L.b2s_most_frequent_value.argtypes = [C.c_void_p, C.c_int]
        L.b2s_learn_frames_from_ms.argtypes = [C.c_int64, C.c_double]
        L.b2s_host_transmission_create.argtypes = [C.POINTER(BandConfig), C.POINTER(C.c_void_p)]
        L.b2s_host_transmission_destroy.argtypes = [C.c_void_p]
        L.b2s_host_transmission_reset.argtypes = [C.c_void_p]
        L.b2s_host_transmission_last_run_ms.argtypes = [C.c_void_p]
        L.b2s_host_transmission_last_run_ms.restype = C.c_double
        L.b2s_host_transmission_push.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int64, C.c_double, C.c_int, C.c_void_p, C.c_void_p]
        for f in ("b2s_pack_spectrogram_message", "b2s_pack_transmission_message"):
            getattr(L, f).argtypes = [C.c_int64, C.c_int32, C.c_int32, C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
        L.b2s_default_config.argtypes = [C.POINTER(BandConfig), C.c_int32, C.c_int32, C.c_int32]
        L.b2s_default_config.restype = None
        _lib = L
    return _lib


def _check(rc: int):
    if rc != 0:
        raise B2SError(f"b2s error {rc}: {lib().b2s_last_error().decode(errors='replace')}")


def _ptr(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _save_state(fn, handle) -> bytes:
    """A b2s_*_save_state snapshot: one call for the size (it returns B2S_E_INVALID with the size), one for the bytes."""
    need = C.c_size_t(0)
    rc = fn(handle, None, 0, C.byref(need))
    if need.value == 0:
        _check(rc)
    buf = np.empty(need.value, np.uint8)
    _check(fn(handle, _ptr(buf), buf.size, C.byref(need)))
    return buf[: need.value].tobytes()


def _load_state(fn, handle, data) -> None:
    data = bytes(data)
    buf = np.frombuffer(data or b"\0", np.uint8)
    _check(fn(handle, _ptr(buf), len(data)))


def _get_events(fn, handle, cap: int, consume: bool):
    """(the oldest `cap` events as (kind, key, shift_hz, frame, time_ms, first_ms, last_ms), the number that were queued)"""
    ev = (SignalEvent * max(cap, 1))()
    count = C.c_int()
    _check(fn(handle, C.cast(ev, C.c_void_p), cap, 1 if consume else 0, C.byref(count)))
    return [ev[i].astuple() for i in range(min(count.value, cap))], count.value


class _Handle:
    """Owns one C-ABI handle `_h`: close() (or garbage collection) passes it to its b2s_*_destroy function once."""

    def __init__(self, destroy):
        self._h = C.c_void_p()
        self._destroy = destroy

    def close(self):
        if self._h:
            self._destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Engine(_Handle):
    """b2s_engine: one per GPU (reference analogue: the process that owns the SdrDevice chains)."""

    def __init__(self, cuda_device: int = 0):
        super().__init__(lib().b2s_engine_destroy)
        _check(lib().b2s_engine_create(cuda_device, C.byref(self._h)))

    def device_name(self) -> str:
        buf = C.create_string_buffer(256)
        _check(lib().b2s_engine_device_name(self._h, buf, 256))
        return buf.value.decode()

    def check_div_const(self, divisor: int) -> int:
        """Mismatches of the engine's exact constant division against IEEE division over its whole guarded range (must be 0)."""
        bad = C.c_uint64()
        lib().b2s_selftest_div_const.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_uint64)]
        _check(lib().b2s_selftest_div_const(self._h, divisor, C.byref(bad)))
        return bad.value

    # ---- stand-alone operators ----
    def average(self, data: np.ndarray, group_size: int, exact: bool = False) -> np.ndarray:
        """average(in, out, size, groupSize), sources/utils/utils.cpp:31-53, row-wise on the GPU."""
        x = np.ascontiguousarray(data, dtype=np.float32)
        rows = 1 if x.ndim == 1 else x.shape[0]
        size = x.shape[-1]
        out = np.empty_like(x)
        _check(lib().b2s_average(self._h, _ptr(x), _ptr(out), size, group_size, rows, 1 if exact else 0))
        return out

    def psd(self, cfg: BandConfig, iq: np.ndarray, n_frames: int, want_linear: bool = False):
        n = cfg.fft_size
        psd = np.empty((n_frames, n), dtype=np.float32)
        lin = np.empty((n_frames, n), dtype=np.float32) if want_linear else None
        iq = np.ascontiguousarray(iq)
        if cfg.flags & FLAG_SUBFRAME_OVERLAP:
            # N / 2 lead-in samples, then every frame's whole stride (include/b2s.h)
            need = (n // 2 + n_frames * cfg.frame_stride_samples) * (2 if cfg.iq_format == IQ_CS8 else 8)
            if iq.nbytes < need:
                raise ValueError(f"overlapping sub-frames read {need} bytes of IQ; {iq.nbytes} were given")
        _check(lib().b2s_psd(self._h, C.byref(cfg), _ptr(iq), n_frames, _ptr(psd), _ptr(lin)))
        return (psd, lin) if want_linear else psd


class Averager(_Handle):
    """Device-backed Averager with the reference's surface (sources/radio/averager.h:8-28)."""

    def __init__(self, engine: Engine, size: int, group_size: int):
        super().__init__(lib().b2s_averager_destroy)
        self._e = engine
        self.size, self.group_size = size, group_size
        _check(lib().b2s_averager_create(engine._h, size, group_size, C.byref(self._h)))

    def push(self, data):
        x = np.ascontiguousarray(data, dtype=np.float32)
        if x.ndim == 2:
            _check(lib().b2s_averager_push_many(self._h, _ptr(x), x.shape[0]))
        else:
            assert x.shape[0] == self.size
            _check(lib().b2s_averager_push(self._h, _ptr(x)))

    def reset(self):
        _check(lib().b2s_averager_reset(self._h))

    def average(self) -> np.ndarray:
        out = np.empty(self.size, dtype=np.float32)
        _check(lib().b2s_averager_average(self._h, _ptr(out)))
        return out

    def data(self) -> np.ndarray:
        out = np.empty((self.group_size, self.size), dtype=np.float32)
        _check(lib().b2s_averager_data(self._h, _ptr(out)))
        return out

    def sum(self):
        out = np.empty(self.size, dtype=np.float32)
        frames = C.c_int32()
        _check(lib().b2s_averager_sum(self._h, _ptr(out), C.byref(frames)))
        return out, frames.value


class Occupancy(NamedTuple):
    """One centre's spectrum occupancy (b2s_band_get_occupancy). above_start / detect_frames is each bin's duty cycle at the start
    level; while `truncated` is nonzero the counts are lower bounds."""
    above_start: np.ndarray  # uint32 [N]
    above_stop: np.ndarray   # uint32 [N]
    max_db: np.ndarray       # float32 [N]
    frames: int
    detect_frames: int
    truncated: int


class PushOutput:
    """Host-side view of one b2s_band_push result."""

    def __init__(self):
        self.transmissions = []  # [(shift_hz, flush, key, power)] after the last frame
        self.frame_tx = None  # list per frame of [(shift_hz, flush, key, power)]
        self.peak_index = None
        self.peak_value = None
        self.psd_db = self.noise_sub_db = self.avg_db = self.box_db = None
        self.n_detect_entries = 0
        self.n_spectrogram_rows = 0


class Band(_Handle):
    """b2s_band: the GPU replacement of one device's decimator..transmission(+spectrogram) chain."""

    def __init__(self, engine: Engine, cfg: BandConfig):
        super().__init__(lib().b2s_band_destroy)
        self._e = engine
        self.cfg = cfg
        self._bank = None
        _check(lib().b2s_band_create(engine._h, C.byref(cfg), C.byref(self._h)))

    def close(self):
        """b2s_band_destroy: an attached bank is detached first and stays usable on its own."""
        super().close()
        if self._bank is not None:
            self._bank._band = None
            self._bank = None

    def attach_recorder_bank(self, bank: Optional["RecorderBank"]):
        """b2s_band_attach_recorder_bank: every later push also runs `bank` over the pushed stream (one upload for both); None
        detaches. The band keeps the bank alive while it is attached."""
        _check(lib().b2s_band_attach_recorder_bank(self._h, bank._h if bank is not None else None))
        if self._bank is not None:
            self._bank._band = None
        self._bank = bank
        if bank is not None:
            bank._band = weakref.ref(self)

    def set_stream(self, cuda_stream: int):
        _check(lib().b2s_band_set_stream(self._h, C.c_void_p(cuda_stream)))

    def push_raw(self, iq_ptr: int, n_frames: int, t0_ms: int, frame_period_ms: float, res: Optional[Result] = None) -> Optional[Result]:
        """Thin call with a raw pointer (host or device per cfg.flags); used by bench.py. In async mode (FLAG_ASYNC) no
        result structure is passed; collect with sync()."""
        if self.cfg.flags & FLAG_ASYNC:
            _check(lib().b2s_band_push(self._h, C.c_void_p(iq_ptr), n_frames, t0_ms, frame_period_ms, None))
            return None
        if res is None:
            res = Result()
        _check(lib().b2s_band_push(self._h, C.c_void_p(iq_ptr), n_frames, t0_ms, frame_period_ms, C.byref(res)))
        return res

    def sync(self, res: Optional[Result] = None) -> Result:
        """b2s_band_sync: wait for outstanding asynchronous pushes; returns the mailbox after the last frame pushed."""
        if res is None:
            res = Result()
        _check(lib().b2s_band_sync(self._h, C.byref(res)))
        return res

    def push(self, iq: np.ndarray, n_frames: int, t0_ms: int, frame_period_ms: float, *, per_frame: bool = False, dense=()) -> PushOutput:
        n = self.cfg.fft_size
        iq = np.ascontiguousarray(iq)
        res = Result()
        keep = []
        out = PushOutput()
        if per_frame:
            cnt = np.zeros(n_frames, dtype=np.int32)
            tx = (Transmission * (n_frames * MAX_TX))()
            pk = np.zeros(n_frames, dtype=np.int32)
            pv = np.zeros(n_frames, dtype=np.float32)
            res.frame_tx_count = cnt.ctypes.data_as(C.POINTER(C.c_int32))
            res.frame_tx = C.cast(tx, C.POINTER(Transmission))
            res.peak_index = pk.ctypes.data_as(C.POINTER(C.c_int32))
            res.peak_value = pv.ctypes.data_as(C.POINTER(C.c_float))
            keep += [cnt, tx, pk, pv]
        for name in dense:
            arr = np.zeros((n_frames, n), dtype=np.float32)
            setattr(res, name, arr.ctypes.data_as(C.POINTER(C.c_float)))
            setattr(out, name, arr)
        _check(lib().b2s_band_push(self._h, _ptr(iq), n_frames, t0_ms, frame_period_ms, C.byref(res)))
        out.transmissions = [(t.shift_hz, t.flush, t.key, t.power) for t in res.transmissions[: res.n_transmissions]]
        if per_frame:
            out.frame_tx = []
            for k in range(n_frames):
                base = k * MAX_TX
                out.frame_tx.append([(tx[base + s].shift_hz, tx[base + s].flush, tx[base + s].key, tx[base + s].power) for s in range(min(cnt[k], MAX_TX))])
            out.peak_index, out.peak_value = pk, pv
        out.n_detect_entries = res.n_detect_entries
        out.n_spectrogram_rows = res.n_spectrogram_rows
        return out

    def set_profiling(self, enable=True):
        """False/0 = off, True/1 = kernel times and byte counts, 2 = also the per-CTA run times of K2."""
        _check(lib().b2s_band_set_profiling(self._h, int(enable)))

    def get_profile(self, reset: bool = True) -> Profile:
        p = Profile()
        _check(lib().b2s_band_get_profile(self._h, C.byref(p), 1 if reset else 0))
        return p

    def reset(self):
        _check(lib().b2s_band_reset(self._h))

    def set_center(self, center_hz: int, lo: int, hi: int):
        _check(lib().b2s_band_set_center(self._h, center_hz, lo, hi))

    def get_averager(self):
        n, y = self.cfg.fft_size, self.cfg.grouping_y
        s = np.empty(n, dtype=np.float32)
        a = np.empty(n, dtype=np.float32)
        r = np.empty((y, n), dtype=np.float32)
        f = C.c_int32()
        _check(lib().b2s_band_get_averager(self._h, _ptr(s), _ptr(a), _ptr(r), C.byref(f)))
        return s, a, r, f.value

    def get_noise(self):
        thr = np.empty(self.cfg.fft_size, dtype=np.float32)
        samples, ready = C.c_int32(), C.c_int32()
        _check(lib().b2s_band_get_noise(self._h, _ptr(thr), C.byref(samples), C.byref(ready)))
        return thr, samples.value, bool(ready.value)

    def get_spectrogram(self, cap: int = 64, consume: bool = True):
        m = self.cfg.spectrogram_out_size
        times = np.zeros(cap, dtype=np.int64)
        centers = np.zeros(cap, dtype=np.int32)
        rows = np.zeros((cap, max(m, 1)), dtype=np.int8)
        count = C.c_int()
        _check(lib().b2s_band_get_spectrogram(self._h, _ptr(times), _ptr(centers), _ptr(rows), cap, 1 if consume else 0, C.byref(count)))
        k = min(count.value, cap)
        return times[:k], centers[:k], rows[:k]

    def get_transmissions(self, cap: int = 4096):
        """The complete mailbox after the last finished push, strongest first: [(shift_hz, flush, key, power)]."""
        tx = (Transmission * cap)()
        count = C.c_int()
        _check(lib().b2s_band_get_transmissions(self._h, C.cast(tx, C.c_void_p), cap, C.byref(count)))
        return [(tx[i].shift_hz, tx[i].flush, tx[i].key, tx[i].power) for i in range(min(count.value, cap))]

    def get_signals(self, cap: int = MAX_TX):
        keys = np.zeros(cap, dtype=np.int32)
        first = np.zeros(cap, dtype=np.int64)
        last = np.zeros(cap, dtype=np.int64)
        power = np.zeros(cap, dtype=np.float32)
        count = C.c_int()
        _check(lib().b2s_band_get_signals(self._h, _ptr(keys), _ptr(first), _ptr(last), _ptr(power), cap, C.byref(count)))
        k = min(count.value, cap)
        return keys[:k], first[:k], last[:k], power[:k]

    def set_event_log(self, enable: bool = True):
        """b2s_band_set_event_log: log every start and stop of a transmission in the pushes after this call."""
        _check(lib().b2s_band_set_event_log(self._h, 1 if enable else 0))

    def get_events(self, cap: int = 65536, consume: bool = True):
        """The oldest `cap` signal events of the finished pushes: [(kind, key, shift_hz, frame, time_ms, first_ms, last_ms)]."""
        return _get_events(lib().b2s_band_get_events, self._h, cap, consume)[0]

    def event_count(self) -> int:
        return _get_events(lib().b2s_band_get_events, self._h, 0, False)[1]

    def record_from(self, channel: int, shift_hz: int, frame: int):
        """b2s_band_record_from: start `channel` of the attached bank at band frame `frame` (as in the signal events), from the bank's
        history, its chunks stamped with that frame's clock."""
        _check(lib().b2s_band_record_from(self._h, channel, shift_hz, frame))

    def set_auto_record(self, enable: bool = True, preroll_frames: int = 0):
        """b2s_band_set_auto_record: after each push the band starts and stops its attached bank's channels itself, as the reference's
        SdrDevice::updateRecordings does, each recording from its transmission's START frame minus `preroll_frames`."""
        _check(lib().b2s_band_set_auto_record(self._h, 1 if enable else 0, preroll_frames))

    def auto_record_actions(self, cap: int = 65536, consume: bool = True):
        """The oldest `cap` auto-record actions: [(kind, channel, shift_hz, key, frame, from_frame, time_ms, duration_ms)]."""
        acts = (AutoRecordAction * max(cap, 1))()
        count = C.c_int()
        _check(lib().b2s_band_get_auto_record_actions(self._h, C.cast(acts, C.c_void_p), cap, 1 if consume else 0, C.byref(count)))
        return [acts[i].astuple() for i in range(min(count.value, cap))]

    def set_occupancy(self, enable: bool = True):
        """b2s_band_set_occupancy: count the spectrum occupancy of the pushes after this call, per centre frequency."""
        _check(lib().b2s_band_set_occupancy(self._h, 1 if enable else 0))

    def occupancy_centers(self, cap: int = 1024):
        """The centres (Hz) with occupancy statistics, ascending."""
        out = np.zeros(max(cap, 1), dtype=np.int32)
        count = C.c_int()
        _check(lib().b2s_band_occupancy_centers(self._h, _ptr(out), cap, C.byref(count)))
        return [int(c) for c in out[: min(count.value, cap)]]

    def occupancy(self, center_hz: int, reset: bool = False) -> Occupancy:
        """b2s_band_get_occupancy: one centre's per-bin counts above the start and stop levels, its max-hold trace and frame counts."""
        n = self.cfg.fft_size
        o = Occupancy(np.zeros(n, np.uint32), np.zeros(n, np.uint32), np.zeros(n, np.float32), 0, 0, 0)
        frames, detect, truncated = C.c_int64(), C.c_int64(), C.c_int64()
        _check(lib().b2s_band_get_occupancy(self._h, center_hz, _ptr(o.above_start), _ptr(o.above_stop), _ptr(o.max_db), C.byref(frames), C.byref(detect),
                                            C.byref(truncated), 1 if reset else 0))
        return o._replace(frames=frames.value, detect_frames=detect.value, truncated=truncated.value)

    def save_state(self) -> bytes:
        """b2s_band_save_state: the band's whole state as an opaque snapshot (outstanding pushes are finished first)."""
        return _save_state(lib().b2s_band_save_state, self._h)

    def load_state(self, data: bytes):
        """b2s_band_load_state: replace the band's whole state with a snapshot of a band created with the same config."""
        _load_state(lib().b2s_band_load_state, self._h, data)


# ---- host helpers (reference semantics) ----
def get_fft(sample_rate_hz: int, max_step_hz: int) -> int:
    return lib().b2s_get_fft(sample_rate_hz, max_step_hz)


def get_tuned_frequency(f: int, step: int) -> int:
    return lib().b2s_get_tuned_frequency(f, step)


class HostTransmission(_Handle):
    """Transmission bookkeeping on host rows (b2s_host_transmission_*): the band's tracker without the GPU. push() returns,
    per frame, the list of (shift_hz, flush, key, power) exactly as Transmission::getSortedTransmissions orders it."""

    def __init__(self, cfg: BandConfig):
        super().__init__(lib().b2s_host_transmission_destroy)
        self.cfg = cfg
        _check(lib().b2s_host_transmission_create(C.byref(cfg), C.byref(self._h)))

    def push(self, box_rows: np.ndarray, q_rows: np.ndarray, t0_ms: int, frame_period_ms: float, use_watch: bool = True):
        box = np.ascontiguousarray(box_rows, dtype=np.float32)
        q = np.ascontiguousarray(q_rows, dtype=np.float32)
        frames = box.shape[0]
        assert box.shape == q.shape == (frames, self.cfg.fft_size)
        count = np.zeros(frames, dtype=np.int32)
        tx = (Transmission * (frames * MAX_TX))()
        _check(lib().b2s_host_transmission_push(self._h, _ptr(box), _ptr(q), frames, int(t0_ms), float(frame_period_ms), 1 if use_watch else 0, _ptr(count),
                                               C.cast(tx, C.c_void_p)))
        return [[(tx[k * MAX_TX + i].shift_hz, tx[k * MAX_TX + i].flush, tx[k * MAX_TX + i].key, tx[k * MAX_TX + i].power) for i in range(min(int(count[k]), MAX_TX))]
                for k in range(frames)]

    def last_run_ms(self) -> float:
        return lib().b2s_host_transmission_last_run_ms(self._h)

    def reset(self):
        _check(lib().b2s_host_transmission_reset(self._h))

    def get_events(self, cap: int = 65536, consume: bool = True):
        """The tracker's signal event log (b2s_host_transmission_get_events), as Band.get_events returns it."""
        return _get_events(lib().b2s_host_transmission_get_events, self._h, cap, consume)[0]


def _pack(fn, time_ms: int, frequency_hz: int, sample_rate_hz: int, data: np.ndarray, count: int, header: int) -> bytes:
    x = np.ascontiguousarray(data, dtype=np.int8)
    out = np.empty(header + x.size, dtype=np.uint8)
    written = C.c_size_t(0)
    _check(fn(time_ms, frequency_hz, sample_rate_hz, _ptr(x), count, _ptr(out), out.size, C.byref(written)))
    return out[: written.value].tobytes()


def pack_spectrogram_message(time_ms: int, center_hz: int, sample_rate_hz: int, row: np.ndarray) -> bytes:
    """DataController::pushSpectrogram payload (data_controller.cpp:44-57) for one int8 spectrogram row."""
    return _pack(lib().b2s_pack_spectrogram_message, time_ms, center_hz, sample_rate_hz, row, int(np.asarray(row).size), 24)


def pack_transmission_message(time_ms: int, frequency_hz: int, sample_rate_hz: int, iq_int8_pairs: np.ndarray) -> bytes:
    """DataController::pushTransmission payload (data_controller.cpp:27-42) for interleaved int8 I/Q samples."""
    x = np.asarray(iq_int8_pairs)
    return _pack(lib().b2s_pack_transmission_message, time_ms, frequency_hz, sample_rate_hz, x, int(x.size // 2), 20)


def get_max_index(data: np.ndarray, index: int, group_size: int) -> int:
    x = np.ascontiguousarray(data, dtype=np.float32)
    return lib().b2s_get_max_index(_ptr(x), x.shape[0], index, group_size)


def contains_with_margin(keys, index: int, margin: int):
    k = np.ascontiguousarray(keys, dtype=np.int32)
    found = C.c_int()
    return (found.value if lib().b2s_contains_with_margin(_ptr(k), k.shape[0], index, margin, C.byref(found)) else None)


def most_frequent_value(values) -> int:
    v = np.ascontiguousarray(values, dtype=np.int32)
    return lib().b2s_most_frequent_value(_ptr(v), v.shape[0])


def get_resamplers_factors(sample_rate_hz: int, bandwidth_hz: int, threshold: int = 125):
    """getResamplersFactors (radio_utils.cpp:129-152): [(interpolation, decimation), ...]."""
    a, b = (C.c_int32 * 16)(), (C.c_int32 * 16)()
    lib().b2s_get_resamplers_factors.argtypes = [C.c_int32, C.c_int32, C.c_int, C.c_void_p, C.c_void_p, C.c_int]
    k = lib().b2s_get_resamplers_factors(sample_rate_hz, bandwidth_hz, threshold, a, b, 16)
    if k < 0:
        _check(k)
    return [(a[i], b[i]) for i in range(k)]


class Recorder(_Handle):
    """The DSP chain of one reference Recorder on the GPU (recorder.cpp:22-40,58-73): rotate by -shift, resample fs -> bandwidth, int8."""

    def __init__(self, engine: Engine, sample_rate_hz: int, bandwidth_hz: int, iq_format: int = IQ_CS8, iq_scale: float = 1.0 / 127.0, on_device: bool = False,
                 max_samples_per_push: int = 0):
        L = lib()
        L.b2s_recorder_create.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int, C.c_float, C.c_int, C.c_size_t, C.POINTER(C.c_void_p)]
        L.b2s_recorder_destroy.argtypes = [C.c_void_p]
        L.b2s_recorder_start.argtypes = [C.c_void_p, C.c_int32]
        L.b2s_recorder_stop.argtypes = [C.c_void_p]
        L.b2s_recorder_push.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
        L.b2s_recorder_stages.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
        L.b2s_recorder_taps.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int]
        super().__init__(L.b2s_recorder_destroy)
        self._e = engine
        self.sample_rate_hz, self.bandwidth_hz, self.iq_format = sample_rate_hz, bandwidth_hz, iq_format
        _check(L.b2s_recorder_create(engine._h, sample_rate_hz, bandwidth_hz, iq_format, iq_scale, FLAG_IQ_ON_DEVICE if on_device else 0, max_samples_per_push, C.byref(self._h)))

    def stages(self):
        a, b, c = (C.c_int32 * 8)(), (C.c_int32 * 8)(), (C.c_int32 * 8)()
        k = lib().b2s_recorder_stages(self._h, a, b, c, 8)
        return [(a[i], b[i], c[i]) for i in range(k)]

    def taps(self, stage: int) -> np.ndarray:
        n = self.stages()[stage][2]
        t = np.empty(n, np.float32)
        assert lib().b2s_recorder_taps(self._h, stage, _ptr(t), n) == n
        return t

    def start(self, shift_hz: int):
        _check(lib().b2s_recorder_start(self._h, shift_hz))

    def stop(self):
        _check(lib().b2s_recorder_stop(self._h))

    def push(self, iq, n_samples: int = None) -> np.ndarray:
        """iq: numpy array of the stream's next samples (int8 pairs or float32 pairs), or a raw device pointer with n_samples."""
        if isinstance(iq, np.ndarray):
            iq = np.ascontiguousarray(iq)
            n_samples = iq.size // 2
            ptr = _ptr(iq)
        else:
            ptr = C.c_void_p(iq)
        cap = n_samples * self.bandwidth_hz // self.sample_rate_hz + 64
        out = np.empty(2 * cap, np.int8)
        n_out = C.c_size_t()
        _check(lib().b2s_recorder_push(self._h, ptr, n_samples, _ptr(out), cap, C.byref(n_out)))
        return out[: 2 * n_out.value]


class RecorderBank(_Handle):
    """A device's pool of Recorders on one IQ stream (SdrDevice::m_recorders, sdr_device.cpp:39-41): n_channels recorders indexed like
    the scan policy's actions. Each push runs every recording channel; each channel keeps Recorder's timestamped chunks for flush()."""

    def __init__(self, engine: Engine, sample_rate_hz: int, bandwidth_hz: int, n_channels: int, iq_format: int = IQ_CS8, iq_scale: float = 1.0 / 127.0,
                 on_device: bool = False, max_samples_per_push: int = 0):
        L = lib()
        L.b2s_recorder_bank_create.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int, C.c_float, C.c_int, C.c_int, C.c_size_t, C.POINTER(C.c_void_p)]
        L.b2s_recorder_bank_destroy.argtypes = [C.c_void_p]
        L.b2s_recorder_bank_start.argtypes = [C.c_void_p, C.c_int, C.c_int32]
        L.b2s_recorder_bank_stop.argtypes = [C.c_void_p, C.c_int]
        L.b2s_recorder_bank_push.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int64, C.c_void_p, C.c_size_t, C.c_void_p]
        L.b2s_recorder_bank_flush.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]
        super().__init__(L.b2s_recorder_bank_destroy)
        self._e = engine
        self.sample_rate_hz, self.bandwidth_hz, self.n_channels, self.iq_format = sample_rate_hz, bandwidth_hz, n_channels, iq_format
        self._band = None  # weak reference to the band this bank is attached to
        _check(L.b2s_recorder_bank_create(engine._h, sample_rate_hz, bandwidth_hz, iq_format, iq_scale, FLAG_IQ_ON_DEVICE if on_device else 0, n_channels,
                                          max_samples_per_push, C.byref(self._h)))

    def close(self):
        """b2s_recorder_bank_destroy: an attached bank is detached from its band first."""
        super().close()
        band = self._band() if self._band is not None else None
        if band is not None and band._bank is self:
            band._bank = None
        self._band = None

    def start(self, channel: int, shift_hz: int):
        _check(lib().b2s_recorder_bank_start(self._h, channel, shift_hz))

    def stop(self, channel: int):
        _check(lib().b2s_recorder_bank_stop(self._h, channel))

    def push(self, iq, t0_ms: int = 0, n_samples: int = None):
        """iq: numpy array of the stream's next samples (int8 pairs or float32 pairs), or a raw device pointer with n_samples.
        Returns one int8 pair array per channel (empty for idle channels)."""
        if isinstance(iq, np.ndarray):
            iq = np.ascontiguousarray(iq)
            n_samples = iq.size // 2
            ptr = _ptr(iq)
        else:
            ptr = C.c_void_p(iq)
        cap = n_samples * self.bandwidth_hz // self.sample_rate_hz + 64
        out = np.empty((self.n_channels, 2 * cap), np.int8)
        n_out = np.zeros(self.n_channels, np.uint64)
        _check(lib().b2s_recorder_bank_push(self._h, ptr, n_samples, int(t0_ms), _ptr(out), cap, _ptr(n_out)))
        return [out[c, : 2 * int(n_out[c])] for c in range(self.n_channels)]

    def flush(self, channel: int, cap: int = 256, consume: bool = True):
        """Recorder::flush: [(time_ms, int8 pairs of one chunk)] for the complete chunks buffered since the last flush, oldest first."""
        count, cs = C.c_int(), C.c_int()
        _check(lib().b2s_recorder_bank_flush(self._h, channel, None, None, 0, 0, C.byref(count), C.byref(cs)))
        k = min(count.value, cap)
        chunks = np.empty((k, 2 * cs.value), np.int8)
        times = np.empty(k, np.int64)
        _check(lib().b2s_recorder_bank_flush(self._h, channel, _ptr(chunks), _ptr(times), k, 1 if consume else 0, C.byref(count), C.byref(cs)))
        return [(int(times[i]), chunks[i]) for i in range(k)]

    def set_history(self, samples: int):
        """b2s_recorder_bank_set_history: keep the newest `samples` samples of the stream on the device (0: none); empties the history."""
        _check(lib().b2s_recorder_bank_set_history(self._h, samples))

    def history(self):
        """(oldest, end): the stream positions the history holds, counted since the last set_history or load_state."""
        oldest, end = C.c_int64(), C.c_int64()
        _check(lib().b2s_recorder_bank_history(self._h, C.byref(oldest), C.byref(end)))
        return oldest.value, end.value

    def start_from(self, channel: int, shift_hz: int, position: int, start_ms: int):
        """b2s_recorder_bank_start_from: start `channel` at stream position `position` of the history; [position, end) is recorded
        at once, its chunks stamped from start_ms."""
        _check(lib().b2s_recorder_bank_start_from(self._h, channel, shift_hz, position, int(start_ms)))

    def save_state(self) -> bytes:
        """b2s_recorder_bank_save_state: every channel's position, carries and unflushed chunks as an opaque snapshot."""
        return _save_state(lib().b2s_recorder_bank_save_state, self._h)

    def load_state(self, data: bytes):
        """b2s_recorder_bank_load_state: replace the bank's state with a snapshot of a bank of the same rate, bandwidth, format and size."""
        _load_state(lib().b2s_recorder_bank_load_state, self._h, data)


class RecorderAction(C.Structure):
    _fields_ = [("kind", C.c_int32), ("recorder", C.c_int32), ("shift_hz", C.c_int32), ("duration_ms", C.c_int64)]


REC_START, REC_STOP, REC_FLUSH, REC_NONE_FREE = 1, 2, 3, 4


def get_range_split_sample_rate(sample_rate_hz: int) -> int:
    lib().b2s_get_range_split_sample_rate.restype = C.c_int32
    return lib().b2s_get_range_split_sample_rate(sample_rate_hz)


class ScanPolicy(_Handle):
    """Scanner's hop rule (scanner.cpp:36-64) and SdrDevice::updateRecordings (sdr_device.cpp:82-144) as a host state machine."""

    def __init__(self, ranges, sample_rate_hz: int, n_recorders: int, scanning_time_ms: int = 500):
        L = lib()
        L.b2s_scan_policy_create.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int32, C.c_int, C.c_int64, C.POINTER(C.c_void_p)]
        L.b2s_scan_policy_destroy.argtypes = [C.c_void_p]
        L.b2s_scan_policy_ranges.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
        L.b2s_scan_policy_begin.argtypes = [C.c_void_p, C.c_int64, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
        L.b2s_scan_policy_notify.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
        lo = np.array([r[0] for r in ranges], np.int32)
        hi = np.array([r[1] for r in ranges], np.int32)
        super().__init__(L.b2s_scan_policy_destroy)
        _check(L.b2s_scan_policy_create(_ptr(lo), _ptr(hi), len(ranges), sample_rate_hz, n_recorders, scanning_time_ms, C.byref(self._h)))

    def ranges(self):
        lo, hi = np.zeros(4096, np.int32), np.zeros(4096, np.int32)
        k = lib().b2s_scan_policy_ranges(self._h, _ptr(lo), _ptr(hi), 4096)
        return [(int(lo[i]), int(hi[i])) for i in range(k)]

    def begin(self, now_ms: int):
        lo, hi = C.c_int32(), C.c_int32()
        _check(lib().b2s_scan_policy_begin(self._h, now_ms, C.byref(lo), C.byref(hi)))
        return lo.value, hi.value

    def notify(self, now_ms: int, transmissions):
        """transmissions: [(shift_hz, flush), ...] as the mailbox holds them. Returns (actions [(kind, recorder, shift, duration)], next range or None)."""
        n = len(transmissions)
        tx = (Transmission * max(n, 1))()
        for i, (shift, flush) in enumerate(transmissions):
            tx[i].shift_hz, tx[i].flush = shift, int(flush)
        acts = (RecorderAction * 256)()
        na, hop, lo, hi = C.c_int(), C.c_int(), C.c_int32(), C.c_int32()
        _check(lib().b2s_scan_policy_notify(self._h, now_ms, C.cast(tx, C.c_void_p), n, C.cast(acts, C.c_void_p), 256, C.byref(na), C.byref(hop), C.byref(lo), C.byref(hi)))
        out = [(acts[i].kind, acts[i].recorder, acts[i].shift_hz, acts[i].duration_ms) for i in range(min(na.value, 256))]
        return out, ((lo.value, hi.value) if hop.value else None)
