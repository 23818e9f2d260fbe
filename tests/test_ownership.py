"""Ownership of the library's CUDA resources: every object returns its device memory when it is destroyed, also when its creation
fails part-way, and only the owner types in csrc/ free buffers, streams and events."""
import gc
import os
import re

import numpy as np
import pytest

from conftest import PKG, load_b2s
from __graft_entry__ import load_synth

b2s = load_b2s()
synth = load_synth()

GiB = 1 << 30
TOLERANCE = GiB  # the GPU may be shared: other work moves its free memory too
N, FS = 16384, 20_000_000


def _free_bytes():
    import torch

    torch.cuda.synchronize()
    return torch.cuda.mem_get_info()[0]


def _assert_returns_memory(step, iterations, bytes_per_iteration):
    """Runs step(i) for i < iterations. If every step leaked bytes_per_iteration (a lower bound of what it allocates), the loss
    would be at least twice the tolerance."""
    assert iterations * bytes_per_iteration >= 2 * TOLERANCE
    for i in (-2, -1):  # first use of each path: module loading and the runtime's own allocations
        step(i)
    gc.collect()
    before = _free_bytes()
    for i in range(iterations):
        step(i)
    gc.collect()
    lost = before - _free_bytes()
    assert lost < TOLERANCE, f"{lost / GiB:.2f} GiB not returned; a leak would lose {iterations * bytes_per_iteration / GiB:.1f} GiB"


@pytest.mark.gpu
def test_bands_return_their_memory(engine):
    """Synchronous and asynchronous bands fed from host memory, at profiling level 2, on two centres. The synchronous band's
    per-frame push runs K3 (a signal fades below the levels before it times out) and fills the dense rows."""
    frames, learn, max_frames = 300, 40, 4096
    iq = synth.make_iq_int8(N, frames, synth.standard_scene(N, frames, learn), seed=synth.seed_for(0), quiet_frames=learn)
    period = synth.frame_period_ms(N, FS)
    t1 = int(frames * period) + 1
    window_launches = []

    def step(i):
        flags = b2s.FLAG_ASYNC if i % 2 else 0
        band = b2s.Band(engine, b2s.make_config(N, FS, learn_frames=learn, max_frames_per_push=max_frames, flags=flags))
        band.set_profiling(2)
        if flags:
            band.push_raw(iq.ctypes.data, frames, 0, period)
            band.set_center(120_000_000, 110_000_000, 130_000_000)
            band.push_raw(iq.ctypes.data, frames, t1, period)
            band.sync()
        else:
            band.push(iq, frames, 0, period, per_frame=True, dense=("noise_sub_db", "avg_db", "box_db"))
            window_launches.append(band.get_profile().window_launches)
            band.set_center(120_000_000, 110_000_000, 130_000_000)
            band.push(iq, frames, t1, period)
        band.close()

    # PSD rows alone: one push slot of [max_frames][N] floats per synchronous band, two per asynchronous one
    _assert_returns_memory(step, 24, max_frames * N * 4)
    assert window_launches and min(window_launches) > 0


@pytest.mark.gpu
def test_a_band_refused_after_allocating_returns_its_memory(engine):
    """grouping_x = 65 with N / spectrogram_out_size = 128 passes the config check, but no K2 CTA width fits: b2s_band_create
    refuses the band after it has created its streams and its spectral tables."""

    def refuse(n):
        cfg = b2s.make_config(n, FS, spectrogram_out_size=n // 128)
        cfg.grouping_x = 65
        with pytest.raises(b2s.B2SError) as e:
            b2s.Band(engine, cfg)
        assert str(e.value) == ("b2s error -1: grouping_x 65 (halo 32 bins per side) with a spectrogram decimation of 128 does not fit a "
                                "K2 CTA of 160 columns")

    refuse(N)
    # at N = 262144 the tables hold at least the window (1 MiB) and the split-mode twiddles (2 MiB)
    _assert_returns_memory(lambda i: refuse(262144), 1024, 3 << 20)


@pytest.mark.gpu
def test_engine_operators_return_their_memory():
    """A fresh engine per step running psd (with the linear rows), both average modes and the division self-test."""
    frames, rows = 1024, 2048
    rng = np.random.default_rng(7)
    iq = rng.integers(-128, 128, size=2 * N * frames, dtype=np.int8)
    data = rng.standard_normal((rows, N)).astype(np.float32)
    cfg = b2s.make_config(N, FS)

    def step(i):
        eng = b2s.Engine(0)
        eng.psd(cfg, iq, frames, want_linear=True)
        eng.average(data, 21, exact=bool(i % 2))
        assert eng.check_div_const(21) == 0
        eng.close()

    # psd: the IQ, the dB rows and the linear rows; average: its input and output rows
    _assert_returns_memory(step, 12, frames * N * (2 + 4 + 4) + 2 * rows * N * 4)


@pytest.mark.gpu
def test_averagers_return_their_memory(engine):
    size, group = 1 << 20, 21
    rows = np.random.default_rng(3).standard_normal((4, size)).astype(np.float32)

    def step(i):
        a = b2s.Averager(engine, size, group)
        a.push(rows)
        a.reset()
        a.average()
        a.close()

    _assert_returns_memory(step, 24, 2 * size * group * 4)  # the two rings


@pytest.mark.gpu
def test_recorders_and_banks_return_their_memory(engine):
    fs, bw, max_in = 40_000_000, 32_000, 1 << 24
    n = 1 << 18
    rng = np.random.default_rng(5)
    x = (rng.standard_normal(2 * n) * 0.05).astype(np.float32)

    def step(i):
        rec = b2s.Recorder(engine, fs, bw, iq_format=b2s.IQ_CF32, max_samples_per_push=max_in)
        rec.start(100_000)
        rec.push(x)
        rec.close()
        bank = b2s.RecorderBank(engine, fs, bw, 2, iq_format=b2s.IQ_CF32, max_samples_per_push=max_in)
        bank.start(0, 100_000)
        bank.start(1, -250_000)
        bank.push(x, 0)
        bank.flush(0)
        bank.flush(1)
        bank.close()

    _assert_returns_memory(step, 16, 2 * max_in * 8)  # the host-input staging of each


def test_only_the_owner_types_free_cuda_resources():
    """cudaFree, cudaFreeHost, cudaStreamDestroy and cudaEventDestroy appear in csrc/ only inside the owner types (CudaBuf,
    CudaHandle), and no object keeps a hand-written release() list."""
    frees = re.compile(r"\bcuda(Free|FreeHost|StreamDestroy|EventDestroy)\b")
    csrc = os.path.join(PKG, "csrc")
    owners_seen = 0
    for f in sorted(os.listdir(csrc)):
        text = open(os.path.join(csrc, f), errors="replace").read()
        for owner in ("struct CudaBuf {", "struct CudaHandle {"):
            start = text.find(owner)
            if start < 0:
                continue
            owners_seen += 1
            depth, end = 0, start
            for end in range(text.index("{", start), len(text)):
                depth += {"{": 1, "}": -1}.get(text[end], 0)
                if depth == 0:
                    break
            text = text[:start] + text[end + 1 :]
        assert not frees.search(text), f"{f}: {frees.search(text).group(0)} outside the owner types"
        assert not re.search(r"\bvoid\s+release\s*\(", text), f"{f}: a release() method"
    assert owners_seen == 2
