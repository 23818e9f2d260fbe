/* b2s — H100 spectrum-scan engine: the C-ABI drop-in boundary.
 *
 * This library replaces, for ONE band (= one SDR device chain), the reference's GNU Radio block chain
 *     decimator -> fft_v(hamming, shift) -> PSD -> NoiseLearner -> Transmission   (+ PSD -> Spectrogram)
 * that is assembled in exactly one place, sources/radio/sdr_device.cpp:161-171 (reference paths are relative to
 * /root/reference). Everything upstream (SoapySDR source, stream_to_vector, Blocker) and downstream
 * (Scanner::worker, SdrDevice::updateRecordings, Recorder, DataController/MQTT) stays the reference's own code;
 * INTEGRATION.md shows the ~40-line gr::sync_block adaptor a maintainer would add.
 *
 * Conventions
 *   - every entry point returns 0 on success or a negative B2S_E_* code; nothing throws or aborts across the ABI.
 *     b2s_last_error() returns a thread-local message for the last failure on the calling thread.
 *     (reference: C++ exceptions at construction, main.cpp:60; work() has no error channel.)
 *   - plain pointers and sizes only. Device pointers are accepted where flagged.
 *   - a band handle is externally synchronised, except b2s_band_reset / b2s_band_set_center, which may be called
 *     from another thread while a push is running (same guarantee as the reference's per-block mutexes,
 *     transmission.cpp:34,43; noise_learner.cpp:40,70). Different bands are independent (own stream + state).
 *   - the hot path runs ONLY on the GPU (sm_90a). There is no CPU fallback: if no CUDA device is usable,
 *     b2s_engine_create fails with B2S_E_CUDA.
 *   - time is injected: frame k of a push is stamped now_k = t0_ms + floor(k * frame_period_ms + 0.5)
 *     (replaces getTime() in noise_learner.cpp:18, transmission.cpp:63, spectrogram.cpp:63).
 */
#ifndef B2S_H
#define B2S_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2S_VERSION 100

#define B2S_OK 0
#define B2S_E_INVALID (-1)   /* bad argument / unsupported configuration */
#define B2S_E_CUDA (-2)      /* CUDA runtime error (sticky errors: destroy and re-create the engine) */
#define B2S_E_NOMEM (-3)
#define B2S_E_OVERFLOW (-4)  /* a frame had more detection entries than detect_capacity: the push completed on truncated lists (state
                                stays consistent), the capacity grows before the next push */
#define B2S_E_STATE (-5)

#define B2S_MAX_IGNORED 16
#define B2S_MAX_TX 64        /* transmissions held INSIDE b2s_result; the signal map itself is not limited to this:
                                n_transmissions_total reports the real count and b2s_band_get_transmissions returns the whole list.
                                Like the reference's std::map, the device-resident map has no cap on live signals */

#define B2S_IQ_CS8 0         /* interleaved int8 I,Q (help_structures.h:17 SimpleComplex) */
#define B2S_IQ_CF32 1        /* interleaved float I,Q (what SdrSource delivers, sdr_source.cpp:52) */

#define B2S_WINDOW_HAMMING 0 /* gr::fft::window::hamming(N), sdr_device.cpp:164 */
#define B2S_WINDOW_USER 1

/* b2s_band_config.flags */
#define B2S_FLAG_IQ_ON_DEVICE 0x100 /* `iq` passed to b2s_band_push is a device pointer */
#define B2S_FLAG_ASYNC 0x200        /* b2s_band_push returns once the GPU work is enqueued; the signal bookkeeping of push k
                                       runs on a worker thread while push k+1 is in the kernels (the reference decouples the
                                       same two halves through its 1-slot mailbox, notification.h:14-26). Results are
                                       collected with b2s_band_sync; b2s_band_push must be given out = NULL. */
/* Sub-frames: detect from every sample of a frame's stride instead of its first fft_size samples only (opt-in; off by default).
 * Frame k has r = floor(frame_stride_samples / fft_size) sub-frames; sub-frame j is the fft_size samples starting at
 * k * frame_stride_samples + j * fft_size (j = 0 ... r-1); samples past r * fft_size in a stride stay unused. Each sub-frame is
 * windowed, transformed, shifted and squared exactly as a frame is without the flag, p_j[b] = |X_j[b]|^2 / fs, and the frame's
 * linear power row is
 *   MEAN: acc = p_0; acc = acc + p_j for j = 1 ... r-1 in that order (fp32, round to nearest); p = acc / (float)r (fp32 division)
 *   MAX:  p = fmaxf over j = 0 ... r-1
 * The dB row, the first maximum (peak_index / peak_value) and b2s_psd's power_lin are then computed from p as without the flag.
 *   - Frames, their clock, event frames, b2s_band_record_from positions, the spectrogram schedule and an attached recorder bank's
 *     input do not change. Noise learning, the Averager, the detector and the tracker see the new rows.
 *   - With r = 1 (frame_stride_samples < 2 * fft_size) either flag changes nothing, bit for bit.
 *   - Both flags together are refused (B2S_E_INVALID) by b2s_band_create and b2s_psd.
 *   - Input: a push (or b2s_psd) of n_frames frames reads (n_frames - 1) * frame_stride_samples + r * fft_size samples, host or
 *     device; with an attached recorder bank the rule stays n_frames * frame_stride_samples.
 *   - A band snapshot records the flags; a load into a band whose two sub-frame bits differ is refused (the learned noise depends
 *     on them).
 * MEAN suits weak continuous signals: the mean of r periodograms has a smaller spread, so the learned noise maximum sits lower.
 * MAX suits bursts shorter than a stride: the mean would dilute a burst that fills one sub-frame by 10 log10(r) dB. */
#define B2S_FLAG_SUBFRAME_MEAN 0x400
#define B2S_FLAG_SUBFRAME_MAX 0x800
/* Overlapping sub-frames (opt-in, with exactly one of B2S_FLAG_SUBFRAME_MEAN / _MAX): back-to-back Hamming sub-frames lose a
 * burst that sits on a sub-frame edge, where both windows taper to 0.08 (about 28 dB for a tone burst of fft_size / 16 samples).
 * With h = fft_size / 2 the sub-frames overlap by half, so every sample lies in the central half of exactly one of them.
 *   - frame_stride_samples must be at least fft_size and a multiple of h (b2s_default_config's strides are); any other use, or the
 *     flag without exactly one of MEAN / MAX, is refused (B2S_E_INVALID) by b2s_band_create and b2s_psd.
 *   - Frame k has m = frame_stride_samples / h sub-frames; sub-frame j (j = 0 ... m-1) is the fft_size samples starting at
 *     k * frame_stride_samples - h + j * h. Sub-frame 0 straddles the end of the previous frame, sub-frame m-1 ends with frame k's
 *     stride, and frame k owns the samples [k * stride - fft_size / 4, (k + 1) * stride - fft_size / 4) (the central halves).
 *     Each is windowed, transformed, shifted and squared as above and folded in ascending j by MEAN (then divided by the count
 *     folded) or MAX.
 *   - The lead-in: frame 0 of a push takes its sub-frame 0's first h samples from the last h samples of the band's previous push,
 *     which the band keeps on the device. There is none on the first push after b2s_band_create, after a b2s_band_set_center that
 *     changes the centre, and after a b2s_band_load_state whose snapshot holds none; that frame then folds sub-frames 1 ... m-1
 *     (MEAN divides by m - 1). b2s_band_reset keeps it: the IQ stream does not break.
 *   - Input: a push reads n_frames * frame_stride_samples samples, the whole stream (host or device, with or without a bank).
 *     b2s_psd reads h + n_frames * frame_stride_samples samples: `iq` points at frame 0's lead-in, and every frame folds all m.
 *   - However a stream is cut into pushes, and however the band cuts a push into pieces, the results are bit for bit the same
 *     (given the same frame clocks).
 *   - A band snapshot holds the lead-in (one extra section, only for bands with the flag); a load into a band whose overlap bit
 *     differs is refused. */
#define B2S_FLAG_SUBFRAME_OVERLAP 0x1000

/* Construction-time parameters. The reference takes them from Config / Device / the setupChains lambdas
 * (sdr_device.cpp:148-167, transmission.h:17-25, config.h:24-38). */
typedef struct b2s_band_config {
  int32_t fft_size;             /* N = getFft(fs, SIGNAL_DETECTION_MAX_STEP); power of two, 256..1048576 (sizes above 16384 run as S = N/16384
                                   16384-point residue classes of the bin index, S up to 64, see csrc/spectral3.cuh) */
  int32_t sample_rate_hz;       /* Device::m_sampleRate (Frequency = int32_t) */
  int32_t frame_stride_samples; /* fftSize * decimatorFactor complex samples between frame starts (sdr_device.cpp:161-163) */
  int32_t iq_format;            /* B2S_IQ_* */
  float iq_scale;               /* CS8: x = (float)i8 * iq_scale; default 1/127 (inverse of recorder.cpp:36) */
  int32_t window_kind;          /* B2S_WINDOW_* */
  const float* window_taps;     /* host pointer, N floats, only read during b2s_band_create when B2S_WINDOW_USER */
  int32_t grouping_x;           /* GROUPING_X (21): frequency boxcar width, transmission.cpp:61 */
  int32_t grouping_y;           /* GROUPING_Y (21): Averager depth, transmission.cpp:24 */
  int32_t group_size_bins;      /* indexStep = ceil(recordingBandwidth / (fs/N)), sdr_device.cpp:151 */
  float start_level;            /* Device::m_startLevel (8 dB) */
  float stop_level;             /* Device::m_stopLevel (5 dB) */
  int32_t learn_frames;         /* noise-learning length in frames (>= 1); see b2s_learn_frames_from_ms */
  int32_t center_hz;            /* SdrDevice::getFrequency() */
  int32_t range_lo_hz;          /* m_frequencyRange.first */
  int32_t range_hi_hz;          /* m_frequencyRange.second */
  int32_t n_ignored;            /* Config::ignoredRanges() */
  int32_t ignored_lo_hz[B2S_MAX_IGNORED];
  int32_t ignored_hi_hz[B2S_MAX_IGNORED];
  int32_t tuning_step_hz;       /* Config::recordingTuningStep() */
  int64_t min_time_ms;          /* Config::recordingMinTime() */
  int64_t timeout_ms;           /* Config::recordingTimeout() */
  int64_t max_time_ms;          /* TRANSMISSION_MAX_TIME (600000) */
  int32_t spectrogram_out_size; /* min(SPECTROGRAM_MAX_FFT, getFft(fs, 1000)), spectrogram.cpp:14; 0 disables */
  int64_t spectrogram_interval_ms; /* SPECTROGRAM_SEND_INTERVAL (1000) */
  int32_t flags;                /* B2S_FLAG_* */
  /* ---- engine-only sizing (ignored by the oracle) ---- */
  int32_t max_frames_per_push;  /* capacity of the per-push device buffers; 0 -> 4096 for N <= 262144, 2^30 / N above (2048 at 524288,
                                   1024 at 1048576). Above N = 262144, max_frames_per_push * N must not exceed 2^30 (4 GiB of PSD rows). */
  int32_t detect_capacity;      /* detection entries kept per FRAME (bins >= min(start,stop)); 0 -> clamp(N/8, 256, 4096); grows on overflow */
  /* ---- noise learning on the frame clock (read by the engine AND the oracle) ---- */
  int64_t noise_learning_ms;    /* > 0: NoiseLearner's own rule (noise_learner.cpp:11,23): a centre frequency is learned from its first frame
                                   (stamped s) up to and including the first frame stamped >= s + noise_learning_ms, however many frames
                                   that is - under a hop schedule the time spent on other centres counts, as in the reference;
                                   learn_frames is ignored. 0: learn_frames frames per centre (equal for a band that never hops).
                                   b2s_default_config sets NOISE_LEARNING_TIME = 2000 (config.h:24). */
} b2s_band_config;

/* Fill cfg with the reference's defaults for a device with this sample rate, exactly as setupChains sizes the chain
 * (sdr_device.cpp:148-152: N, indexStep, decimatorFactor) and config.h:24-38 / config.example.json:9-13. */
void b2s_default_config(b2s_band_config* cfg, int32_t sample_rate_hz, int32_t center_hz, int32_t recording_bandwidth_hz);

/* One FrequencyFlush (help_structures.h:15) as Transmission::getSortedTransmissions emits it (transmission.cpp:166-176). */
typedef struct b2s_transmission {
  int32_t shift_hz; /* getTunedFrequency(indexToShift(key), tuningStep) */
  int32_t flush;    /* Signal::needFlush(now) */
  int32_t key;      /* map key (bin index) — extra, for diagnostics */
  float power;      /* Signal::getPower() — extra */
} b2s_transmission;

/* Result buffers for one push; every pointer is optional (NULL = not wanted) and caller-owned HOST memory. */
typedef struct b2s_result {
  /* the mailbox content after the last frame (what Notification::notify last received, transmission.cpp:67) */
  int32_t n_transmissions;
  b2s_transmission transmissions[B2S_MAX_TX];
  /* per-frame lists for parity tests / callers that want every notification */
  int32_t* frame_tx_count;          /* [n_frames] */
  b2s_transmission* frame_tx;       /* [n_frames][B2S_MAX_TX] */
  int32_t* peak_index;              /* [n_frames] argmax of the raw PSD row (noise_learner.cpp:53-59) */
  float* peak_value;                /* [n_frames] raw PSD at peak_index */
  /* dense rows, [n_frames][N] each — debug / parity only (they cost PCIe time) */
  float* psd_db;                    /* PSD::work output (psd.cpp:18) */
  float* noise_sub_db;              /* NoiseLearner::work output */
  float* avg_db;                    /* Averager::average() after each push */
  float* box_db;                    /* average(avg, GROUPING_X) */
  /* statistics */
  int32_t n_detect_entries;         /* bins >= min(start,stop) level found in this push */
  int32_t n_spectrogram_rows;       /* rows completed during this push (fetch with b2s_band_get_spectrogram) */
  int32_t n_transmissions_total;    /* live transmissions after the last frame; when > B2S_MAX_TX, transmissions[] holds the
                                       B2S_MAX_TX strongest and b2s_band_get_transmissions the complete list */
} b2s_result;

typedef struct b2s_engine b2s_engine;
typedef struct b2s_band b2s_band;

const char* b2s_last_error(void);
int b2s_version(void);

/* ---- engine / band lifetime (reference: SdrDevice ctor/dtor, sdr_device.cpp:17-52) ---- */
int b2s_engine_create(int cuda_device, b2s_engine** out);
int b2s_engine_destroy(b2s_engine* e);
int b2s_engine_device_name(b2s_engine* e, char* buf, size_t cap);
int b2s_band_create(b2s_engine* e, const b2s_band_config* cfg, b2s_band** out);
int b2s_band_destroy(b2s_band* b);
/* run this band's kernels on a caller-owned CUDA stream (cudaStream_t); NULL restores the band's own stream */
int b2s_band_set_stream(b2s_band* b, void* cuda_stream);

/* ---- data path: replaces the work() calls of Decimator..Transmission (+Spectrogram) for n_frames input items ----
 * iq: n_frames frames, frame k starting at sample k*frame_stride_samples; host memory (pageable or pinned) or,
 * with B2S_FLAG_IQ_ON_DEVICE, device memory. Read-only; may be reused as soon as the call returns. */
int b2s_band_push(b2s_band* b, const void* iq, size_t n_frames, int64_t t0_ms, double frame_period_ms, b2s_result* out);

/* Async mode: wait for every outstanding push; `out` (optional) receives the mailbox after the last frame pushed so far
 * and the statistics accumulated since the previous sync. A no-op returning the last mailbox in synchronous mode. */
int b2s_band_sync(b2s_band* b, b2s_result* out);

/* ---- profiling (bench.py): per-kernel device time measured with CUDA events on the band's stream ---- */
typedef struct b2s_profile {
  double spectral_ms;        /* K1 k_spectrum: unpack+window+FFT+PSD */
  double detect_ms;          /* K2 k_detect: noise/averager/boxcar/threshold/spectrogram */
  double window_ms;          /* K3 k_window_query (only when the tracker needs sub-threshold window maxima) */
  double tracker_host_ms;    /* host time spent on the results of a push (wall clock): reading K4's result, or tracker.h when every frame's list is wanted */
  int64_t spectral_launches, detect_launches, window_launches;
  int64_t pushes, frames;
  int64_t h2d_bytes, d2h_bytes; /* bytes moved by b2s_band_push itself */
  /* load balance of K2 (one CTA per 128 bins): per-CTA run time in ms, median and slowest, summed over launches */
  double detect_cta_median_ms, detect_cta_max_ms;
  double track_ms;           /* K4 k_track + k_track_wide: the signal map on the device (runs beside the next push's K1) */
  int64_t track_launches;    /* K4 launches that ran a push: one per device-tracked push, two when k_track left it to k_track_wide */
  int64_t track_evals, track_events, track_best_index;  /* K4 work counters: block evaluations, event frames replayed, getBestIndex calls */
} b2s_profile;
int b2s_band_set_profiling(b2s_band* b, int enable); /* 0 off, 1 kernel times and byte counts, 2 also K2 per-CTA run times */
int b2s_band_get_profile(b2s_band* b, b2s_profile* out, int reset);

/* ---- side channels ---- */
int b2s_band_reset(b2s_band* b); /* Transmission::resetBuffers (transmission.cpp:42-55): drop signals, Averager::reset; noise kept */
int b2s_band_set_center(b2s_band* b, int32_t center_hz, int32_t range_lo_hz, int32_t range_hi_hz); /* retune, sdr_device.cpp:66-77 */

/* ---- state introspection (reference: Averager::average()/data(), averager.h:15-16) ---- */
int b2s_band_get_averager(b2s_band* b, float* sum /*[N]*/, float* avg /*[N]*/, float* ring /*[Y][N] oldest->newest*/, int32_t* frames);
int b2s_band_get_noise(b2s_band* b, float* threshold /*[N]*/, int32_t* samples, int32_t* ready);
/* completed spectrogram rows (Spectrogram::send, spectrogram.cpp:62-75), oldest first: up to `cap` rows are copied, *count is
 * the number available; with consume != 0 the rows copied out (and only those) are dropped from the band's list */
int b2s_band_get_spectrogram(b2s_band* b, int64_t* times_ms, int32_t* centers_hz, int8_t* rows /*[cap][out_size]*/, int cap, int consume, int* count);
/* the complete mailbox after the last finished push (Transmission::getSortedTransmissions, transmission.cpp:166-176), strongest
 * first; up to `cap` entries are copied, *count is the number of live transmissions */
int b2s_band_get_transmissions(b2s_band* b, b2s_transmission* out, int cap, int* count);
/* live signals (the std::map<Index, Signal> of transmission.h:49) */
int b2s_band_get_signals(b2s_band* b, int32_t* keys, int64_t* first_ms, int64_t* last_ms, float* power, int cap, int* count);

/* ---- signal event log: every change of the signal map, in the order Transmission::process makes them ----
 * The mailbox shows the map after the last frame of a push only. The log (off by default) also keeps every insertion and erasure
 * that happened in the frames of a push, so a transmission that starts and times out inside one push is still reported, and a
 * start or stop comes with its frame. It replaces the Logger::info lines of transmission.cpp:75-80,101-107.
 * Order: by frame; within a frame the STARTs in the order addSignals inserted them (strongest uncovered candidate first), then
 * the STOPs in ascending key (the map order clearSignals walks). b2s_band_reset and b2s_band_set_center log nothing
 * (resetBuffers is silent in the reference), and the events of frames pushed before them stay in the log. */
#define B2S_EV_START 1  /* addSignals inserted the key (transmission.cpp:108) */
#define B2S_EV_STOP 2   /* clearSignals erased it: isTimeout or isMaximalTime (transmission.cpp:73-81) */
#define B2S_EV_LOST 3   /* `key` events of one device pass did not fit the device log (fft_size records per pass) and are missing at
                           this point; frame and time_ms repeat the last event kept */
typedef struct b2s_signal_event {
  int32_t kind;      /* B2S_EV_* */
  int32_t key;       /* map key (bin); for B2S_EV_LOST the number of events lost */
  int32_t shift_hz;  /* getTunedFrequency(indexToShift(key), tuningStep): the value b2s_transmission.shift_hz carries */
  int32_t reserved;
  int64_t frame;     /* frames pushed to this band before the event's frame, counted from b2s_band_create (reset and retune do not
                        restart it) */
  int64_t time_ms;   /* the frame's injected clock */
  int64_t first_ms;  /* Signal::m_firstDataTime (= time_ms for START) */
  int64_t last_ms;   /* Signal::m_lastDataTime when erased (= time_ms for START) */
} b2s_signal_event;
/* enable != 0 turns the log on for the pushes after this call; turning it off drops nothing already logged */
int b2s_band_set_event_log(b2s_band* b, int enable);
/* events of the finished pushes, oldest first: up to `cap` are copied, *count is the number available; with consume != 0 the
 * events copied out (and only those) are dropped from the log */
int b2s_band_get_events(b2s_band* b, b2s_signal_event* out, int cap, int consume, int* count);

/* ---- spectrum occupancy: how often each bin is busy, and how strong it gets, per centre frequency ----
 * Accumulated on the device over the pushes since occupancy was enabled or the centre's statistics were last reset, so a band that runs
 * all day can tell which frequencies are busy and for how much of the time (to choose start_level, stop_level, the scanned ranges and
 * ignored ranges) without dense debug rows.
 *   - Per centre: a centre's statistics (3 x N x 4 B of device memory) are allocated the first time a push runs at that centre with
 *     occupancy on. They count only the frames pushed at that centre.
 *   - frames: every frame pushed at the centre while occupancy was on. detect_frames: those past noise learning, the frames the
 *     detector produces entries for.
 *   - above_start[b] / above_stop[b]: the detect frames whose boxcar value (b2s_result.box_db) of bin b is >= start_level / >= stop_level,
 *     decided on the detection entries with the predicate the signal bookkeeping uses. Every bin counts: the scanned range and the
 *     ignored ranges do not apply. above_start[b] / detect_frames is bin b's duty cycle at the start level.
 *   - max_db[b]: the largest raw PSD value (b2s_result.psd_db, after sub-frame folding) of bin b over all `frames`, learning frames
 *     included; -inf before the first frame.
 *   - truncated: the pieces of pushes (b2s_band_push works in pieces of at most max_frames_per_push frames) whose detection lists
 *     overflowed detect_capacity (the push returned B2S_E_OVERFLOW) among those counted. While it is nonzero, above_start and above_stop
 *     are lower bounds.
 *   - The counters are 32-bit and wrap after 2^32 frames (2.7 years at 50 frames/s).
 * The band's own results (mailbox, map, spectrogram rows, events, Averager, noise, an attached bank's output) are bit for bit those of
 * the same band with occupancy off. b2s_band_reset and b2s_band_set_center clear nothing. Occupancy is not part of a snapshot. */
/* enable != 0: the pushes after this call are counted (off by default); turning it off keeps what was accumulated, readable as before */
int b2s_band_set_occupancy(b2s_band* b, int enable);
/* the centres with statistics, ascending: up to `cap` are copied, *count is the number there are */
int b2s_band_occupancy_centers(b2s_band* b, int32_t* centers_hz, int cap, int* count);
/* The statistics of one centre. Outstanding pushes are finished first (as b2s_band_save_state does). With reset != 0 the centre's counts
 * and max-hold are cleared after they are copied out. Every pointer is required; B2S_E_INVALID for a centre without statistics. */
int b2s_band_get_occupancy(b2s_band* b, int32_t center_hz, uint32_t* above_start /*[N]*/, uint32_t* above_stop /*[N]*/, float* max_db /*[N]*/,
                           int64_t* frames, int64_t* detect_frames, int64_t* truncated, int reset);

/* ---- snapshots: save a band's whole state and restore it into another band, in this process or another, on any engine ----
 * A band restored from a snapshot continues exactly like the band that saved it: the noise thresholds of every centre visited, the
 * Averager, the live signals, the spectrogram accumulators, the frame counter of the event log, the current centre and range, the
 * mailbox, the spectrogram rows and events not yet collected, the statistics since the last sync and the detection capacity.
 * Profiling counters and the attachment to a recorder bank are not part of it (attach the restored bank again).
 * The snapshot is an opaque, versioned, checksummed byte string in HOST memory; its format is internal (DESIGN.md §3) and a load of
 * another format version is refused.
 * b2s_band_save_state first finishes every outstanding push (as b2s_band_sync does, but it collects and resets nothing). Calling it
 * with cap too small (including buf == NULL, cap == 0) returns B2S_E_INVALID with *written = the required size, as the b2s_pack_*
 * functions do. */
int b2s_band_save_state(b2s_band* b, void* buf, size_t cap, size_t* written);
/* Replace the band's whole state with a saved one. The band may be new or used, on any engine or device, synchronous or asynchronous,
 * host or device IQ. Outstanding pushes are finished first. The band must have been created with the snapshot's config, except for
 * center_hz, range_lo_hz and range_hi_hz (taken from the snapshot), flags, max_frames_per_push and detect_capacity (the detection
 * capacity becomes the larger of the band's and the snapshot's); floats and B2S_WINDOW_USER taps are compared bit for bit.
 * A refused load (B2S_E_INVALID: damaged, truncated or incompatible snapshot; B2S_E_NOMEM) changes nothing else. */
int b2s_band_load_state(b2s_band* b, const void* buf, size_t len);

/* ---- stand-alone operators (operator-level parity with the reference's unit tests) ---- */
/* device-backed Averager with the reference's surface (averager.h:8-28) */
typedef struct b2s_averager b2s_averager;
int b2s_averager_create(b2s_engine* e, int size, int group_size, b2s_averager** out);
int b2s_averager_destroy(b2s_averager* a);
int b2s_averager_push(b2s_averager* a, const float* data);                /* Averager::push, one row */
int b2s_averager_push_many(b2s_averager* a, const float* rows, int count); /* count rows in one launch */
int b2s_averager_reset(b2s_averager* a);
int b2s_averager_average(b2s_averager* a, float* out);                    /* Averager::average() */
int b2s_averager_data(b2s_averager* a, float* out);                       /* Averager::data(), [group][size] oldest->newest */
int b2s_averager_sum(b2s_averager* a, float* out, int32_t* frames);       /* m_sum, m_frames */
/* average(in,out,size,groupSize) (utils.cpp:31-53) for `rows` rows on the device.
 * exact == 0: the engine's fused form (independent window sums, <= 1e-5 dB from the reference's running sum);
 * exact != 0: the reference's serial running sum, bit-exact (one thread per row). */
int b2s_average(b2s_engine* e, const float* in, float* out, int size, int group_size, int rows, int exact);
/* IQ -> raw PSD rows (unpack, window, FFT, shift, dB) only; power_lin optional (|X|^2/fs) */
int b2s_psd(b2s_engine* e, const b2s_band_config* cfg, const void* iq, size_t n_frames, float* psd_db, float* power_lin);

/* ---- recorder chain (SURVEY.md 8(f)#1): what one reference Recorder computes (sources/radio/recorder.cpp:22-40,58-73) ----
 * rotator_cc(-shift) -> rational_resampler(f1, f2) per pair of getResamplersFactors(fs, bandwidth, RESAMPLER_THRESHOLD = 125)
 * -> complex_to_interleaved_char(x 127): a continuous IQ stream at fs in, int8 IQ at `bandwidth` samples/s out. The resamplers use
 * GNU Radio's default taps (Kaiser low-pass, beta 7, fractional bandwidth 0.4); history is zero at b2s_recorder_start.
 * Chunking into messages (recorder.cpp:35) and the wire format stay host work: b2s_pack_transmission_message. */
typedef struct b2s_recorder b2s_recorder;
int b2s_get_resamplers_factors(int32_t sample_rate_hz, int32_t bandwidth_hz, int threshold, int32_t* interp, int32_t* decim, int cap); /* radio_utils.cpp:129-152; returns the count */
int b2s_recorder_create(b2s_engine* e, int32_t sample_rate_hz, int32_t bandwidth_hz, int iq_format, float iq_scale, int flags /* B2S_FLAG_IQ_ON_DEVICE */,
                        size_t max_samples_per_push /* 0 -> 4 Mi */, b2s_recorder** out);
int b2s_recorder_destroy(b2s_recorder* r);
int b2s_recorder_start(b2s_recorder* r, int32_t shift_hz); /* Recorder::startRecording: rotator phase_inc = 2 pi (-shift) / fs, empty buffers */
int b2s_recorder_stop(b2s_recorder* r);                    /* Recorder::stopRecording */
/* n_samples consecutive IQ samples of the stream (host memory, or device memory with B2S_FLAG_IQ_ON_DEVICE) -> *n_out int8 I/Q pairs in out_iq (host) */
int b2s_recorder_push(b2s_recorder* r, const void* iq, size_t n_samples, int8_t* out_iq, size_t cap_samples, size_t* n_out);
int b2s_recorder_stages(b2s_recorder* r, int32_t* interp, int32_t* decim, int32_t* n_taps, int cap); /* returns the number of stages */
int b2s_recorder_taps(b2s_recorder* r, int stage, float* taps, int cap);                            /* returns the number of taps */

/* ---- scan policy (SURVEY.md 8(f)#3): Scanner's hop rule and SdrDevice's recorder assignment as a host state machine ----
 * Scanner::worker (scanner.cpp:36-64): stay on a range while now <= start + RANGE_SCANNING_TIME or the last notification was not
 * empty. SdrDevice::updateRecordings (sdr_device.cpp:82-144): stop recorders whose shift left the list, flush / start the others.
 * Ranges are split like Scanner's constructor does (splitRanges(ranges, getRangeSplitSampleRate(fs)), radio_utils.cpp:162-199).
 * The caller owns the loop: each mailbox list obtained from b2s_band_push / b2s_band_sync is one notification. */
#define B2S_REC_START 1      /* Recorder::startRecording(frequency, shift) on recorder `recorder` */
#define B2S_REC_STOP 2       /* Recorder::stopRecording; duration_ms = Recorder::getDuration() */
#define B2S_REC_FLUSH 3      /* Recorder::flush */
#define B2S_REC_NONE_FREE 4  /* no recorder available for this shift (logged once, sdr_device.cpp:129-132) */
typedef struct b2s_recorder_action {
  int32_t kind;      /* B2S_REC_* */
  int32_t recorder;  /* index into the pool, -1 for B2S_REC_NONE_FREE */
  int32_t shift_hz;
  int64_t duration_ms;
} b2s_recorder_action;
typedef struct b2s_scan_policy b2s_scan_policy;
int b2s_scan_policy_create(const int32_t* range_lo_hz, const int32_t* range_hi_hz, int n_ranges, int32_t sample_rate_hz, int n_recorders, int64_t scanning_time_ms /* 0 -> 500 */,
                           b2s_scan_policy** out);
int b2s_scan_policy_destroy(b2s_scan_policy* p);
int b2s_scan_policy_ranges(b2s_scan_policy* p, int32_t* lo_hz, int32_t* hi_hz, int cap);              /* the split ranges; returns their number */
int b2s_scan_policy_begin(b2s_scan_policy* p, int64_t now_ms, int32_t* lo_hz, int32_t* hi_hz);          /* first setFrequencyRange */
/* one notification: recorder actions in the reference's order; *hop != 0 when the scanner retunes, then next_lo/next_hi hold the range */
int b2s_scan_policy_notify(b2s_scan_policy* p, int64_t now_ms, const b2s_transmission* list, int n, b2s_recorder_action* actions, int cap, int* n_actions, int* hop,
                           int32_t* next_lo_hz, int32_t* next_hi_hz);
int32_t b2s_get_range_split_sample_rate(int32_t sample_rate_hz);                                         /* radio_utils.cpp:162-172 */

/* Self-test: the 3-instruction exact division by a small constant that the Averager (m_sum / GROUPING_Y, averager.cpp:52-60) and
 * boxcar fast paths use, compared with IEEE division for EVERY float with |x| in [2^-60, 2^61) and +-0. *mismatches must be 0. */
int b2s_selftest_div_const(b2s_engine* e, int divisor, uint64_t* mismatches);

/* ---- host helpers with the reference's semantics (used by the tracker; exported for the adaptor and for tests) ---- */
int b2s_get_fft(int32_t sample_rate_hz, int32_t max_step_hz);                                  /* radio_utils.cpp:98-104 */
int32_t b2s_get_tuned_frequency(int32_t frequency_hz, int32_t step_hz);                        /* radio_utils.cpp:86-96 */
int b2s_get_max_index(const float* data, int size, int index, int group_size);                 /* collection_utils.h:9-14 */
int b2s_contains_with_margin(const int* keys, int n_keys, int index, int margin, int* found);  /* collection_utils.h:17-27 */
int b2s_most_frequent_value(const int* data, int n);                                           /* collection_utils.h:30-50 */
int b2s_learn_frames_from_ms(int64_t learning_ms, double frame_period_ms);                     /* NOISE_LEARNING_TIME -> frames */
int b2s_decimator_factor(int32_t sample_rate_hz, int32_t fft_size);                            /* sdr_device.cpp:150-152 */


/* ---- Transmission bookkeeping on HOST rows (operator-level parity with transmission.cpp:57-176; no GPU involved) ----
 * The same host tracker that follows K2's detection entries inside b2s_band_push, fed from dense rows instead:
 * box_rows[n_frames][N] = average(Averager::average(), GROUPING_X) and q_rows[n_frames][N] = the NoiseLearner output rows
 * (the Averager ring that getBestIndex votes on). Frames are stamped like b2s_band_push stamps them. With use_watch != 0 the
 * per-frame window maxima / candidate flags that K2 reports for the live keys are emulated as well (the path the band
 * takes in steady state); the lists must not depend on it. tx_count[n_frames], tx[n_frames][B2S_MAX_TX] (either may be
 * NULL). State (signal map, last Y rows of q) carries over between calls. */
typedef struct b2s_host_transmission b2s_host_transmission;
int b2s_host_transmission_create(const b2s_band_config* cfg, b2s_host_transmission** out);
int b2s_host_transmission_destroy(b2s_host_transmission* h);
int b2s_host_transmission_reset(b2s_host_transmission* h); /* Transmission::resetBuffers: drop the signals and the ring */
double b2s_host_transmission_last_run_ms(b2s_host_transmission* h); /* wall time of the bookkeeping of the last push (measurement) */
int b2s_host_transmission_push(b2s_host_transmission* h, const float* box_rows, const float* q_rows, int n_frames, int64_t t0_ms,
                               double frame_period_ms, int use_watch, int32_t* tx_count, b2s_transmission* tx);
/* the tracker's signal event log (always kept here; conventions of b2s_band_get_events): `frame` counts the frames pushed since
 * create */
int b2s_host_transmission_get_events(b2s_host_transmission* h, b2s_signal_event* out, int cap, int consume, int* count);

/* ---- wire formats of the reference's MQTT payloads (network/data_controller.cpp:27-57), little-endian, packed ----
 * so that rows / recordings produced here can be published to an unchanged sdr-hub. Both return 0 and the payload length in
 * *written, or B2S_E_INVALID when `cap` is too small (then *written holds the required size).
 * spectrogram ("sdr/<dev>/spectrogram"):        u64 time_ms, i32 start_hz, i32 stop_hz, i32 step_hz, u32 size, int8[size]
 * transmission ("sdr/<dev>/transmission/uint8"): u64 time_ms, i32 start_hz, i32 stop_hz, u32 sample_rate, uint8 IQ pairs (int8 ^ 0x80) */
int b2s_pack_spectrogram_message(int64_t time_ms, int32_t center_hz, int32_t sample_rate_hz, const int8_t* row, int size, uint8_t* out, size_t cap,
                                 size_t* written); /* DataController::pushSpectrogram, data_controller.cpp:44-57 */
int b2s_pack_transmission_message(int64_t time_ms, int32_t frequency_hz, int32_t sample_rate_hz, const int8_t* iq, int n_samples, uint8_t* out,
                                  size_t cap, size_t* written); /* DataController::pushTransmission, data_controller.cpp:27-42 */

/* ---- recorder bank: a device's pool of Recorders on one IQ stream (SdrDevice::m_recorders, sdr_device.cpp:39-41,82-144) ----
 * n_channels recorders that share one source, indexed like the scan policy's b2s_recorder_action.recorder. A channel computes exactly
 * the bytes of a b2s_recorder with the same rate, bandwidth, format and scale, started with the same shift before the same push and
 * fed the same pushes, whatever the other channels do. One push runs every recording channel: at most one host-to-device copy, one
 * launch per stage (per 64 recording channels), one device-to-host copy and one synchronise.
 * Like Recorder (recorder.cpp:35-39, buffer.h:22-55) each channel cuts its int8 output into chunks of
 * chunk_samples = roundUp(bandwidth * 100 / 1000, 4096) samples; chunk j (from 0) of a recording is stamped
 * start_ms + floor((j + 1) * chunk_samples * 1000 / bandwidth + 0.5), start_ms = t0_ms of the first non-empty push after start.
 * A push that would not fit (n_samples > max_samples_per_push, or an output longer than cap_samples) returns B2S_E_INVALID
 * before any work and changes nothing. */
typedef struct b2s_recorder_bank b2s_recorder_bank;
int b2s_recorder_bank_create(b2s_engine* e, int32_t sample_rate_hz, int32_t bandwidth_hz, int iq_format, float iq_scale,
                             int flags /* B2S_FLAG_IQ_ON_DEVICE */, int n_channels, size_t max_samples_per_push /* 0 -> 4 Mi */,
                             b2s_recorder_bank** out);
int b2s_recorder_bank_destroy(b2s_recorder_bank* k);
int b2s_recorder_bank_start(b2s_recorder_bank* k, int channel, int32_t shift_hz); /* Recorder::startRecording; B2S_E_STATE when recording */
int b2s_recorder_bank_stop(b2s_recorder_bank* k, int channel);                    /* Recorder::stopRecording: discards buffered output; B2S_E_STATE when idle */
/* the stream's next n_samples (t0_ms = injected time of the first one) through every recording channel.
   out_iq: optional [n_channels][cap_samples] int8 pairs (host); n_out: optional [n_channels] (0 for idle channels) */
int b2s_recorder_bank_push(b2s_recorder_bank* k, const void* iq, size_t n_samples, int64_t t0_ms,
                           int8_t* out_iq, size_t cap_samples, size_t* n_out);
/* Recorder::flush: the complete chunks buffered since the last flush, oldest first; up to `cap` are copied, *count = chunks available;
   with consume != 0 the chunks copied out (and only those) are dropped */
int b2s_recorder_bank_flush(b2s_recorder_bank* k, int channel, int8_t* chunks /*[cap][chunk_samples][2]*/, int64_t* times_ms,
                            int cap, int consume, int* count, int* chunk_samples);
/* Snapshot of a bank (conventions of b2s_band_save_state / b2s_band_load_state): the raw-sample carry and, per channel, whether it
 * records, its rotator and stream position, its rows of every stage's carry and its unflushed chunks. Saving first settles the piece
 * an asynchronous band left pending. A load needs the same sample rate, bandwidth, iq_format, iq_scale and channel count;
 * max_samples_per_push and the flags may differ. */
int b2s_recorder_bank_save_state(b2s_recorder_bank* k, void* buf, size_t cap, size_t* written);
int b2s_recorder_bank_load_state(b2s_recorder_bank* k, const void* buf, size_t len);
/* History: a recording can start at a sample already pushed to the bank, such as the first frame of a transmission that the band
 * reports only some frames later.
 * Keep the newest `samples` samples of the bank's stream on the device (0, the default: keep none). Every later push of the bank,
 * stand-alone or through an attached band, appends its samples. Positions count the samples pushed to the bank since the last
 * set_history or b2s_recorder_bank_load_state, which both empty the history. The call finishes the bank's outstanding work first.
 * A refused call (B2S_E_NOMEM) keeps the previous history. The history is not part of a snapshot. */
int b2s_recorder_bank_set_history(b2s_recorder_bank* k, size_t samples);
/* The positions the history holds: [*oldest, *end). */
int b2s_recorder_bank_history(b2s_recorder_bank* k, int64_t* oldest, int64_t* end);
/* Recorder::startRecording, but from stream position `position` (oldest <= position <= end) instead of from the next push. The samples
 * [position, end) are recorded at once ("catch-up"), cut every max_samples_per_push samples from `position`. The channel then continues
 * with the following pushes. Its chunks are stamped from start_ms. Its bytes and chunk times equal those of a channel of a fresh
 * stand-alone bank with the same settings, started with shift_hz and pushed [position, end) in those cuts (the first push at start_ms),
 * then the same later pushes; for position == end that is b2s_recorder_bank_start. B2S_E_STATE when the channel records; B2S_E_INVALID
 * for a position outside the history, or when the bank keeps none. */
int b2s_recorder_bank_start_from(b2s_recorder_bank* k, int channel, int32_t shift_hz, int64_t position, int64_t start_ms);

/* Record from the band's own pushes: every later b2s_band_push also runs `bank` over the pushed stream, reading the IQ the band
 * has already staged on the device (or the caller's device pointer). bank == NULL detaches. (SdrDevice connects its recorders to
 * the same source as the detection chain, sdr_device.cpp:39-41.)
 *   - Compatibility: the bank is on the band's engine, has the band's sample_rate_hz, iq_format and iq_scale, and its
 *     max_samples_per_push is at least max_frames_per_push * frame_stride_samples. A band has at most one bank and a bank is attached
 *     to at most one band; attaching a second bank is refused (detach first). Any other case returns B2S_E_INVALID and changes
 *     neither object. The bank's own B2S_FLAG_IQ_ON_DEVICE does not matter while it is attached.
 *   - What the bank sees: while a bank is attached, `iq` of b2s_band_push must hold the whole stream, n_frames * frame_stride_samples
 *     samples (without a bank, (n_frames - 1) * frame_stride_samples + fft_size are enough). A push of up to max_frames_per_push
 *     frames is exactly one bank push of n_frames * frame_stride_samples samples at the push's t0_ms; a longer push is cut every
 *     max_frames_per_push frames, piece j stamped t0_ms + floor(j * max_frames_per_push * frame_period_ms + 0.5). The band's own
 *     pipeline chunks and its cuts at the spectrogram emission limit do not show in the bank's pushes.
 *   - One upload: host IQ crosses PCIe once (b2s_profile.h2d_bytes grows by n_frames * frame_stride_samples * bytes per sample per
 *     push); the bank reads the band's copy. The band's results are those of the same band without a bank, bit for bit.
 *   - Device input: as without a bank, `iq` may be reused in the band's stream order once the call returns: work enqueued on the
 *     band's stream afterwards waits for the bank's reads of it, even when they are still running on the bank's own stream.
 *   - Completion: with a synchronous band the bank has consumed the push when b2s_band_push returns. With B2S_FLAG_ASYNC, b2s_band_push
 *     does not wait for the bank's kernels of the push's last piece; the bank's host side of that piece (the copy of the channels'
 *     output, the chunks) is done by the next b2s_band_push, b2s_band_sync or b2s_recorder_bank_* call on the bank, whichever comes
 *     first. start / stop act on the pushes after them, as for a stand-alone bank.
 *   - An attached bank is externally synchronised with its band: its calls must not run concurrently with that band's push.
 *   - Lifetimes: destroying an attached bank detaches it first (which drains the band's outstanding pushes); destroying a band
 *     detaches its bank, which stays usable. After a detach the bank's stream position continues: a stand-alone b2s_recorder_bank_push
 *     of the following samples continues the same recordings byte for byte. b2s_band_reset, b2s_band_set_center and noise learning do
 *     not touch the bank. */
int b2s_band_attach_recorder_bank(b2s_band* b, b2s_recorder_bank* bank);
/* Start channel `channel` of the band's attached bank at the first sample of band frame `frame` (counted like b2s_signal_event.frame),
 * stamped with that frame's injected clock: b2s_recorder_bank_start_from at the frame's position. Refused (B2S_E_INVALID, nothing
 * changes) when
 * - no bank is attached or it keeps no history;
 * - the frame is not yet pushed or no longer in the history;
 * - the frame was pushed before the bank was attached, before its last set_history, before the band's last b2s_band_load_state,
 *   or before the last b2s_band_set_center that changed the centre (that IQ belongs to another centre).
 * b2s_band_reset does not limit it. B2S_E_STATE when the channel records. With B2S_FLAG_ASYNC the frame may lie in a push whose
 * kernels are still running: the catch-up follows the bank's reads of it. Typical use: on B2S_REC_START from the scan policy, take
 * the START event with the same shift_hz and call this with event.frame minus a pre-roll instead of b2s_recorder_bank_start. */
int b2s_band_record_from(b2s_band* b, int channel, int32_t shift_hz, int64_t frame);

/* ---- auto-record: the band drives its attached bank the way SdrDevice::updateRecordings drives m_recorders (sdr_device.cpp:82-144) ----
 * After each push with at least one frame is finished, the band runs the reference's recorder assignment on that push's mailbox (the
 * list b2s_band_sync would return) at the clock of the push's last frame, and starts and stops the bank's channels itself. With a
 * synchronous band that happens before b2s_band_push returns; with B2S_FLAG_ASYNC in the next b2s_band_push (before it feeds the bank)
 * or b2s_band_sync, whichever comes first, after the push's bookkeeping has finished. The actions are exactly those a b2s_scan_policy
 * with n_channels recorders returns from b2s_scan_policy_notify for the same lists (its recorder half: hopping stays the caller's).
 *   - START: the band takes the latest START of the entry's key that K4 (or the host tracker) logged, and starts the channel at
 *     max(START frame - preroll_frames, the oldest frame b2s_band_record_from accepts), stamped with that frame's clock: what
 *     b2s_band_record_from does at that frame. All channels started by one decision catch up together. It starts the channel like
 *     b2s_recorder_bank_start instead (from the next push on, from_frame = -1) when the bank keeps no history, when
 *     b2s_band_record_from would refuse the START frame, when the START was logged before auto-record was enabled, or when the device
 *     log lost records (B2S_EV_LOST) at or after it. preroll_frames = 0 without history is exactly the reference's behaviour.
 *   - STOP stops the channel as b2s_recorder_bank_stop does (Recorder::stopRecording drops what was not flushed). FLUSH and NONE_FREE
 *     only report: collecting chunks with b2s_recorder_bank_flush stays the caller's.
 *   - The START records come from an internal log that does not depend on b2s_band_set_event_log: with the event log off,
 *     b2s_band_get_events still returns nothing, and consuming events does not affect auto-record. The band's own results (mailbox,
 *     map, spectrogram rows, events) are bit for bit those of the same band without auto-record.
 * Enabling needs an attached bank whose channels are all idle (B2S_E_INVALID without a bank, B2S_E_STATE with a recording channel;
 * nothing changes). While it is on, b2s_recorder_bank_start, b2s_recorder_bank_stop, b2s_recorder_bank_start_from and
 * b2s_band_record_from on the bank return B2S_E_STATE and change nothing. Enabling it again while on only changes preroll_frames.
 * Turning it off (enable = 0, detaching the bank, destroying either object, b2s_band_load_state) leaves the channels as they are, for
 * the caller to drive, and drops a decision not yet made. b2s_band_reset and b2s_band_set_center stop no recording: the next mailbox
 * does, as in the reference. Auto-record is not part of a snapshot. */
int b2s_band_set_auto_record(b2s_band* b, int enable, int32_t preroll_frames);
typedef struct b2s_auto_record_action {
  int32_t kind;        /* B2S_REC_START / STOP / FLUSH / NONE_FREE, as b2s_recorder_action */
  int32_t channel;     /* bank channel, -1 for NONE_FREE */
  int32_t shift_hz;
  int32_t key;         /* map key of the transmission */
  int64_t frame;       /* band frame of the push's last frame: when the reference would have acted */
  int64_t from_frame;  /* START: the band frame the recording starts at; -1 = started at the next push (no usable history) */
  int64_t time_ms;     /* injected clock of `frame`; START: the clock of from_frame, which stamps the chunks */
  int64_t duration_ms; /* STOP: Recorder::getDuration() */
} b2s_auto_record_action;
/* the actions taken, oldest first (conventions of b2s_band_get_events): up to `cap` are copied, *count is the number available; with
 * consume != 0 the actions copied out (and only those) are dropped */
int b2s_band_get_auto_record_actions(b2s_band* b, b2s_auto_record_action* out, int cap, int consume, int* count);

#ifdef __cplusplus
}
#endif
#endif /* B2S_H */
