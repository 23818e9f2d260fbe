// b2s_band: per-band state, the two halves of a push (GPU enqueue / result finish) and the optional result worker.
// Included by b2s_api.cu after its helpers (fail, CU, DevBuf, PinBuf, Stream, Event, launch_spectrum, SpectralTables).
//
// A push (or each pipeline chunk of one) goes through
//   enqueue_chunk : K1 -> K2 -> entry ordering on the band's stream, non-blocking on the host
//   finish_chunk  : read back the ordered detection entries, run the signal bookkeeping (tracker.h, K3 on demand),
//                   collect spectrogram rows / requested dense rows
// In the default (synchronous) mode both run on the caller's thread, one after the other. With B2S_FLAG_ASYNC the finish
// half runs on a worker thread with its own stream and a second set of per-push buffers ("slots"), so the kernels of
// push k+1 overlap the bookkeeping of push k — the same decoupling the reference gets from its 1-slot mailbox between
// the Transmission block thread and the Scanner thread (transmission.cpp:67, notification.h:14-26).
#pragma once

#include <condition_variable>
#include <deque>
#include <thread>

struct NoiseSlot {
  DevBuf<float> threshold[2];  // [cur]: the thresholds after the last enqueued push; K2 reads [cur] and writes [cur ^ 1]
  int cur = 0;
  float* now() { return threshold[cur].p; }
  int samples = 0;
  bool ready = false;
  // noise_learning_ms > 0 (NoiseLearner's own rule): Noise::m_startLearningTime = the stamp of the first frame this centre saw
  // (noise_learner.cpp:9,42: Noise() runs inside the first work() call on that centre)
  bool started = false;
  int64_t start_ms = 0;
};
struct SpectroSlot {
  DevBuf<float> sum;
  int counter = 0;
  int64_t last_send = 0;
};
// spectrum occupancy of one centre (b2s_band_set_occupancy): the device counts and max-hold, and the host's frame counts
struct OccupancySlot {
  DevBuf<unsigned int> above_start, above_stop;  // [N]
  DevBuf<float> max_db;                          // [N]
  int64_t frames = 0, detect_frames = 0;
  int64_t truncated = 0;  // counted chunks whose entry lists overflowed detect_capacity (written by the finish half, under qmutex)
};
struct SentRow {
  int64_t time;
  int32_t center;
  std::vector<int8_t> row;
};

constexpr int kPushSlots = 2;
constexpr int kRings = 3;  // ring before push k must survive while push k+1 writes its own "after" ring

struct PushSlot {
  // device buffers owned by the slot (live until the slot's finish half is done)
  DevBuf<float> psd, ckpt, dense_q, dense_avg, dense_box, peak_val;
  DevBuf<int> peak_idx, offsets, max_count;
  DevBuf<DetectEntry> sorted;
  DevBuf<signed char> spec_rows;
  DevBuf<unsigned int> watch_max;
  DevBuf<unsigned long long> cta_ns, peak_packed;
  CUtensorMap psd_map;  // PSD rows [max_frames][N] as a 2-D tensor, box = [32 frames][128 + 2*halo columns] (K2's tile)
  DevBuf<int> cand_flag;
  // device tracker (K4): runs of the frames' entries, the last frame's boxcar row, the push's result
  DevBuf<float> box_last;
  DevBuf<int> run_lo, run_hi, run_count;  // RunFold arrays of the chunk
  DevBuf<TrackResult> d_result;
  DevBuf<b2s_transmission> d_tx;  // [N] the push's whole sorted list (TrackArgs::tx)
  PinBuf<TrackResult> h_result;
  DevBuf<TrackEvent> d_log;  // [N] the signal event records of the chunk's K4 (TrackArgs::log); allocated while the log is on
  bool log_on = false;       // the event log was on when the chunk was enqueued
  bool log_starts = false;   // auto-record was on: K4 logs even with the event log off, and the STARTs go to the band's start_of
  int64_t frame_base = 0;    // frames pushed to the band before the chunk's first
  OccupancySlot* occ = nullptr;  // the centre's occupancy slot when occupancy was on at enqueue time
  Event sorted_done, tev[2];
  bool host_track = false;  // this chunk's bookkeeping runs on the host (the caller asked for every frame's list)
  int epoch = 0;            // reset_epoch when the chunk was enqueued
  PinBuf<int> h_offsets, h_cand_flag;
  PinBuf<unsigned int> h_watch_max;
  PinBuf<DetectEntry> h_entries;
  int n_watch = 0;
  int watch_key[kMaxWatch] = {0};
  Event gpu_done, ev[4];
  // context of the chunk in flight
  bool busy = false;
  int T = 0;
  int64_t t0_ms = 0;
  double period_ms = 0.0;
  size_t frame_offset = 0;
  int noise_samples = 0, learn_frames = 0, avg_frames_before = 0, ring_before = 0;  // frame t of the push was a learning frame iff noise_samples + t < learn_frames
  const float* threshold = nullptr;
  int32_t center = 0;
  int n_emit = 0;
  std::vector<int64_t> emit_time;
  bool dense_q_on = false, dense_avg_on = false, dense_box_on = false;
  b2s_result* out = nullptr;  // synchronous mode only
  std::vector<float> thr_host;
  bool thr_host_valid = false;
};

struct b2s_band : public DeviceQueries {
  b2s_engine* engine = nullptr;
  b2s_band_config cfg{};
  std::vector<float> user_window;  // the taps of a B2S_WINDOW_USER band, which a snapshot must match
  std::mutex mutex;  // serialises API calls on this band
  // The streams are declared before every buffer, so they are destroyed after them.
  Stream own_stream, finish_stream, copy_stream;
  Stream track_stream;            // K4 of push k runs here, beside K1 of push k+1 on `stream`
  cudaStream_t stream = nullptr;  // own_stream, or the caller's stream (b2s_band_set_stream)
  // the signal map (device resident; tracker.signals mirrors it only inside a host-tracked push): the live count and arrays of
  // N entries (TrackMap), and k_track_wide's hit words and sort keys. About 180 B per bin with the slots' d_tx.
  DevBuf<int> d_map_n, d_map_key;
  DevBuf<long long> d_map_first, d_map_last;
  DevBuf<float> d_map_power;
  DevBuf<unsigned int> d_track_hit;
  DevBuf<unsigned long long> d_track_sort;
  TrackMap track_map() { return TrackMap{d_map_n.p, d_map_key.p, d_map_first.p, d_map_last.p, d_map_power.p}; }
  Event copy_done[2], iq_prev_use[2];
  int iq_slot = 0;
  // recorder bank fed from this band's pushes (b2s_band_attach_recorder_bank). While one is attached, host input is staged with every
  // frame's whole stride: the synchronous path stages a whole piece of up to max_frames frames in d_whole (pipeline chunks at their
  // offsets), the asynchronous path reads d_iq, whose copy also waits for bank_prev_use[slot] (the bank's stage 0 of the last push that
  // read the buffer). push_ready marks, on `stream`, the start of a push with device input; the bank's stream waits for it. bank_read
  // marks, on the bank's stream, the end of its reads of the last piece from d_whole or the caller's device buffer: the next copy into
  // d_whole, and with device input the band's stream after the piece's kernels, wait for it.
  b2s_recorder_bank* bank = nullptr;
  DevBuf<unsigned char> d_whole;
  Event bank_prev_use[2], push_ready, bank_read;
  // The pieces fed to the bank while it keeps history, oldest first (b2s_band_record_from): the band frame and bank stream position of
  // each piece's first frame, and the clock of its push (frame `first` of the push starts the piece). Pieces that left the history
  // are dropped. Emptied when a bank is attached, when the centre changes and by a load; rows of an earlier history of the bank
  // (another hist_epoch) are void.
  struct HistPiece {
    int64_t frame, n_frames;
    long long position;
    int64_t t0_ms;
    double period_ms;
    size_t first;
  };
  std::deque<HistPiece> hist_pieces;
  uint64_t hist_epoch = 0;
  // Auto-record (b2s_band_set_auto_record): after each push the band runs the reference's recorder assignment on the push's mailbox and
  // starts and stops the attached bank's channels itself. `policy` holds the recorders' state; `key` the map key each channel was started
  // for; `due` marks a push whose decision has not run yet (its last frame and that frame's clock in frame, time_ms).
  struct AutoRecord {
    bool on = false;
    int32_t preroll = 0;
    int64_t enabled_at = 0;  // frames_pushed when it was enabled: START records of earlier frames are not used
    std::unique_ptr<host::ScanPolicy> policy;
    std::vector<int32_t> key;
    bool due = false;
    int64_t frame = 0, time_ms = 0;
  } autorec;
  std::deque<b2s_auto_record_action> auto_actions;  // not yet collected by b2s_band_get_auto_record_actions
  // The latest START record of each key from the device log (or the host tracker's) while auto-record is on, as (band frame, clock), and
  // the last frame of the newest chunk whose device log lost records (guarded by qmutex: the worker writes them)
  std::map<int32_t, std::pair<int64_t, int64_t>> start_of;
  int64_t start_lost_through = -1;
  int max_frames = 0;
  int slot_capacity = 0;  // detection entries per frame
  int detect_bins = kDetectBinsPerCta;  // bins per K2 CTA (DetectArgs::bins_per_cta)
  int wanted_capacity = 0;  // > slot_capacity after a push overflowed: applied by grow_capacity() before the next push
  bool async_mode = false;

  SpectralTables tables;
  DevBuf<unsigned char> d_iq[2];
  // B2S_FLAG_SUBFRAME_OVERLAP: frame 0's sub-frame 0 of the chunk K1 reads next, N samples: the lead-in (the last N / 2 samples of the
  // chunk before, kept here in stream order), then the chunk's first N / 2. has_lead: the next chunk's frame 0 has a lead-in.
  DevBuf<unsigned char> d_lead;
  bool has_lead = false;
  DevBuf<float> d_sum[2], d_ring[kRings], d_avg_last;  // m_sum: [sum_cur] after the last enqueued push (K2 reads it, writes the other)
  int sum_cur = 0;
  int ring_cur = 0;  // d_ring[ring_cur] = ring after the last enqueued push
  int avg_frames = 0;
  DevBuf<DetectEntry> d_slots;
  DevBuf<int> d_slot_count;
  DevBuf<float> d_wq_val;
  DevBuf<int> d_wq_idx;
  PinBuf<WindowWork> h_work;
  PushSlot slots[kPushSlots];
  int next_slot = 0;

  std::map<int32_t, NoiseSlot> noise;
  std::map<int32_t, SpectroSlot> spectro;
  // spectrum occupancy (off by default): one slot per centre pushed while it was on; turning it off keeps them. Not in a snapshot.
  bool occupancy = false;
  std::map<int32_t, OccupancySlot> occ;
  std::vector<SentRow> sent;
  int32_t center = 0;
  Tracker tracker;

  // result of the most recently finished chunk (the mailbox) + statistics since the last sync
  std::vector<b2s_transmission> mailbox;  // the complete list, strongest first (guarded by qmutex against reset_buffers)
  int reset_epoch = 0;                    // bumped by reset_buffers
  int stat_entries = 0, stat_rows = 0;
  // the signal event log (b2s_band_set_event_log): the events of the finished chunks, oldest first (guarded by qmutex)
  bool event_log = false;
  std::deque<b2s_signal_event> events;
  int64_t frames_pushed = 0;  // frames enqueued since the band was created: b2s_signal_event::frame of the next chunk's first

  // profiling
  bool profiling = false;
  bool profile_ctas = false;  // level 2: also per-CTA run times of K2 (one small D2H + sort per push)
  b2s_profile prof{};

  // worker (async mode)
  std::thread worker;
  std::mutex qmutex;
  std::condition_variable qcv;
  std::deque<int> queue;
  bool stop_worker = false;
  int worker_rc = 0;
  std::string worker_error;

  PushSlot* cur = nullptr;  // slot whose finish half is running (DeviceQueries context)
  cudaStream_t fstream() const { return async_mode ? finish_stream : stream; }

  // The worker reads the slots and the band's state until it stops: join it before any member is destroyed. The members then
  // free themselves.
  ~b2s_band() { shutdown_worker(); }

  // ---------------------------------------------------------------------------------------------------------
  int alloc_noise(NoiseSlot& s) {
    int rc = s.threshold[0].alloc(cfg.fft_size);
    if (!rc) rc = s.threshold[1].alloc(cfg.fft_size);
    return rc;
  }
  int noise_slot(NoiseSlot** out) {
    auto it = noise.find(center);
    if (it == noise.end()) {
      it = noise.emplace(center, NoiseSlot{}).first;
      int rc = alloc_noise(it->second);
      if (rc) return rc;
      std::vector<float> init(cfg.fft_size, -std::numeric_limits<float>::max());  // noise_learner.cpp:16
      CU(cudaMemcpyAsync(it->second.threshold[0].p, init.data(), sizeof(float) * cfg.fft_size, cudaMemcpyHostToDevice, stream));
      CU(cudaStreamSynchronize(stream));
    }
    *out = &it->second;
    return 0;
  }
  // counts zeroed, max-hold -inf, on `stream` (the next push's occupancy kernels follow in stream order)
  int clear_occupancy(OccupancySlot& o) {
    const size_t n = cfg.fft_size;
    CU(cudaMemsetAsync(o.above_start.p, 0, sizeof(unsigned int) * n, stream));
    CU(cudaMemsetAsync(o.above_stop.p, 0, sizeof(unsigned int) * n, stream));
    k_fill<<<static_cast<unsigned>((n + 255) / 256), 256, 0, stream>>>(o.max_db.p, -INFINITY, static_cast<int>(n));
    CU(cudaGetLastError());
    o.frames = o.detect_frames = o.truncated = 0;
    return 0;
  }
  // the current centre's occupancy slot, allocated and cleared on the first push at that centre
  int occupancy_slot(OccupancySlot** out) {
    auto it = occ.find(center);
    if (it == occ.end()) {
      OccupancySlot o;
      const size_t n = cfg.fft_size;
      int rc = o.above_start.alloc(n);
      if (!rc) rc = o.above_stop.alloc(n);
      if (!rc) rc = o.max_db.alloc(n);
      if (!rc) rc = clear_occupancy(o);
      if (rc) return rc;
      it = occ.emplace(center, std::move(o)).first;
    }
    *out = &it->second;
    return 0;
  }

  // ---- DeviceQueries (called from the tracker during the finish half; read the slot's buffers) ----
  int fetch_ring_window(int frame_first, int rows, int bin_lo, int width, float* out) override {
    PushSlot& s = *cur;
    const int n = cfg.fft_size, Y = cfg.grouping_y;
    cudaStream_t st = fstream();
    if (!s.thr_host_valid) {
      s.thr_host.resize(n);
      CU(cudaMemcpyAsync(s.thr_host.data(), s.threshold, sizeof(float) * n, cudaMemcpyDeviceToHost, st));
      CU(cudaStreamSynchronize(st));
      s.thr_host_valid = true;
    }
    const float* ring_before = d_ring[s.ring_before].p;  // ring as it was when this push began
    for (int r = 0; r < rows; ++r) {
      const int f = frame_first + r;
      float* dst = out + static_cast<size_t>(r) * width;
      if (f >= 0) {
        CU(cudaMemcpyAsync(dst, s.psd.p + static_cast<size_t>(f) * n + bin_lo, sizeof(float) * width, cudaMemcpyDeviceToHost, st));
      } else if (Y + f >= 0) {  // f = -1 is the newest pre-push row
        CU(cudaMemcpyAsync(dst, ring_before + static_cast<size_t>(Y + f) * n + bin_lo, sizeof(float) * width, cudaMemcpyDeviceToHost, st));
      } else {
        for (int i = 0; i < width; ++i) dst[i] = 0.0f;
      }
    }
    CU(cudaStreamSynchronize(st));
    for (int r = 0; r < rows; ++r) {
      const int f = frame_first + r;
      if (f < 0) continue;
      float* dst = out + static_cast<size_t>(r) * width;
      if (s.noise_samples + f < s.learn_frames) {
        for (int i = 0; i < width; ++i) dst[i] = kNoData;
      } else {
        for (int i = 0; i < width; ++i) dst[i] = dst[i] - s.thr_host[bin_lo + i];  // same IEEE subtraction as the kernel
      }
    }
    return 0;
  }

  int query_windows(const std::vector<Window>& w, std::vector<std::vector<float>>& values, std::vector<std::vector<int>>& indices) override {
    PushSlot& s = *cur;
    cudaStream_t st = fstream();
    std::vector<WindowWork> work;
    std::vector<int> offset(w.size());
    int total = 0, max_width = 0;
    const int half = cfg.grouping_x / 2;
    for (size_t q = 0; q < w.size(); ++q) {
      offset[q] = total;
      for (int f = w[q].frame_lo; f < w[q].frame_hi;) {
        const int end = std::min(w[q].frame_hi, (f / kCheckpointEvery + 1) * kCheckpointEvery);
        work.push_back(WindowWork{w[q].bin_lo, w[q].bin_hi, f, end, total + (f - w[q].frame_lo)});
        f = end;
      }
      total += w[q].frame_hi - w[q].frame_lo;
      max_width = std::max(max_width, w[q].bin_hi - w[q].bin_lo + 1 + 2 * half + 2 * kBoxSegment);
    }
    // the (small) work list stays in pinned host memory and is read by the kernel through its device alias: a
    // host->device copy here would queue behind the bulk IQ copy of the next pipeline chunk
    int rc = h_work.alloc(work.size());
    if (rc) return rc;
    if ((rc = d_wq_val.alloc(total))) return rc;
    if ((rc = d_wq_idx.alloc(total))) return rc;
    std::memcpy(h_work.p, work.data(), sizeof(WindowWork) * work.size());
    WindowWork* work_dev = nullptr;
    CU(cudaHostGetDevicePointer(reinterpret_cast<void**>(&work_dev), h_work.p, 0));
    WindowArgs a{};
    a.n = cfg.fft_size;
    a.group_y = cfg.grouping_y;
    a.group_x = cfg.grouping_x;
    a.psd = s.psd.p;
    a.threshold = s.threshold;
    a.noise_samples = s.noise_samples;
    a.learn_frames = s.learn_frames;
    a.ring_in = d_ring[s.ring_before].p;
    a.avg_frames = s.avg_frames_before;
    a.checkpoints = s.ckpt.p;
    a.work = work_dev;
    a.out_value = d_wq_val.p;
    a.out_index = d_wq_idx.p;
    const size_t smem = sizeof(float) * 2 * max_width;
    {  // a window of up to 4096 bins plus the boxcar halos: opt in once per device
      int rc2 = prepare_kernel(engine, k_window_query, 256, 64 * 1024, nullptr);
      if (rc2) return rc2;
      if (smem > 64 * 1024) return fail(B2S_E_INVALID, "window query of %zu bytes exceeds the kernel's shared-memory budget", smem);
    }
    Event w0, w1;
    if (profiling) {
      CU(cudaEventCreate(&w0.h));
      CU(cudaEventCreate(&w1.h));
      CU(cudaEventRecord(w0, st));
    }
    k_window_query<<<static_cast<unsigned>(work.size()), 256, smem, st>>>(a);
    CU(cudaGetLastError());
    if (profiling) CU(cudaEventRecord(w1, st));
    prof.window_launches += 1;
    std::vector<float> v(total);
    std::vector<int> ix(total);
    CU(cudaMemcpyAsync(v.data(), d_wq_val.p, sizeof(float) * total, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(ix.data(), d_wq_idx.p, sizeof(int) * total, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    prof.d2h_bytes += (sizeof(float) + sizeof(int)) * total;
    if (profiling) {
      float ms = 0.0f;
      CU(cudaEventElapsedTime(&ms, w0, w1));
      prof.window_ms += ms;
    }
    values.resize(w.size());
    indices.resize(w.size());
    for (size_t q = 0; q < w.size(); ++q) {
      const int len = w[q].frame_hi - w[q].frame_lo;
      values[q].assign(v.begin() + offset[q], v.begin() + offset[q] + len);
      indices[q].assign(ix.begin() + offset[q], ix.begin() + offset[q] + len);
    }
    return 0;
  }

  // ---------------------------------------------------------------------------------------------------------
  int init(b2s_engine* e, const b2s_band_config& c) {
    engine = e;
    cfg = c;
    CU(cudaSetDevice(e->device));
    max_frames = c.max_frames_per_push > 0 ? c.max_frames_per_push : default_max_frames(c.fft_size);
    // detection entries kept per frame: every bin of a wideband emitter is one (a 200 kHz FM carrier at 250 Hz/bin is 800), so the
    // default scales with N; an overflowing push still completes on the truncated lists, reports B2S_E_OVERFLOW and the
    // capacity grows before the next push (grow_capacity)
    slot_capacity = c.detect_capacity > 0 ? c.detect_capacity : std::max(256, std::min(4096, c.fft_size / 8));
    async_mode = (c.flags & B2S_FLAG_ASYNC) != 0;
    center = c.center_hz;
    CU(cudaStreamCreateWithFlags(&own_stream.h, cudaStreamNonBlocking));
    CU(cudaStreamCreateWithFlags(&finish_stream.h, cudaStreamNonBlocking));
    CU(cudaStreamCreateWithFlags(&track_stream.h, cudaStreamNonBlocking));
    stream = own_stream;
    int rc = tables.build(c);
    if (rc) return rc;
    if (overlapped(c)) {
      const size_t lead_bytes = static_cast<size_t>(c.fft_size) * (c.iq_format == B2S_IQ_CS8 ? 2 : 8);
      if ((rc = d_lead.alloc(lead_bytes))) return rc;
      CU(cudaMemset(d_lead.p, 0, lead_bytes));  // a snapshot taken before the first push saves defined bytes
    }
    if (c.window_kind == B2S_WINDOW_USER) user_window.assign(c.window_taps, c.window_taps + c.fft_size);
    cfg.window_taps = nullptr;
    const size_t n = c.fft_size, Y = c.grouping_y;
    const int n_slots = async_mode ? kPushSlots : 1;
    // K2's CTA width (one CTA per SM: its shared-memory ring takes the SM): 112 bins, unless 128 bins need fewer waves of CTAs.
    // On the 132 SMs of an H100, N = 16384 is 128 CTAs of 128 bins in one wave, where 112 bins would be 147 CTAs in two.
    // A spectrogram column of d raw bins must not straddle two CTAs, and the bins plus both boxcar halos have to fit the SUM
    // warps' columns.
    {
      const int d = c.spectrogram_out_size > 0 ? c.fft_size / c.spectrogram_out_size : 1;
      const int hp = (c.grouping_x / 2 + 3) & ~3;
      auto fits = [&](int bins) { return bins % d == 0 && bins + 2 * hp <= kSumThreads; };
      auto waves = [&](int bins) { return ((c.fft_size + bins - 1) / bins + e->sm_count - 1) / e->sm_count; };
      detect_bins = 0;
      if (c.fft_size >= 8192) {
        for (int bins : {112, 128, 96, 64}) {
          if (fits(bins)) {
            detect_bins = bins;
            break;
          }
        }
        if (detect_bins == 112 && fits(128) && waves(128) < waves(112)) detect_bins = 128;
      } else {
        // a small FFT has few columns: narrower CTAs (more halo per bin, but up to one CTA per SM) instead of 37 CTAs at N = 4096
        for (int bins = kBoxSegment; bins <= kDetectBinsPerCta; bins += kBoxSegment) {
          if (bins % d == 0 && bins + 2 * hp <= kSumThreads && (c.fft_size + bins - 1) / bins <= e->sm_count) {
            detect_bins = bins;
            break;
          }
        }
        if (!detect_bins && 112 % d == 0 && 112 + 2 * hp <= kSumThreads) detect_bins = 112;
      }
      if (!detect_bins)
        return fail(B2S_E_INVALID, "grouping_x %d (halo %d bins per side) with a spectrogram decimation of %d does not fit a K2 CTA of %d columns", c.grouping_x, hp, d, kSumThreads);
    }
    for (int i = 0; i < n_slots; ++i) {
      PushSlot& s = slots[i];
      if ((rc = s.psd.alloc(static_cast<size_t>(max_frames) * n))) return rc;
      {
        const int hp = (c.grouping_x / 2 + 3) & ~3;
        if ((rc = make_tile_map(&s.psd_map, s.psd.p, n, max_frames, detect_bins + 2 * hp, kDetectTileFrames))) return rc;
      }
      if ((rc = s.peak_idx.alloc(max_frames))) return rc;
      if ((rc = s.peak_val.alloc(max_frames))) return rc;
      if (tables.split > 1 && (rc = s.peak_packed.alloc(max_frames))) return rc;
      if ((rc = s.ckpt.alloc((static_cast<size_t>(max_frames) / kCheckpointEvery + 1) * n))) return rc;
      if ((rc = s.sorted.alloc(static_cast<size_t>(max_frames) * slot_capacity))) return rc;
      if ((rc = s.offsets.alloc(max_frames + 1))) return rc;
      if ((rc = s.max_count.alloc(1))) return rc;
      if ((rc = s.h_offsets.alloc(max_frames + 2))) return rc;
      if ((rc = s.h_entries.alloc(static_cast<size_t>(max_frames) * 64))) return rc;
      if ((rc = s.watch_max.alloc(static_cast<size_t>(max_frames) * kMaxWatch))) return rc;
      if ((rc = s.cand_flag.alloc(max_frames))) return rc;
      if ((rc = s.h_watch_max.alloc(static_cast<size_t>(max_frames) * kMaxWatch))) return rc;
      if ((rc = s.h_cand_flag.alloc(max_frames))) return rc;
      CU(cudaEventCreateWithFlags(&s.gpu_done.h, cudaEventDisableTiming));
      CU(cudaEventCreateWithFlags(&s.sorted_done.h, cudaEventDisableTiming));
      if ((rc = s.box_last.alloc(n))) return rc;
      if ((rc = s.run_lo.alloc(static_cast<size_t>(2 * kRunCap) * max_frames))) return rc;
      if ((rc = s.run_hi.alloc(static_cast<size_t>(2 * kRunCap) * max_frames))) return rc;
      if ((rc = s.run_count.alloc(static_cast<size_t>(2) * max_frames))) return rc;
      if ((rc = s.d_result.alloc(1))) return rc;
      if ((rc = s.d_tx.alloc(n))) return rc;
      if ((rc = s.h_result.alloc(1))) return rc;
    }
    if ((rc = d_map_n.alloc(1)) || (rc = d_map_key.alloc(n)) || (rc = d_map_first.alloc(n)) || (rc = d_map_last.alloc(n)) || (rc = d_map_power.alloc(n))) return rc;
    CU(cudaMemset(d_map_n.p, 0, sizeof(int)));
    if ((rc = d_track_hit.alloc(n * kTrackWords))) return rc;
    {
      size_t sort_cap = 2;
      while (sort_cap < n) sort_cap <<= 1;
      if ((rc = d_track_sort.alloc(sort_cap))) return rc;
    }
    if ((rc = d_sum[0].alloc(n))) return rc;
    if ((rc = d_sum[1].alloc(n))) return rc;
    for (auto& r : d_ring) {
      if ((rc = r.alloc(Y * n))) return rc;
    }
    if ((rc = d_avg_last.alloc(n))) return rc;
    if ((rc = d_slots.alloc(static_cast<size_t>((max_frames + 31) & ~31) * slot_capacity))) return rc;
    if ((rc = d_slot_count.alloc(max_frames))) return rc;
    rc = reset_averager();
    if (rc) return rc;
    TrackerParams& p = tracker.p;
    p.n = c.fft_size;
    p.sample_rate = c.sample_rate_hz;
    p.center = c.center_hz;
    p.range_lo = c.range_lo_hz;
    p.range_hi = c.range_hi_hz;
    p.n_ignored = c.n_ignored;
    for (int i = 0; i < c.n_ignored; ++i) {
      p.ignored_lo[i] = c.ignored_lo_hz[i];
      p.ignored_hi[i] = c.ignored_hi_hz[i];
    }
    p.group_size = c.group_size_bins;
    p.group_y = c.grouping_y;
    p.start_level = c.start_level;
    p.stop_level = c.stop_level;
    p.tuning_step = c.tuning_step_hz;
    p.min_time = c.min_time_ms;
    p.timeout = c.timeout_ms;
    p.max_time = c.max_time_ms;
    if (async_mode) {
      for (int i = 0; i < 2; ++i) {
        CU(cudaEventCreateWithFlags(&iq_prev_use[i].h, cudaEventDisableTiming));
        CU(cudaEventRecord(iq_prev_use[i], stream));
      }
      worker = std::thread([this]() { worker_loop(); });
    }
    return 0;
  }

  // ---- the signal map: device resident (K4); mirrored into tracker.signals around a host-tracked push ----
  // bins whose frequency (indexToFrequency, sdr_device.cpp:153) lies in [f_lo, f_hi]: the frequency is monotonic in the bin
  void bins_between(int32_t f_lo, int32_t f_hi, int* lo, int* hi) const {
    const int n = tracker.p.n;
    int a = 0, b = n;  // first bin with frequency >= f_lo
    while (a < b) {
      const int m = (a + b) / 2;
      if (tracker.index_to_frequency(m) < f_lo) a = m + 1; else b = m;
    }
    *lo = a;
    a = 0, b = n;      // first bin with frequency > f_hi
    while (a < b) {
      const int m = (a + b) / 2;
      if (tracker.index_to_frequency(m) <= f_hi) a = m + 1; else b = m;
    }
    *hi = a - 1;
  }
  TrackParams track_params() {
    TrackParams tp{};
    tracker.p.center = center;
    const TrackerParams& p = tracker.p;
    tp.n = p.n;
    tp.sample_rate = p.sample_rate;
    tp.center = center;
    bins_between(p.range_lo, p.range_hi, &tp.bin_lo, &tp.bin_hi);
    tp.n_ignored = p.n_ignored;
    for (int i = 0; i < p.n_ignored; ++i) bins_between(p.ignored_lo[i], p.ignored_hi[i], &tp.ignored_lo[i], &tp.ignored_hi[i]);
    tp.group_size = p.group_size;
    tp.group_y = p.group_y;
    tp.start_level = p.start_level;
    tp.stop_level = p.stop_level;
    tp.tuning_step = p.tuning_step;
    tp.min_time = p.min_time;
    tp.timeout = p.timeout;
    tp.max_time = p.max_time;
    return tp;
  }
  struct HostMap {
    std::vector<int> key;
    std::vector<long long> first, last;
    std::vector<float> power;
  };
  int download_state(HostMap& h) {
    CU(cudaStreamSynchronize(track_stream));
    int count = 0;
    CU(cudaMemcpy(&count, d_map_n.p, sizeof(int), cudaMemcpyDeviceToHost));
    h.key.resize(count);
    h.first.resize(count);
    h.last.resize(count);
    h.power.resize(count);
    if (count > 0) {
      CU(cudaMemcpy(h.key.data(), d_map_key.p, sizeof(int) * count, cudaMemcpyDeviceToHost));
      CU(cudaMemcpy(h.first.data(), d_map_first.p, sizeof(long long) * count, cudaMemcpyDeviceToHost));
      CU(cudaMemcpy(h.last.data(), d_map_last.p, sizeof(long long) * count, cudaMemcpyDeviceToHost));
      CU(cudaMemcpy(h.power.data(), d_map_power.p, sizeof(float) * count, cudaMemcpyDeviceToHost));
    }
    return 0;
  }
  int state_to_host_tracker() {
    HostMap h;
    int rc = download_state(h);
    if (rc) return rc;
    tracker.signals.clear();
    for (size_t i = 0; i < h.key.size(); ++i) tracker.signals[h.key[i]] = TrackedSignal{h.first[i], h.last[i], h.power[i], -1};
    return 0;
  }
  int host_tracker_to_state() {
    HostMap h;
    for (const auto& kv : tracker.signals) {
      h.key.push_back(kv.first);
      h.first.push_back(kv.second.first);
      h.last.push_back(kv.second.last);
      h.power.push_back(kv.second.power);
    }
    const int count = static_cast<int>(h.key.size());
    if (count > 0) {
      CU(cudaMemcpy(d_map_key.p, h.key.data(), sizeof(int) * count, cudaMemcpyHostToDevice));
      CU(cudaMemcpy(d_map_first.p, h.first.data(), sizeof(long long) * count, cudaMemcpyHostToDevice));
      CU(cudaMemcpy(d_map_last.p, h.last.data(), sizeof(long long) * count, cudaMemcpyHostToDevice));
      CU(cudaMemcpy(d_map_power.p, h.power.data(), sizeof(float) * count, cudaMemcpyHostToDevice));
    }
    CU(cudaMemcpy(d_map_n.p, &count, sizeof(int), cudaMemcpyHostToDevice));
    return 0;
  }

  // Averager::reset (averager.cpp:27-34) / constructor state (averager.cpp:7-12)
  int reset_averager() {
    const size_t n = cfg.fft_size, Y = cfg.grouping_y;
    // Stream-ordered and non-blocking: the buffers the NEXT push's K2 reads (m_sum, the current ring) are cleared behind the
    // kernels already enqueued; the rings / sums older pushes still read (K4's getBestIndex) are not touched.
    CU(cudaMemsetAsync(d_sum[sum_cur].p, 0, sizeof(float) * n, stream));
    CU(cudaMemsetAsync(d_ring[ring_cur].p, 0, sizeof(float) * Y * n, stream));
    k_fill<<<static_cast<unsigned>((n + 255) / 256), 256, 0, stream>>>(d_avg_last.p, kNoData, static_cast<int>(n));
    CU(cudaGetLastError());
    avg_frames = 0;
    return 0;
  }
  // Transmission::resetBuffers (transmission.cpp:42-55): signals.clear() + Averager::reset(); the noise thresholds stay. Enqueued
  // behind the pushes already in flight (Scanner hops every 500 ms, scanner.cpp:46-60: a hop must not drain the pipeline).
  int reset_buffers() {
    tracker.reset();
    CU(cudaMemsetAsync(d_map_n.p, 0, sizeof(int), track_stream));  // behind the K4 of every earlier push, before the next one's
    {
      std::lock_guard<std::mutex> lk(qmutex);
      reset_epoch += 1;  // a chunk enqueued before this moment must not publish its (pre-reset) list afterwards
      mailbox.clear();
    }
    return reset_averager();
  }

  // after an overflow: enlarge the per-frame entry lists (no chunk may be in flight)
  int grow_capacity() {
    if (wanted_capacity <= slot_capacity) return 0;
    int rc = drain();
    if (rc) return rc;
    CU(cudaStreamSynchronize(stream));
    const int cap = std::min(cfg.fft_size, wanted_capacity);
    const int n_slots = async_mode ? kPushSlots : 1;
    for (int i = 0; i < n_slots; ++i) {
      if ((rc = slots[i].sorted.alloc(static_cast<size_t>(max_frames) * cap))) return rc;
    }
    if ((rc = d_slots.alloc(static_cast<size_t>((max_frames + 31) & ~31) * cap))) return rc;
    slot_capacity = cap;
    return 0;
  }

  // ---- snapshot (b2s_band_save_state / b2s_band_load_state; the format is snapshot.h's): everything the next push reads and everything
  // not yet collected ----
  // the per-frame entry capacity of the next push (grow_capacity applies a pending growth first)
  int next_capacity() const { return std::min(cfg.fft_size, std::max(slot_capacity, wanted_capacity)); }

  int save_state(std::vector<uint8_t>& out) {
    int rc = drain();
    if (rc) return rc;
    CU(cudaStreamSynchronize(stream));
    CU(cudaStreamSynchronize(track_stream));
    snapshot::BandImage s;
    s.center = center, s.range_lo = tracker.p.range_lo, s.range_hi = tracker.p.range_hi, s.frames_pushed = frames_pushed;
    s.event_log = event_log, s.stat_entries = stat_entries, s.stat_rows = stat_rows, s.capacity = next_capacity();
    for (auto& kv : noise) s.noise.push_back({kv.first, kv.second.samples, kv.second.ready, kv.second.started, kv.second.start_ms, kv.second.now()});
    for (auto& kv : spectro) s.spectro.push_back({kv.first, kv.second.counter, kv.second.last_send, kv.second.sum.p});
    s.avg_frames = avg_frames, s.avg_sum = d_sum[sum_cur].p, s.avg_last = d_avg_last.p, s.ring = d_ring[ring_cur].p;
    CU(cudaMemcpy(&s.live, d_map_n.p, sizeof(int), cudaMemcpyDeviceToHost));
    s.key = d_map_key.p, s.first = d_map_first.p, s.last = d_map_last.p, s.power = d_map_power.p;
    s.has_lead = has_lead, s.lead = d_lead.p;
    std::lock_guard<std::mutex> lk(qmutex);
    return snapshot::write(snapshot::kBand, stream, out,
                           [&](snapshot::Writer& w) { snapshot::band_sections(w, s, mailbox, events, sent, cfg, user_window.data()); });
  }

  int load_state(const void* buf, size_t len) {
    int rc = drain();
    if (rc) return rc;
    CU(cudaStreamSynchronize(stream));
    CU(cudaStreamSynchronize(track_stream));
    // ---- read and check everything before anything changes ----
    snapshot::BandImage s;
    std::vector<b2s_transmission> s_mailbox;
    std::deque<b2s_signal_event> s_events;
    std::vector<SentRow> s_sent;
    if ((rc = snapshot::read(buf, len, snapshot::kBand, "b2s_band_load_state", [&](snapshot::Reader& r) {
           snapshot::band_sections(r, s, s_mailbox, s_events, s_sent, cfg, user_window.data());
         })))
      return rc;
    const size_t n = cfg.fft_size, Y = cfg.grouping_y, M = std::max(cfg.spectrogram_out_size, 0);

    // ---- allocate: the new noise and spectrogram slots, and the larger entry lists ----
    std::map<int32_t, NoiseSlot> new_noise;
    for (const snapshot::NoiseImage& x : s.noise) {
      NoiseSlot& ns = new_noise[x.center];
      if ((rc = alloc_noise(ns))) return rc;
      ns.samples = x.samples, ns.ready = x.ready, ns.started = x.started, ns.start_ms = x.start_ms;
    }
    std::map<int32_t, SpectroSlot> new_spectro;
    for (const snapshot::SpectroImage& x : s.spectro) {
      SpectroSlot& ss = new_spectro[x.center];
      if ((rc = ss.sum.alloc(M))) return rc;
      ss.counter = x.counter, ss.last_send = x.last_send;
    }
    const int wanted_before = wanted_capacity;
    wanted_capacity = std::max(wanted_capacity, s.capacity);
    if ((rc = grow_capacity())) {
      wanted_capacity = wanted_before;
      return rc;
    }

    // ---- replace ----
    for (const snapshot::NoiseImage& x : s.noise) CU(cudaMemcpyAsync(new_noise[x.center].threshold[0].p, x.thr, sizeof(float) * n, cudaMemcpyHostToDevice, stream));
    for (const snapshot::SpectroImage& x : s.spectro) CU(cudaMemcpyAsync(new_spectro[x.center].sum.p, x.sum, sizeof(float) * M, cudaMemcpyHostToDevice, stream));
    CU(cudaMemcpyAsync(d_sum[sum_cur].p, s.avg_sum, sizeof(float) * n, cudaMemcpyHostToDevice, stream));
    CU(cudaMemcpyAsync(d_avg_last.p, s.avg_last, sizeof(float) * n, cudaMemcpyHostToDevice, stream));
    CU(cudaMemcpyAsync(d_ring[ring_cur].p, s.ring, sizeof(float) * n * Y, cudaMemcpyHostToDevice, stream));
    const size_t live = s.live;
    CU(cudaMemcpyAsync(d_map_key.p, s.key, sizeof(int) * live, cudaMemcpyHostToDevice, stream));
    CU(cudaMemcpyAsync(d_map_first.p, s.first, sizeof(long long) * live, cudaMemcpyHostToDevice, stream));
    CU(cudaMemcpyAsync(d_map_last.p, s.last, sizeof(long long) * live, cudaMemcpyHostToDevice, stream));
    CU(cudaMemcpyAsync(d_map_power.p, s.power, sizeof(float) * live, cudaMemcpyHostToDevice, stream));
    CU(cudaMemcpyAsync(d_map_n.p, &s.live, sizeof(int), cudaMemcpyHostToDevice, stream));
    if (d_lead.p) CU(cudaMemcpyAsync(d_lead.p, s.lead, d_lead.n / 2, cudaMemcpyHostToDevice, stream));
    CU(cudaStreamSynchronize(stream));  // K4 reads the map on track_stream, which waits for `stream` in every push
    has_lead = s.has_lead;
    noise.swap(new_noise);
    spectro.swap(new_spectro);
    center = tracker.p.center = s.center, tracker.p.range_lo = s.range_lo, tracker.p.range_hi = s.range_hi, frames_pushed = s.frames_pushed;
    event_log = s.event_log, stat_entries = s.stat_entries, stat_rows = s.stat_rows, avg_frames = s.avg_frames;
    tracker.signals.clear();
    sent.swap(s_sent);
    // the frames pushed before belong to another stream: so do the bank history's pieces, auto-record and its START records
    hist_pieces.clear();
    autorec = AutoRecord{};
    std::lock_guard<std::mutex> lk(qmutex);
    mailbox.swap(s_mailbox);
    events.swap(s_events);
    start_of.clear();
    return 0;
  }

  // ---- worker ----
  void worker_loop() {
    cudaSetDevice(engine->device);
    for (;;) {
      int idx;
      {
        std::unique_lock<std::mutex> lk(qmutex);
        qcv.wait(lk, [&] { return stop_worker || !queue.empty(); });
        if (queue.empty()) return;
        idx = queue.front();
      }
      const int rc = finish_chunk(slots[idx]);
      {
        std::lock_guard<std::mutex> lk(qmutex);
        if (rc && !worker_rc) {
          worker_rc = rc;
          worker_error = g_error;
        }
        queue.pop_front();
        slots[idx].busy = false;
      }
      qcv.notify_all();
    }
  }
  void shutdown_worker() {
    if (worker.joinable()) {
      {
        std::lock_guard<std::mutex> lk(qmutex);
        stop_worker = true;
      }
      qcv.notify_all();
      worker.join();
    }
  }
  // wait until every enqueued chunk has been finished; surfaces a worker error once
  int drain() {
    if (!async_mode) return 0;
    std::unique_lock<std::mutex> lk(qmutex);
    qcv.wait(lk, [&] { return queue.empty(); });
    if (worker_rc) {
      const int rc = worker_rc;
      g_error = worker_error;
      worker_rc = 0;
      return rc;
    }
    return 0;
  }
  int wait_slot_free(int idx) {
    if (!async_mode) return 0;
    std::unique_lock<std::mutex> lk(qmutex);
    qcv.wait(lk, [&] { return !slots[idx].busy; });
    return 0;
  }

  // Longest prefix of `frames` frames starting at push frame `frame_offset` during which at most kMaxSpecEmits spectrogram rows
  // complete (Spectrogram::send fires on the first frame later than last_send + interval, spectrogram.cpp:62-64). Pure: the
  // slot's clock state is only advanced by enqueue_chunk.
  size_t emit_limited_length(int64_t t0_ms, double period_ms, size_t frame_offset, size_t frames) const {
    if (cfg.spectrogram_out_size <= 0) return frames;
    int64_t last_send = host::frame_time(t0_ms, period_ms, frame_offset);  // a new centre starts its clock on its first frame
    auto it = spectro.find(center);
    if (it != spectro.end()) last_send = it->second.last_send;
    int emits = 0;
    for (size_t t = 0; t < frames; ++t) {
      const int64_t now = host::frame_time(t0_ms, period_ms, frame_offset + t);
      if (last_send + cfg.spectrogram_interval_ms < now) {
        if (emits == kMaxSpecEmits) return t;
        ++emits;
        last_send = now;
      }
    }
    return frames;
  }

  int enqueue_chunk(PushSlot& s, const void* iq_dev, size_t frames, int64_t t0_ms, double period_ms, size_t frame_offset, b2s_result* out);
  int finish_chunk(PushSlot& s);
  int push_chunk(const void* iq_dev, size_t frames, int64_t t0_ms, double period_ms, size_t frame_offset, b2s_result* out) {
    // a chunk may complete at most kMaxSpecEmits spectrogram rows (they travel as kernel arguments): cut it there
    const size_t stride_bytes = static_cast<size_t>(cfg.frame_stride_samples) * (cfg.iq_format == B2S_IQ_CS8 ? 2 : 8);
    for (size_t done = 0; done < frames;) {
      const size_t len = emit_limited_length(t0_ms, period_ms, frame_offset + done, frames - done);
      int rc = push_piece(static_cast<const char*>(iq_dev) + done * stride_bytes, len, t0_ms, period_ms, frame_offset + done, out);
      if (rc) return rc;
      done += len;
    }
    return 0;
  }
  int push_piece(const void* iq_dev, size_t frames, int64_t t0_ms, double period_ms, size_t frame_offset, b2s_result* out) {
    const int idx = async_mode ? next_slot : 0;
    int rc = wait_slot_free(idx);
    if (rc) return rc;
    PushSlot& s = slots[idx];
    if ((rc = enqueue_chunk(s, iq_dev, frames, t0_ms, period_ms, frame_offset, out))) return rc;
    if (!async_mode) return finish_chunk(s);
    {
      std::lock_guard<std::mutex> lk(qmutex);
      s.busy = true;
      queue.push_back(idx);
    }
    qcv.notify_all();
    next_slot = (next_slot + 1) % kPushSlots;
    return 0;
  }
};

// GPU half: everything is enqueued on `stream`; the host does not wait.
int b2s_band::enqueue_chunk(PushSlot& s, const void* iq_dev, size_t frames, int64_t t0_ms, double period_ms, size_t frame_offset, b2s_result* out) {
  const int n = cfg.fft_size, Y = cfg.grouping_y;
  const int T = static_cast<int>(frames);
  const size_t bytes_per_sample = cfg.iq_format == B2S_IQ_CS8 ? 2 : 8;
  int rc;
  s.epoch = reset_epoch;
  s.host_track = out && out->frame_tx_count;  // every frame's list is wanted: the bookkeeping runs on the host (tracker.h)
  s.log_on = event_log;
  s.log_starts = autorec.on;
  s.frame_base = frames_pushed;
  s.occ = nullptr;
  if (occupancy && (rc = occupancy_slot(&s.occ))) return rc;
  if ((s.log_on || s.log_starts) && !s.host_track && (rc = s.d_log.alloc(n))) return rc;
  if (s.host_track && (rc = state_to_host_tracker())) return rc;
  s.dense_q_on = out && out->noise_sub_db;
  s.dense_avg_on = out && out->avg_db;
  s.dense_box_on = out && out->box_db;
  if (s.dense_q_on && (rc = s.dense_q.alloc(static_cast<size_t>(max_frames) * n))) return rc;
  if (s.dense_avg_on && (rc = s.dense_avg.alloc(static_cast<size_t>(max_frames) * n))) return rc;
  if (s.dense_box_on && (rc = s.dense_box.alloc(static_cast<size_t>(max_frames) * n))) return rc;
  if (profiling) {
    for (auto& e : s.ev) {
      if (!e) CU(cudaEventCreate(&e.h));
    }
  }

  // ---- K1: spectra ----
  SpectralArgs sa{};
  sa.iq = iq_dev;
  sa.frame_stride_bytes = static_cast<long long>(cfg.frame_stride_samples) * bytes_per_sample;
  sa.n_frames = T;
  tables.fill(sa);
  sa.peak_packed = s.peak_packed.p;
  sa.reserve_sms = 1;  // K4 (one CTA, on track_stream) runs beside this K1: the persistent grid leaves it an SM
  sa.inv_fs = 1.0f / static_cast<float>(cfg.sample_rate_hz);
  sa.psd_db = s.psd.p;
  sa.power_lin = nullptr;
  sa.peak_index = s.peak_idx.p;
  sa.peak_value = s.peak_val.p;
  sa.zero_per_frame[0] = d_slot_count.p;  // K2's per-frame counters are zeroed by K1 (no memsets between the two kernels)
  sa.zero_per_frame[1] = s.cand_flag.p;
  sa.zero_scalar = s.max_count.p;
  const size_t half_bytes = static_cast<size_t>(n / 2) * bytes_per_sample;
  if (d_lead.p) {  // overlapping sub-frames: frame 0's sub-frame 0 is the lead-in and the chunk's first N / 2 samples, or is dropped
    CU(cudaMemcpyAsync(d_lead.p + half_bytes, iq_dev, half_bytes, cudaMemcpyDeviceToDevice, stream));
    sa.sub_lead = has_lead ? d_lead.p : nullptr;
    sa.sub_first = has_lead ? 0 : 1;
  }
  if (profiling) CU(cudaEventRecord(s.ev[0], stream));
  if ((rc = launch_spectrum(engine, n, cfg.iq_format, sa, stream))) return rc;
  if (profiling) CU(cudaEventRecord(s.ev[1], stream));
  if (d_lead.p) {  // the next chunk's lead-in: this one's last N / 2 samples, behind this K1's reads of d_lead
    CU(cudaMemcpyAsync(d_lead.p, static_cast<const char*>(iq_dev) + T * sa.frame_stride_bytes - half_bytes, half_bytes, cudaMemcpyDeviceToDevice, stream));
    has_lead = true;
  }

  // ---- plan the spectrogram emissions of this chunk from the clock (Spectrogram::send, spectrogram.cpp:62-75) ----
  int n_emit = 0;
  int emit_frames[kMaxSpecEmits] = {0}, emit_divs[kMaxSpecEmits] = {0};
  SpectroSlot* ss = nullptr;
  const int M = cfg.spectrogram_out_size;
  s.emit_time.clear();
  if (M > 0) {
    auto it = spectro.find(center);
    if (it == spectro.end()) {
      it = spectro.emplace(center, SpectroSlot{}).first;
      if ((rc = it->second.sum.alloc(M))) return rc;
      CU(cudaMemsetAsync(it->second.sum.p, 0, sizeof(float) * M, stream));
      it->second.counter = 0;  // the reference leaves m_counter uninitialised (spectrogram.cpp:9); defined as 0
      it->second.last_send = host::frame_time(t0_ms, period_ms, frame_offset);  // Container ctor: getTime()
    }
    ss = &it->second;
    for (int t = 0; t < T; ++t) {
      const int64_t now = host::frame_time(t0_ms, period_ms, frame_offset + t);
      ss->counter++;
      if (ss->last_send + cfg.spectrogram_interval_ms < now) {
        if (n_emit >= kMaxSpecEmits) return fail(B2S_E_STATE, "internal: chunk not cut at the spectrogram emission limit");  // push_chunk cuts chunks with emit_limited_length
        emit_frames[n_emit] = t;
        emit_divs[n_emit] = ss->counter;
        ++n_emit;
        s.emit_time.push_back(now);
        ss->counter = 0;
        ss->last_send = now;
      }
    }
    if (n_emit > 0 && (rc = s.spec_rows.alloc(static_cast<size_t>(n_emit) * M))) return rc;
  }

  // ---- K2: noise / averager / boxcar / detect / spectrogram ----
  NoiseSlot* ns = nullptr;
  if ((rc = noise_slot(&ns))) return rc;
  s.n_watch = 0;
  if (s.host_track) {  // the host tracker is helped by K2's watched-window maxima of the keys that are live now
    for (const auto& kv : tracker.signals) {
      if (s.n_watch < kMaxWatch) s.watch_key[s.n_watch++] = kv.first;
    }
  }
  if (s.n_watch > 0) CU(cudaMemsetAsync(s.watch_max.p, 0, sizeof(unsigned int) * static_cast<size_t>(T) * kMaxWatch, stream));
  const int ring_in = ring_cur, ring_out = (ring_cur + 1) % kRings;
  DetectArgs da{};
  da.n = n;
  da.n_frames = T;
  da.group_y = Y;
  da.group_x = cfg.grouping_x;
  da.psd = s.psd.p;
  da.threshold = ns->threshold[ns->cur].p;
  da.threshold_out = ns->threshold[ns->cur ^ 1].p;
  // learning frames of this push: frame t is one iff noise_samples + t < learn_frames (K2, K3 and K4 share the predicate)
  bool ready_after = ns->ready;
  int learned_here = 0;
  if (ns->ready) {
    da.noise_samples = da.learn_frames = 0;
  } else if (cfg.noise_learning_ms > 0) {
    // NoiseLearner's own rule on the frame clock (noise_learner.cpp:11,23): every frame up to AND INCLUDING the first one stamped at or
    // after start + NOISE_LEARNING_TIME is a learning frame; the time the band spent on other centres counts
    if (!ns->started) {
      ns->started = true;
      ns->start_ms = host::frame_time(t0_ms, period_ms, frame_offset);
    }
    int last = -1;
    for (int t = 0; t < T; ++t) {
      if (ns->start_ms + cfg.noise_learning_ms <= host::frame_time(t0_ms, period_ms, frame_offset + t)) {
        last = t;
        break;
      }
    }
    da.noise_samples = 0;
    da.learn_frames = last >= 0 ? last + 1 : T + 1;  // T + 1: all T frames of this push, and not finished
    learned_here = last >= 0 ? last + 1 : T;
    ready_after = last >= 0;
  } else {
    da.noise_samples = ns->samples;
    da.learn_frames = cfg.learn_frames;
    learned_here = std::min(T, cfg.learn_frames - ns->samples);
    ready_after = ns->samples + T >= cfg.learn_frames;
  }
  da.avg_sum = d_sum[sum_cur].p;
  da.avg_sum_out = d_sum[sum_cur ^ 1].p;
  da.ring_in = d_ring[ring_in].p;
  da.ring_out = d_ring[ring_out].p;
  da.avg_frames = avg_frames;
  da.avg_last = d_avg_last.p;
  da.checkpoints = s.ckpt.p;
  da.detect_level = std::min(cfg.start_level, cfg.stop_level);
  // an interior boxcar window holds 2 * (X / 2) + 1 bins (X + 1 for an even X), and that is what its sum is divided by
  da.detect_sum = least_sum_reaching(da.detect_level, 2 * (cfg.grouping_x / 2) + 1);
  da.start_sum = least_sum_reaching(cfg.start_level, 2 * (cfg.grouping_x / 2) + 1);
  da.slots = d_slots.p;
  da.slot_count = d_slot_count.p;
  da.slot_capacity = slot_capacity;
  da.n_watch = s.n_watch;
  for (int i = 0; i < s.n_watch; ++i) da.watch_key[i] = s.watch_key[i];
  da.group_size = cfg.group_size_bins;
  da.start_level = cfg.start_level;
  da.watch_max = s.watch_max.p;
  da.cand_flag = s.cand_flag.p;
  da.spec_out = M;
  da.spec_sum = ss ? ss->sum.p : nullptr;
  da.n_emit = n_emit;
  for (int i = 0; i < n_emit; ++i) {
    da.emit_frame[i] = emit_frames[i];
    da.emit_div[i] = emit_divs[i];
  }
  da.spec_rows = s.spec_rows.p;
  da.box_last = s.host_track ? nullptr : s.box_last.p;
  da.cta_ns = nullptr;
  if (profiling && profile_ctas) {
    if ((rc = s.cta_ns.alloc(2 * ((n + detect_bins - 1) / detect_bins)))) return rc;
    da.cta_ns = s.cta_ns.p;
  }
  da.dense_q = s.dense_q_on ? s.dense_q.p : nullptr;
  da.dense_avg = s.dense_avg_on ? s.dense_avg.p : nullptr;
  da.dense_box = s.dense_box_on ? s.dense_box.p : nullptr;
  {
    const int half = cfg.grouping_x / 2;
    const int hp = (half + 3) & ~3;
    const int width = detect_bins + 2 * hp;
    da.bins_per_cta = detect_bins;
    constexpr size_t kSmemBudget = 220 * 1024;
    const size_t fixed = sizeof(float) * (kAvgBuffers * width * (kDetectTileFrames + 1) + kBoxGroups * kDetectBinsPerCta * kDetectTileFrames);
    const size_t per_tile = sizeof(float) * kDetectTileFrames * width;
    da.n_buffers = static_cast<int>(std::min<size_t>(kDetectBuffers, (kSmemBudget - fixed) / per_tile));
    const size_t smem = fixed + per_tile * da.n_buffers;
    const int grid = (n + detect_bins - 1) / detect_bins;
    if ((rc = prepare_kernel(engine, k_detect<21, 10, 152>, kDetectThreads, 220 * 1024, nullptr))) return rc;
    if ((rc = prepare_kernel(engine, k_detect<21, 10, 136>, kDetectThreads, 220 * 1024, nullptr))) return rc;
    if ((rc = prepare_kernel(engine, k_detect<21, 10, 56>, kDetectThreads, 220 * 1024, nullptr))) return rc;
    if ((rc = prepare_kernel(engine, k_detect<21, 10>, kDetectThreads, 220 * 1024, nullptr))) return rc;
    if ((rc = prepare_kernel(engine, k_detect<0, -1>, kDetectThreads, 220 * 1024, nullptr))) return rc;
    if (profiling) CU(cudaEventRecord(s.ev[2], stream));
    if (half == 10 && Y == 21 && width == 152) {
      k_detect<21, 10, 152><<<grid, kDetectThreads, smem, stream>>>(da, s.psd_map);  // N >= 16384 on 132 SMs: 128 bins + 2 x 12 halo columns
    } else if (half == 10 && Y == 21 && width == 136) {
      k_detect<21, 10, 136><<<grid, kDetectThreads, smem, stream>>>(da, s.psd_map);  // N = 8192: 112 bins + 2 x 12 halo columns
    } else if (half == 10 && Y == 21 && width == 56) {
      k_detect<21, 10, 56><<<grid, kDetectThreads, smem, stream>>>(da, s.psd_map);   // N = 4096: 32 bins + 2 x 12
    } else if (half == 10 && Y == 21) {
      k_detect<21, 10><<<grid, kDetectThreads, smem, stream>>>(da, s.psd_map);
    } else {
      k_detect<0, -1><<<grid, kDetectThreads, smem, stream>>>(da, s.psd_map);
    }
    CU(cudaGetLastError());
    // order the per-frame slot lists by bin into one dense array
    k_entries_prefix<<<1, 1024, 0, stream>>>(d_slot_count.p, slot_capacity, T, s.offsets.p, s.max_count.p);
    CU(cudaGetLastError());
    RunFold fold{};
    TrackParams tp{};
    if (!s.host_track) {  // K4 works on runs of the ordered entries
      tp = track_params();
      fold.stop_level = tp.stop_level;
      fold.start_level = tp.start_level;
      fold.bin_lo = tp.bin_lo;
      fold.bin_hi = tp.bin_hi;
      fold.n_ignored = tp.n_ignored;
      for (int i = 0; i < tp.n_ignored; ++i) {
        fold.ignored_lo[i] = tp.ignored_lo[i];
        fold.ignored_hi[i] = tp.ignored_hi[i];
      }
      fold.lo = s.run_lo.p;
      fold.hi = s.run_hi.p;
      fold.count = s.run_count.p;
    }
    k_entries_sort<<<(T * 32 + 255) / 256, 256, 0, stream>>>(d_slots.p, d_slot_count.p, slot_capacity, T, s.offsets.p, s.sorted.p, fold);
    CU(cudaGetLastError());
    if (profiling) CU(cudaEventRecord(s.ev[3], stream));
  }
  if (!s.host_track) {
    // ---- K4 on its own stream: the signal map advances on the device while `stream` is free for the next push's K1 ----
    CU(cudaEventRecord(s.sorted_done, stream));
    CU(cudaStreamWaitEvent(track_stream, s.sorted_done, 0));
    TrackArgs ta{};
    ta.p = track_params();
    ta.run_lo = s.run_lo.p;
    ta.run_hi = s.run_hi.p;
    ta.run_count = s.run_count.p;
    ta.n_frames = T;
    ta.t0_ms = t0_ms;
    ta.period_ms = period_ms;
    ta.frame_offset = static_cast<long long>(frame_offset);
    ta.entries = s.sorted.p;
    ta.offsets = s.offsets.p;
    ta.max_count = s.max_count.p;
    ta.box_last = s.box_last.p;
    ta.psd = s.psd.p;
    ta.threshold = da.threshold_out;
    ta.noise_samples = da.noise_samples;
    ta.learn_frames = da.learn_frames;
    ta.ring_before = d_ring[ring_in].p;
    ta.state = track_map();
    ta.result = s.d_result.p;
    ta.tx = s.d_tx.p;
    ta.hit = d_track_hit.p;
    ta.sort_keys = d_track_sort.p;
    ta.log = s.log_on || s.log_starts ? s.d_log.p : nullptr;
    ta.log_cap = n;
    // k_track runs the push unless it would pass its shared tables; then it leaves the map untouched and sets the result's
    // hand-off flag, and k_track_wide, always enqueued behind it, runs the push from the same map. Otherwise k_track_wide exits.
    const bool len14 = run_len_bits(cfg.fft_size) == 14;
    auto* track = len14 ? k_track<14> : k_track<12>;
    auto* wide = len14 ? k_track_wide<14> : k_track_wide<12>;
    if ((rc = prepare_kernel(engine, track, kTrackThreads, sizeof(TrackShared), nullptr))) return rc;
    if ((rc = prepare_kernel(engine, wide, kTrackThreads, sizeof(TrackWideShared), nullptr))) return rc;
    if (profiling) {
      for (auto& e : s.tev) {
        if (!e) CU(cudaEventCreate(&e.h));
      }
      CU(cudaEventRecord(s.tev[0], track_stream));
    }
    track<<<1, kTrackThreads, sizeof(TrackShared), track_stream>>>(ta);
    CU(cudaGetLastError());
    wide<<<1, kTrackThreads, sizeof(TrackWideShared), track_stream>>>(ta);
    CU(cudaGetLastError());
    if (profiling) CU(cudaEventRecord(s.tev[1], track_stream));
    // the result header and the first B2S_MAX_TX transmissions (the rest, if any, is fetched by the finish half)
    CU(cudaMemcpyAsync(s.h_result.p, s.d_result.p, sizeof(TrackResult), cudaMemcpyDeviceToHost, track_stream));
    CU(cudaEventRecord(s.gpu_done, track_stream));
    prof.track_launches += 1;
  } else {
    CU(cudaEventRecord(s.gpu_done, stream));
  }

  // ---- occupancy: behind the list ordering on `stream`, after the events K4 and the finish half wait for, so neither waits for it.
  // The slot's PSD rows are next written by the K1 of the push after next, which `stream` runs after these kernels. ----
  if (s.occ) {
    OccupancySlot& o = *s.occ;
    const int learning = std::min(T, std::max(0, da.learn_frames - da.noise_samples));  // frames t with noise_samples + t < learn_frames
    o.frames += T;
    o.detect_frames += T - learning;
    if (T > learning) {
      const long long bound = static_cast<long long>(T) * slot_capacity;
      const int grid = static_cast<int>(std::max(1LL, std::min<long long>((bound + 255) / 256, 8LL * engine->sm_count)));
      k_occupancy_count<<<grid, 256, 0, stream>>>(s.sorted.p, s.offsets.p, T, cfg.start_level, cfg.stop_level, o.above_start.p, o.above_stop.p);
      CU(cudaGetLastError());
    }
    // more row groups per CTA while N / 32 CTAs would leave threads idle (up to 128 x 8 threads, 16 KB of shared memory)
    const int ctas = n / kOccupancyBins;
    int groups = 32;
    while (groups < 128 && static_cast<long long>(ctas) * groups * kOccupancyCols * 2 <= 2048LL * engine->sm_count) groups *= 2;
    const int threads = groups * kOccupancyCols;
    k_occupancy_max<<<ctas, threads, sizeof(float4) * threads, stream>>>(s.psd.p, n, T, o.max_db.p);
    CU(cudaGetLastError());
  }

  // context for the finish half
  s.T = T;
  s.t0_ms = t0_ms;
  s.period_ms = period_ms;
  s.frame_offset = frame_offset;
  s.noise_samples = da.noise_samples;
  s.learn_frames = da.learn_frames;
  s.avg_frames_before = avg_frames;
  s.ring_before = ring_in;
  s.threshold = da.threshold_out;  // the thresholds as of the end of this push
  s.center = center;
  s.n_emit = n_emit;
  s.out = out;
  s.thr_host_valid = false;
  // host mirrors of the scalar state advance at enqueue time (they do not depend on the results)
  if (!ns->ready) {
    ns->samples += learned_here;
    ns->ready = ready_after;
  }
  ns->cur ^= 1;
  sum_cur ^= 1;
  avg_frames = std::min(avg_frames + T, Y);
  ring_cur = ring_out;
  frames_pushed += T;
  prof.frames += T;
  prof.spectral_launches += 1;
  prof.detect_launches += 1;  // k_detect (+ the two small list-ordering kernels, timed with it)
  return 0;
}

// Result half: blocks on the slot's GPU work, then collects the results. Uses fstream() for its own transfers.
// Device-tracked chunks (the normal case) only read K4's result back; host-tracked chunks (the caller wants every frame's
// list) read the detection entries back and run tracker.h.
int b2s_band::finish_chunk(PushSlot& s) {
  cur = &s;
  cudaStream_t st = fstream();
  const int n = cfg.fft_size, T = s.T, M = cfg.spectrogram_out_size;
  int rc;
  b2s_result* out = s.out;
  int n_entries = 0;
  bool overflow = false;
  int worst_count = 0;
  if (!s.host_track) {
    CU(cudaEventSynchronize(s.gpu_done));  // K1, K2, ordering, K4 and the result copy
    if (st != stream) CU(cudaStreamWaitEvent(st, s.gpu_done, 0));
    const auto host_t0 = std::chrono::steady_clock::now();
    const TrackResult& r = *s.h_result.p;
    prof.d2h_bytes += sizeof(TrackResult);
    prof.track_launches += r.handoff;  // k_track_wide ran the push
    n_entries = r.n_entries;
    worst_count = r.max_count;
    prof.track_evals += r.n_evals;
    prof.track_events += r.n_events;
    prof.track_best_index += r.n_best;
    overflow = worst_count > slot_capacity;
    std::vector<b2s_transmission> list(r.n_tx);
    std::memcpy(list.data(), r.tx, sizeof(b2s_transmission) * std::min(r.n_tx, B2S_MAX_TX));
    if (r.n_tx > B2S_MAX_TX) {  // rare: the tail of a long list
      CU(cudaMemcpyAsync(list.data() + B2S_MAX_TX, s.d_tx.p + B2S_MAX_TX, sizeof(b2s_transmission) * (r.n_tx - B2S_MAX_TX), cudaMemcpyDeviceToHost, st));
      CU(cudaStreamSynchronize(st));
      prof.d2h_bytes += sizeof(b2s_transmission) * (r.n_tx - B2S_MAX_TX);
    }
    {
      std::lock_guard<std::mutex> lk(qmutex);
      if (s.epoch == reset_epoch) mailbox.swap(list);  // (a reset issued after this chunk was enqueued has emptied the mailbox: keep it so)
    }
    if ((s.log_on || s.log_starts) && r.n_log > 0) {  // the chunk's signal events: in-launch frames become frames of the band
      std::vector<TrackEvent> rec(std::min(r.n_log, n));
      CU(cudaMemcpyAsync(rec.data(), s.d_log.p, sizeof(TrackEvent) * rec.size(), cudaMemcpyDeviceToHost, st));
      CU(cudaStreamSynchronize(st));
      prof.d2h_bytes += sizeof(TrackEvent) * rec.size();
      std::lock_guard<std::mutex> lk(qmutex);
      if (s.log_on) {
        for (const TrackEvent& e : rec) events.push_back(b2s_signal_event{e.kind, e.key, e.shift_hz, 0, s.frame_base + e.frame, e.time, e.first, e.last});
        if (r.n_log > n) events.push_back(b2s_signal_event{B2S_EV_LOST, r.n_log - n, 0, 0, events.back().frame, events.back().time_ms, 0, 0});
      }
      if (s.log_starts) {
        for (const TrackEvent& e : rec)
          if (e.kind == B2S_EV_START) start_of[e.key] = {s.frame_base + e.frame, e.time};
        if (r.n_log > n) start_lost_through = s.frame_base + T - 1;  // a later START of any key may be among the lost
      }
    }
    if (profiling && s.tev[0]) {
      float ms = 0.0f;
      CU(cudaEventElapsedTime(&ms, s.tev[0], s.tev[1]));
      prof.track_ms += ms;
    }
    prof.tracker_host_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - host_t0).count();
  } else {
    if (st != stream) CU(cudaStreamWaitEvent(st, s.gpu_done, 0));
    int* h_off = s.h_offsets.p;
    int* h_max = s.h_offsets.p + max_frames + 1;
    CU(cudaMemcpyAsync(h_off, s.offsets.p, sizeof(int) * (T + 1), cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(h_max, s.max_count.p, sizeof(int), cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(s.h_cand_flag.p, s.cand_flag.p, sizeof(int) * T, cudaMemcpyDeviceToHost, st));
    if (s.n_watch > 0) CU(cudaMemcpyAsync(s.h_watch_max.p, s.watch_max.p, sizeof(unsigned int) * static_cast<size_t>(T) * kMaxWatch, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    n_entries = h_off[T];
    prof.d2h_bytes += sizeof(int) * (2 * T + 2) + (s.n_watch > 0 ? sizeof(unsigned int) * static_cast<size_t>(T) * kMaxWatch : 0);
    const auto host_t0 = std::chrono::steady_clock::now();
    worst_count = *h_max;
    overflow = worst_count > slot_capacity;  // the push completes on the truncated lists (device and host state stay in step); reported below
    if (n_entries > 0) {
      if ((rc = s.h_entries.alloc(n_entries))) return rc;
      CU(cudaMemcpyAsync(s.h_entries.p, s.sorted.p, sizeof(DetectEntry) * n_entries, cudaMemcpyDeviceToHost, st));
      CU(cudaStreamSynchronize(st));
      prof.d2h_bytes += sizeof(DetectEntry) * n_entries;
    }
    std::vector<Tracker::FrameState> states;
    tracker.p.center = s.center;
    Tracker::Watch watch{s.n_watch, s.watch_key, s.h_watch_max.p, s.h_cand_flag.p};
    std::vector<b2s_signal_event> logged;
    tracker.log = s.log_on || s.log_starts ? &logged : nullptr;
    tracker.log_frame_base = s.frame_base;
    rc = tracker.run(s.h_entries.p, h_off, T, s.t0_ms, s.period_ms, s.frame_offset, *this, true, watch, states);
    tracker.log = nullptr;
    if (rc) return rc;
    if (!logged.empty()) {
      std::lock_guard<std::mutex> lk(qmutex);
      if (s.log_on) events.insert(events.end(), logged.begin(), logged.end());
      if (s.log_starts) {
        for (const b2s_signal_event& e : logged)
          if (e.kind == B2S_EV_START) start_of[e.key] = {e.frame, e.time_ms};
      }
    }
    prof.tracker_host_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - host_t0).count();
    // the mailbox after the last frame of this chunk (Notification::notify, transmission.cpp:67)
    mailbox.clear();
    if (!states.empty() && states.back().frame == T - 1) {
      mailbox.resize(states.back().keys.size());
      tracker.sorted_transmissions(states.back(), mailbox.data(), static_cast<int>(mailbox.size()));
    }
    for (int t = 0; t < T; ++t) out->frame_tx_count[s.frame_offset + t] = 0;
    for (const auto& fs : states) {
      out->frame_tx_count[s.frame_offset + fs.frame] =
          tracker.sorted_transmissions(fs, out->frame_tx ? out->frame_tx + (s.frame_offset + fs.frame) * B2S_MAX_TX : nullptr, out->frame_tx ? B2S_MAX_TX : 0);
    }
    if ((rc = host_tracker_to_state())) return rc;  // the device copy of the map follows the host's
  }
  if (profiling && s.ev[0]) {
    float ms = 0.0f;
    CU(cudaEventElapsedTime(&ms, s.ev[0], s.ev[1]));
    prof.spectral_ms += ms;
    CU(cudaEventElapsedTime(&ms, s.ev[2], s.ev[3]));
    prof.detect_ms += ms;
    if (profile_ctas && s.cta_ns.p) {
      const int grid = (n + detect_bins - 1) / detect_bins;
      std::vector<unsigned long long> ns(2 * grid);
      CU(cudaMemcpyAsync(ns.data(), s.cta_ns.p, sizeof(unsigned long long) * ns.size(), cudaMemcpyDeviceToHost, st));
      CU(cudaStreamSynchronize(st));
      std::vector<double> dur(grid);
      for (int i = 0; i < grid; ++i) dur[i] = static_cast<double>(ns[2 * i + 1] - ns[2 * i]) * 1e-6;
      std::sort(dur.begin(), dur.end());
      prof.detect_cta_median_ms += dur[grid / 2];
      prof.detect_cta_max_ms += dur[grid - 1];
    }
  }
  if (overflow) wanted_capacity = std::max(wanted_capacity, 2 * worst_count);
  stat_entries += n_entries;
  stat_rows += s.n_emit;
  if (out) {
    out->n_detect_entries += n_entries;
    out->n_spectrogram_rows += s.n_emit;
    out->n_transmissions_total = static_cast<int32_t>(mailbox.size());
    out->n_transmissions = std::min<int32_t>(out->n_transmissions_total, B2S_MAX_TX);
    std::memcpy(out->transmissions, mailbox.data(), sizeof(b2s_transmission) * out->n_transmissions);
    if (out->peak_index) CU(cudaMemcpyAsync(out->peak_index + s.frame_offset, s.peak_idx.p, sizeof(int) * T, cudaMemcpyDeviceToHost, st));
    if (out->peak_value) CU(cudaMemcpyAsync(out->peak_value + s.frame_offset, s.peak_val.p, sizeof(float) * T, cudaMemcpyDeviceToHost, st));
    const size_t row_bytes = sizeof(float) * static_cast<size_t>(T) * n, off = s.frame_offset * n;
    if (out->psd_db) CU(cudaMemcpyAsync(out->psd_db + off, s.psd.p, row_bytes, cudaMemcpyDeviceToHost, st));
    if (out->noise_sub_db) CU(cudaMemcpyAsync(out->noise_sub_db + off, s.dense_q.p, row_bytes, cudaMemcpyDeviceToHost, st));
    if (out->avg_db) CU(cudaMemcpyAsync(out->avg_db + off, s.dense_avg.p, row_bytes, cudaMemcpyDeviceToHost, st));
    if (out->box_db) CU(cudaMemcpyAsync(out->box_db + off, s.dense_box.p, row_bytes, cudaMemcpyDeviceToHost, st));
  }
  if (s.n_emit > 0) {
    std::vector<int8_t> rows(static_cast<size_t>(s.n_emit) * M);
    CU(cudaMemcpyAsync(rows.data(), s.spec_rows.p, rows.size(), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    for (int i = 0; i < s.n_emit; ++i) {
      sent.push_back(SentRow{s.emit_time[i], s.center, std::vector<int8_t>(rows.begin() + static_cast<size_t>(i) * M, rows.begin() + static_cast<size_t>(i + 1) * M)});
    }
  }
  CU(cudaStreamSynchronize(st));
  cur = nullptr;
  if (overflow && s.occ) {  // the occupancy counts of this chunk came from the truncated lists
    std::lock_guard<std::mutex> lk(qmutex);
    s.occ->truncated += 1;
  }
  if (overflow)
    return fail(B2S_E_OVERFLOW, "a frame produced %d detection entries but detect_capacity is %d per frame: the frame's list was truncated (the push completed on the "
                "truncated lists); the capacity grows to %d before the next push", worst_count, slot_capacity, std::min(cfg.fft_size, wanted_capacity));
  return 0;
}
