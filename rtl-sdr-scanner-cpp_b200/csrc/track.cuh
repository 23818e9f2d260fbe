// K4 — the Transmission block's signal map on the device (one CTA per band and push).
//   addSignals / getBestIndex        reference sources/radio/blocks/transmission.cpp:88-111,132-154
//   updateSignals / Signal::newData  reference sources/radio/blocks/transmission.cpp:113-130, sources/radio/signal.cpp:16-24
//   clearSignals / isTimeout ...     reference sources/radio/blocks/transmission.cpp:70-86, sources/radio/signal.cpp:26-32
//   getSortedTransmissions           reference sources/radio/blocks/transmission.cpp:166-176
// The reference runs this per frame on the host; tracker.h does the same from K2's detection entries (and stays the path for
// callers that ask for every frame's list). Here the map lives in device memory across pushes and the host only reads the
// mailbox of the last frame, so a push costs the host one small device->host copy and no bookkeeping.
//
// The map only changes at EVENTS: a frame with a start-level bin that no live key covers (containsWithMargin), a time-out,
// or the 10-minute limit. Between events every frame is independent: a key's m_lastDataTime is the time of the latest frame
// whose window [key - g/2, key + g/2] holds a bin at or above the stop level. So the kernel walks the push in blocks of 1024
// frames, one thread per frame, finds the first event frame of the block in parallel, commits the frames before it in
// parallel, replays the event frame exactly like the reference (candidates by power, getBestIndex on the Averager ring rows,
// update, clear) and continues behind it. Each thread first folds its frame's detection entries into runs of consecutive bins
// (one per emitter and level), so the per-frame work does not grow with the width of a signal.
// The kernel is one CTA: K1 leaves one SM free for it (b2s_band keeps it off `stream`), so it runs beside the next push's K1.
//
// m_power (only read when the list is emitted) is taken for the last frame of the push from K2's boxcar row of that frame.
// Tie rules left open by the reference's unstable std::sort are the oracle's: candidates (power desc, bin asc), transmissions
// (power desc, key asc).
//
// The signal event log (b2s_signal_event; TrackArgs::log, null = off): where an event frame inserts a key the kernels append a
// START record, where clearSignals drops one a STOP record with the Signal's two times, in the order Transmission::process makes
// the changes: a frame's inserts first, then its erasures in ascending key. k_track appends from thread 0, which alone edits its
// map; k_track_wide from thread 0 at an insert, and in clearSignals from the thread that holds the erased key, at the key's rank
// among the erased, which is its index minus its rank among the kept that the compaction scan computes. The number of records
// is published in the epilogue with the rest of the result, so a k_track that hands off leaves no count behind: k_track_wide
// counts from 0 and writes over what k_track had appended.
#pragma once
#include "../../include/b2s.h"
#include "detect.cuh"

namespace b2s {

// k_track holds the map and one event frame's candidates in shared memory, up to these caps. A push that would pass either
// is left to k_track_wide, whose tables live in global memory and hold any input.
constexpr int kMaxSignals = 256;   // live signals
// k_track packs a run into 32 bits as (first bin << LEN_BITS) | (length - 1), and replays a frame with a longer run from its raw
// entries. The first bin takes the other 32 - LEN_BITS bits: LEN_BITS = 14 up to N = 2^18, 12 up to N = 2^20.
constexpr int run_len_bits(int n) { return n > (1 << 18) ? 12 : 14; }
constexpr int kTrackThreads = 1024, kTrackFrames = 1024, kTrackWords = kTrackFrames / 32;
constexpr int kMaxCand = 2048;     // start-level candidates replayed in one event frame
constexpr int kTrackSortChunk = 2 * kTrackThreads;  // k_track_wide's sort: keys per shared-memory pass

struct TrackParams {  // Transmission's construction-time parameters (transmission.h:17-25) + the index lambdas of sdr_device.cpp:153-158
  int n, sample_rate, center;
  // isIndexInRange / isIndexIgnored (sdr_device.cpp:155-158, transmission.cpp:156-164) as BIN intervals: indexToFrequency is
  // monotonic in the index, so each frequency interval is one interval of bins; the host finds the bounds with the reference's
  // own double-precision expression (FP64 is far too slow on this part to evaluate per detection entry)
  int bin_lo, bin_hi;  // bins whose frequency lies in [range_lo, range_hi]
  int n_ignored, ignored_lo[B2S_MAX_IGNORED], ignored_hi[B2S_MAX_IGNORED];  // bins (inclusive; lo > hi when empty)
  int group_size, group_y;
  float start_level, stop_level;
  int tuning_step;
  long long min_time, timeout, max_time;
};

// std::map<Index, Signal> (transmission.h:49) in device memory, keys ascending. Every key is a distinct bin, so arrays of N
// entries hold any map.
struct TrackMap {
  int* n;  // live signals
  int* key;
  long long *first, *last;
  float* power;
};

struct TrackEvent {  // one record of the signal event log
  int kind, key, shift_hz;  // B2S_EV_START / B2S_EV_STOP, the map key, b2s_transmission::shift_hz of the key
  int frame;                // in-launch frame index
  long long time, first, last;
};

struct TrackResult {  // what the host reads back per push
  int n_tx, n_entries, max_count;
  int handoff;  // k_track stopped before writing any state and left the push to k_track_wide (which keeps the flag set)
  long long last_now;
  int n_evals, n_events, n_best;  // work counters of the push: block evaluations, event frames replayed, getBestIndex calls
  int n_log;                      // records the push appended to TrackArgs::log, also past log_cap (written only when the log is on)
  b2s_transmission tx[B2S_MAX_TX];     // the first B2S_MAX_TX of TrackArgs::tx
};

struct TrackArgs {
  TrackParams p;
  int n_frames;
  long long t0_ms;
  double period_ms;
  long long frame_offset;
  const DetectEntry* entries;  // ordered by (frame, bin)
  const int* offsets;          // [T + 1]
  const int* max_count;        // largest per-frame entry count (overflow report)
  const int* run_lo;           // runs of the frames' entries, folded by k_entries_sort (RunFold layout)
  const int* run_hi;
  const int* run_count;
  const float* box_last;       // [N] boxcar row of the last frame
  // getBestIndex inputs: noise-subtracted rows = the Averager ring
  const float* psd;            // [T][N]
  const float* threshold;      // [N]
  int noise_samples, learn_frames;
  const float* ring_before;    // [Y][N] ring before the push, oldest -> newest
  TrackMap state;
  TrackResult* result;
  b2s_transmission* tx;            // [N] getSortedTransmissions after the last frame
  unsigned int* hit;               // k_track_wide: [N][kTrackWords] the keys' hit words of a block
  unsigned long long* sort_keys;   // k_track_wide: [N rounded up to a power of two] sort scratch
  TrackEvent* log;                 // [log_cap] the push's signal events in order, or null: no log. The count is TrackResult::n_log
  int log_cap;
};

__device__ __forceinline__ long long track_frame_time(long long t0, double period, long long k) {
  return t0 + static_cast<long long>(floor(__dadd_rn(__dmul_rn(static_cast<double>(k), period), 0.5)));  // host::frame_time
}
__device__ __forceinline__ int track_index_to_shift(const TrackParams& p, int i) {  // sdr_device.cpp:150,154
  const double step = __ddiv_rn(static_cast<double>(p.sample_rate), static_cast<double>(p.n));
  return static_cast<int>(__dmul_rn(step, __dadd_rn(static_cast<double>(i), 0.5))) - p.sample_rate / 2;
}
__device__ __forceinline__ bool track_candidate_bin(const TrackParams& p, int i) {  // isIndexInRange && !isIndexIgnored, transmission.cpp:91,156-164
  if (i < p.bin_lo || i > p.bin_hi) return false;
  for (int r = 0; r < p.n_ignored; ++r) {
    if (p.ignored_lo[r] <= i && i <= p.ignored_hi[r]) return false;
  }
  return true;
}
__device__ __forceinline__ int track_tuned(int f, int step) {  // getTunedFrequency, radio_utils.cpp:86-96
  int r = f % step;
  if (f < 0) r += step;
  const int below = f - r;
  return (r < step - r) ? below : below + step;
}
__device__ __forceinline__ int track_margin(int g) { return (g % 2 == 0) ? g / 2 : g / 2 + 1; }  // collection_utils.h:17-27

// first index with keys[i] >= v
__device__ __forceinline__ int track_lower_bound(const int* keys, int n, int v) {
  int a = 0, b = n;
  while (a < b) {
    const int m = (a + b) >> 1;
    if (keys[m] < v) a = m + 1; else b = m;
  }
  return a;
}
__device__ __forceinline__ bool track_within_margin(const int* keys, int n, int index, int margin) {
  const int i = track_lower_bound(keys, n, index - margin);
  return i < n && keys[i] <= index + margin;
}
// record `at` of the log; records past the capacity are counted, not stored
__device__ __forceinline__ void track_log(const TrackArgs& a, int at, int kind, int key, int frame, long long now, long long first, long long last) {
  if (at < a.log_cap) a.log[at] = TrackEvent{kind, key, track_tuned(track_index_to_shift(a.p, key), a.p.tuning_step), frame, now, first, last};
}
__device__ __forceinline__ void track_write_header(const TrackArgs& a, int n_tx, long long last_now, int handoff, int n_evals, int n_events, int n_best, int n_log) {
  TrackResult* r = a.result;
  r->n_tx = n_tx;
  r->n_entries = a.n_frames > 0 ? a.offsets[a.n_frames] : 0;
  r->max_count = a.max_count ? *a.max_count : 0;
  r->handoff = handoff;
  r->last_now = last_now;
  r->n_evals = n_evals;
  r->n_events = n_events;
  r->n_best = n_best;
  if (a.log) r->n_log = n_log;
}

// ------------------------------------------------------------------------------------------------------------
// k_track
// ------------------------------------------------------------------------------------------------------------
struct TrackShared {
  int n;                            // live signals
  int key[kMaxSignals];
  long long first[kMaxSignals], last[kMaxSignals];
  unsigned int hit[kMaxSignals][kTrackWords];  // bit f of word w: frame (block start + 32 w + f) has a stop-level bin in the key's window
  unsigned int evmask[kTrackWords];             // event frames of the block under the current key set
  unsigned int runs[2][kRunCap][kTrackFrames];  // per frame (thread): packed runs of [0] stop-level bins, [1] start-level candidates
  long long time[kTrackFrames];                 // frame clock of the block's frames
  int votes[128], tied[128];                    // getBestIndex scratch (thread 0)
  int changed, handoff, best_key;
  int n_log;                        // signal event records appended so far (thread 0)
  int row_idx[128];                 // getBestIndex: first maximum of each ring row (-1 = below the start level)
  // event-frame scratch (the output lists reuse it after the last frame)
  int n_cand, n_open;
  int cand_bin[kMaxCand];
  float cand_val[kMaxCand];
  int cand_order[kMaxCand];
  int open_rank[kMaxCand];          // ranks of the candidates no key covered when the frame began, ascending
  unsigned char open_flag[kMaxCand];
};

// getBestIndex (transmission.cpp:132-154) for candidate bin `index` at in-push frame `frame`, by the whole CTA: one warp per ring
// row finds the row's first maximum around the bin, thread 0 takes the mode of the rows that reach the start level.
template <class Shared>
__device__ void track_best_index(const TrackArgs& a, Shared& s, int index, int frame) {
  const TrackParams& p = a.p;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int total = p.group_y, rows = total - total / 2;  // rows [total/2, total) of the ring = the newest `rows` frames
  const int lo = max(0, index - p.group_size / 2), hi = min(p.n - 1, index + p.group_size / 2);
  for (int r = warp; r < rows; r += kTrackThreads / 32) {
    const int f = frame - rows + 1 + r;
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    for (int b = lo + lane; b <= hi; b += 32) {
      float v;
      if (f >= 0) {
        v = (a.noise_samples + f < a.learn_frames) ? kNoData : __fsub_rn(a.psd[static_cast<size_t>(f) * p.n + b], a.threshold[b]);
      } else if (total + f >= 0) {
        v = a.ring_before[static_cast<size_t>(total + f) * p.n + b];
      } else {
        v = 0.0f;
      }
      argmax_combine(bv, bi, v, b);  // first maximum: ties keep the lower bin (getMaxIndex, collection_utils.h:9-14)
    }
    warp_argmax(bv, bi);
    if (lane == 0) s.row_idx[r] = (p.start_level <= bv) ? bi : -1;
  }
  __syncthreads();
  if (tid == 0) {
    // mostFrequentValue (collection_utils.h:30-50): the mode; among equally frequent values the one at position size/2 of the
    // ascending tied set. No vote at all: the reference indexes an empty vector (collection_utils.h:46-49); defined as "keep the bin".
    int* votes = s.votes;
    int* tied = s.tied;
    int n_votes = 0;
    for (int r = 0; r < rows; ++r) {
      if (s.row_idx[r] >= 0) votes[n_votes++] = s.row_idx[r];
    }
    int result = index;
    if (n_votes > 0) {
      for (int i = 1; i < n_votes; ++i) {  // insertion sort, ascending
        const int v = votes[i];
        int j = i - 1;
        while (j >= 0 && votes[j] > v) {
          votes[j + 1] = votes[j];
          --j;
        }
        votes[j + 1] = v;
      }
      int best = 0, n_tied = 0;
      for (int i = 0; i < n_votes;) {
        int j = i;
        while (j < n_votes && votes[j] == votes[i]) ++j;
        if (j - i > best) {
          best = j - i;
          n_tied = 0;
        }
        if (j - i == best) tied[n_tied++] = votes[i];
        i = j;
      }
      result = tied[n_tied / 2];
    }
    s.best_key = result;
  }
  __syncthreads();
}

template <int LEN_BITS>
__global__ void __launch_bounds__(kTrackThreads, 1) k_track(const TrackArgs a) {
  static_assert(LEN_BITS == 12 || LEN_BITS == 14, "run_len_bits");
  constexpr int kRunLenBits = LEN_BITS;
  extern __shared__ __align__(16) unsigned char track_smem[];
  TrackShared& s = *reinterpret_cast<TrackShared*>(track_smem);
  const TrackParams& p = a.p;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int T = a.n_frames;
  const int gh = p.group_size / 2, margin = track_margin(p.group_size);
  int n_evals = 0, n_events = 0, n_best = 0;  // (thread 0's copies are reported)

  // ---- load the map; a map larger than the shared tables is k_track_wide's ----
  if (tid == 0) {
    s.n = *a.state.n;
    s.n_log = 0;
    s.handoff = s.n > kMaxSignals ? 1 : 0;
    if (s.handoff) a.result->handoff = 1;
  }
  __syncthreads();
  if (s.handoff) return;
  for (int i = tid; i < s.n; i += kTrackThreads) {
    s.key[i] = a.state.key[i];
    s.first[i] = a.state.first[i];
    s.last[i] = a.state.last[i];
  }
  __syncthreads();

  for (int bs = 0; bs < T; bs += kTrackFrames) {  // blocks of 1024 frames, one thread per frame
    const int be = min(T, bs + kTrackFrames);
    const int t = bs + tid;
    const bool in_block = t < be;
    // My frame's runs (consecutive bins at or above the stop level / start-level candidates, folded by k_entries_sort), packed
    // into shared memory for every evaluation of this block; s.time holds the frames' clock (FP64 is slow here: once per frame)
    int n_stop = 0, n_start = 0;
    s.time[tid] = track_frame_time(a.t0_ms, a.period_ms, a.frame_offset + t);
    bool long_run = false;
    if (in_block) {
      n_stop = a.run_count[t];
      n_start = a.run_count[T + t];
#pragma unroll
      for (int L = 0; L < 2; ++L) {
        const int cnt = min(L == 0 ? n_stop : n_start, kRunCap);
#pragma unroll
        for (int r = 0; r < kRunCap; ++r) {
          if (r < cnt) {
            const int lo = a.run_lo[static_cast<size_t>(L * kRunCap + r) * T + t], hi = a.run_hi[static_cast<size_t>(L * kRunCap + r) * T + t];
            long_run = long_run || hi - lo >= (1 << kRunLenBits);
            s.runs[L][r][tid] = (static_cast<unsigned>(lo) << kRunLenBits) | static_cast<unsigned>(min(hi - lo, (1 << kRunLenBits) - 1));
          }
        }
      }
    }
    if (long_run) n_stop = kRunCap + 1;  // a stretch too long to pack: replay the frame from its raw entries
    const long long now = s.time[tid];
    const bool complex_frame = n_stop > kRunCap || n_start > kRunCap;  // replayed from its raw entries
    __syncthreads();
    int ts = bs;  // first frame of the block not yet applied (uniform)
    while (ts < be) {
      // ================= evaluation: events of the frames [ts, be) under the current key set =================
      ++n_evals;
      const bool mine = in_block && t >= ts;
      const int K = s.n;
      bool event = mine && complex_frame;
      if (mine && !event) {
        // addSignals can fire when a candidate bin lies outside every key's margin interval (containsWithMargin)
        for (int r = 0; r < n_start && !event; ++r) {
          const unsigned run = s.runs[1][r][tid];
          int pos = static_cast<int>(run >> kRunLenBits);
          const int end = pos + static_cast<int>(run & ((1u << kRunLenBits) - 1u));
          int i = track_lower_bound(s.key, K, pos - margin);
          while (pos <= end) {
            if (i >= K || s.key[i] - margin > pos) {
              event = true;
              break;
            }
            pos = s.key[i] + margin + 1;
            ++i;
          }
        }
      }
      for (int q = 0; q < K; ++q) {  // hit bits of every key
        const int lo = max(0, s.key[q] - gh), hi = min(p.n - 1, s.key[q] + gh);
        bool h = false;
        if (mine) {
          for (int r = 0; r < min(n_stop, kRunCap); ++r) {
            const unsigned run = s.runs[0][r][tid];
            const int rl = static_cast<int>(run >> kRunLenBits);
            h = h || (rl <= hi && rl + static_cast<int>(run & ((1u << kRunLenBits) - 1u)) >= lo);
          }
        }
        const unsigned m = __ballot_sync(0xffffffffu, h);
        if (lane == 0) s.hit[q][warp] = m;
      }
      __syncthreads();
      if (mine && !event) {
        for (int q = 0; q < K; ++q) {
          // time of the key's latest hit at or before my frame (Signal::newData sets m_lastDataTime = now on such frames)
          long long last = s.last[q];
          unsigned m = s.hit[q][warp] & (0xffffffffu >> (31 - lane));
          int w = warp;
          while (m == 0u && w > 0) m = s.hit[q][--w];
          if (m != 0u) last = s.time[32 * w + (31 - __clz(m))];
          if (last + p.timeout <= now || s.first[q] + p.max_time <= now) {  // isTimeout / isMaximalTime, signal.cpp:28-30
            event = true;
            break;
          }
        }
      }
      {
        const unsigned m = __ballot_sync(0xffffffffu, event);
        if (lane == 0) s.evmask[warp] = m;
      }
      if (tid == 0) s.changed = 0;
      __syncthreads();
      // ================= walk the event frames in order until one of them changes the key set =================
      int cur = ts;
      while (true) {
        int te = be;  // next event frame at or after cur
        {
          int w = (cur - bs) >> 5;
          unsigned m = w < kTrackWords ? (s.evmask[w] & (0xffffffffu << ((cur - bs) & 31))) : 0u;
          while (m == 0u && ++w < kTrackWords) m = s.evmask[w];
          if (m != 0u) te = min(be, bs + 32 * w + (__ffs(m) - 1));
        }
        // commit the steady frames [cur, te): every key's m_lastDataTime = its newest hit among them
        if (tid < K && te > cur) {
          const int last_f = te - 1 - bs;
          int w = last_f >> 5;
          unsigned m = s.hit[tid][w] & (0xffffffffu >> (31 - (last_f & 31)));
          const int w_min = (cur - bs) >> 5;
          while (m == 0u && w > w_min) m = s.hit[tid][--w];
          if (w == w_min) m &= 0xffffffffu << ((cur - bs) & 31);
          if (m != 0u) s.last[tid] = s.time[32 * w + (31 - __clz(m))];
        }
        __syncthreads();
        if (te >= be) {
          ts = be;
          break;
        }
        // ---- the event frame te, exactly as Transmission::process orders it (transmission.cpp:57-68) ----
        ++n_events;
        const long long ev_now = s.time[te - bs];
        const int e0 = a.offsets[te], e1 = a.offsets[te + 1];
        if (tid == 0) {
          s.n_cand = 0;
          s.n_open = 0;
        }
        __syncthreads();
        // addSignals: candidates = start-level bins in range and not ignored, strongest first (transmission.cpp:88-96)
        for (int e = e0 + tid; e < e1; e += kTrackThreads) {
          const DetectEntry d = a.entries[e];
          if (p.start_level <= d.value && track_candidate_bin(p, d.bin)) {
            const int i = atomicAdd(&s.n_cand, 1);
            if (i < kMaxCand) {
              s.cand_bin[i] = d.bin;
              s.cand_val[i] = d.value;
            }
          }
        }
        __syncthreads();
        if (s.n_cand > kMaxCand) {  // before any state is written: k_track_wide runs the push from the same map
          if (tid == 0) a.result->handoff = 1;
          return;
        }
        const int nc = s.n_cand;
        for (int i = tid; i < nc; i += kTrackThreads) {  // rank sort: (value desc, bin asc); bins are distinct
          const float v = s.cand_val[i];
          const int b = s.cand_bin[i];
          int rank = 0;
          for (int k = 0; k < nc; ++k) rank += (s.cand_val[k] > v || (s.cand_val[k] == v && s.cand_bin[k] < b)) ? 1 : 0;
          s.cand_order[rank] = i;
        }
        __syncthreads();
        // candidates that no key covers right now (containsWithMargin, transmission.cpp:99), in rank order
        for (int r = tid; r < nc; r += kTrackThreads) s.open_flag[r] = track_within_margin(s.key, s.n, s.cand_bin[s.cand_order[r]], margin) ? 0 : 1;
        __syncthreads();
        if (tid == 0) {
          int m = 0;
          for (int r = 0; r < nc; ++r) {
            if (s.open_flag[r]) s.open_rank[m++] = r;
          }
          s.n_open = m;
        }
        __syncthreads();
        const int n_open = s.n_open;
        for (int u = 0; u < n_open; ++u) {
          const int idx = s.cand_bin[s.cand_order[s.open_rank[u]]];
          if (track_within_margin(s.key, s.n, idx, margin)) continue;  // a key inserted for a stronger candidate covers it now (uniform)
          ++n_best;
          track_best_index(a, s, idx, te);
          if (tid == 0) {
            const int key = s.best_key;
            const int pos = track_lower_bound(s.key, s.n, key);
            if (!(pos < s.n && s.key[pos] == key)) {  // std::map::insert keeps an existing element
              if (s.n >= kMaxSignals) {
                s.handoff = 1;
              } else {
                for (int i = s.n; i > pos; --i) {
                  s.key[i] = s.key[i - 1];
                  s.first[i] = s.first[i - 1];
                  s.last[i] = s.last[i - 1];
                }
                s.key[pos] = key;
                s.first[pos] = ev_now;  // Signal(now): m_firstDataTime = m_lastDataTime = now (signal.cpp:6-14)
                s.last[pos] = ev_now;
                s.n += 1;
                s.changed = 1;
                if (a.log) track_log(a, s.n_log++, B2S_EV_START, key, te, ev_now, ev_now, ev_now);
              }
            }
          }
          __syncthreads();
          if (s.handoff) {
            if (tid == 0) a.result->handoff = 1;
            return;
          }
        }
        // updateSignals: a stop-level bin inside the key's window refreshes m_lastDataTime (transmission.cpp:113-130, signal.cpp:16-24)
        for (int i = tid; i < s.n; i += kTrackThreads) {
          const int lo = max(0, s.key[i] - gh), hi = min(p.n - 1, s.key[i] + gh);
          int x = e0, y = e1;
          while (x < y) {  // first entry of the frame with bin >= lo
            const int m = (x + y) >> 1;
            if (a.entries[m].bin < lo) x = m + 1; else y = m;
          }
          bool h = false;
          for (int e = x; e < e1 && a.entries[e].bin <= hi; ++e) h = h || (p.stop_level <= a.entries[e].value);
          if (h) s.last[i] = ev_now;
        }
        __syncthreads();
        // clearSignals (transmission.cpp:70-86)
        if (tid == 0) {
          int w = 0;
          for (int i = 0; i < s.n; ++i) {
            if (s.last[i] + p.timeout <= ev_now || s.first[i] + p.max_time <= ev_now) {
              s.changed = 1;
              if (a.log) track_log(a, s.n_log++, B2S_EV_STOP, s.key[i], te, ev_now, s.first[i], s.last[i]);
              continue;
            }
            s.key[w] = s.key[i];
            s.first[w] = s.first[i];
            s.last[w] = s.last[i];
            ++w;
          }
          s.n = w;
        }
        __syncthreads();
        cur = te + 1;
        if (s.changed) {  // the hit words and the predicted events belong to the old key set: evaluate again from here
          ts = cur;
          break;
        }
        if (cur >= be) {
          ts = be;
          break;
        }
      }
      __syncthreads();
    }
  }

  // ---- after the last frame: m_power, getSortedTransmissions, state back to global memory ----
  const int K = s.n;
  float* tx_power = s.cand_val;  // (the event scratch is free now)
  int* tx_order = s.cand_order;
  const long long last_now = T > 0 ? track_frame_time(a.t0_ms, a.period_ms, a.frame_offset + T - 1) : 0;
  for (int i = tid; i < K; i += kTrackThreads) {
    const int lo = max(0, s.key[i] - gh), hi = min(p.n - 1, s.key[i] + gh);
    float pw = a.box_last[lo];
    for (int b = lo + 1; b <= hi; ++b) pw = fmaxf(pw, a.box_last[b]);  // getMaxIndex(avgPower, ...): the window maximum
    tx_power[i] = pw;
  }
  __syncthreads();
  for (int i = tid; i < K; i += kTrackThreads) {  // power descending, equal powers by ascending key
    const float v = tx_power[i];
    int rank = 0;
    for (int k = 0; k < K; ++k) rank += (tx_power[k] > v || (tx_power[k] == v && k < i)) ? 1 : 0;
    tx_order[rank] = i;
  }
  __syncthreads();
  for (int r = tid; r < K; r += kTrackThreads) {
    const int i = tx_order[r];
    b2s_transmission tx;
    tx.shift_hz = track_tuned(track_index_to_shift(p, s.key[i]), p.tuning_step);
    tx.flush = (s.last[i] == last_now && s.first[i] + p.min_time <= last_now) ? 1 : 0;  // Signal::needFlush, signal.cpp:26,32
    tx.key = s.key[i];
    tx.power = tx_power[i];
    a.tx[r] = tx;
    if (r < B2S_MAX_TX) a.result->tx[r] = tx;
    a.state.key[i] = s.key[i];
    a.state.first[i] = s.first[i];
    a.state.last[i] = s.last[i];
    a.state.power[i] = tx_power[i];
  }
  if (tid == 0) {
    *a.state.n = K;
    track_write_header(a, K, last_now, 0, n_evals, n_events, n_best, s.n_log);
  }
}

// ------------------------------------------------------------------------------------------------------------
// k_track_wide: k_track with its tables in global memory, for the pushes k_track hands off
// ------------------------------------------------------------------------------------------------------------
// The map is edited in place in TrackArgs::state, the hit words live in TrackArgs::hit and the sort keys in
// TrackArgs::sort_keys, each sized for N entries, so no input overflows them. The frames' runs and clock stay in shared memory
// (they are per frame, not per key). The event walk, the tie rules and the counters are k_track's; what does not scale is
// CTA-wide here: the candidate order is a bitonic sort, the key insertion a parallel shift, clearSignals a scan and compaction.
struct TrackWideShared {
  int n;                                        // live signals
  unsigned int evmask[kTrackWords];
  unsigned int runs[2][kRunCap][kTrackFrames];
  long long time[kTrackFrames];
  int votes[128], tied[128];                    // getBestIndex scratch (thread 0)
  int changed, best_key;
  int n_log;                                    // signal event records appended so far
  int row_idx[128];
  int n_open;
  int warp_sum[kTrackThreads / 32];
  unsigned long long sort[kTrackSortChunk];
};

// Ascending order of the key = (v descending, id ascending), the order of k_track's rank sorts; -0 and +0 compare equal there.
__device__ __forceinline__ unsigned long long track_sort_key(float v, int id) {
  unsigned u = __float_as_uint(v == 0.0f ? 0.0f : v);
  u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);  // ascending in v
  return (static_cast<unsigned long long>(~u) << 32) | static_cast<unsigned>(id);
}

// one compare-exchange step of a bitonic sort over x[0, 2 * pairs); `base` is x's offset in the whole sequence
__device__ __forceinline__ void track_bitonic_step(unsigned long long* x, int base, int pairs, int k, int j) {
  for (int p = threadIdx.x; p < pairs; p += kTrackThreads) {
    const int i = 2 * (p & ~(j - 1)) + (p & (j - 1));
    const unsigned long long u = x[i], v = x[i + j];
    if ((u > v) == (((base + i) & k) == 0)) {
      x[i] = v;
      x[i + j] = u;
    }
  }
}

// Sorts g[0, n) ascending, by the whole CTA. g has room for n rounded up to a power of two; the padding sorts last. Steps whose
// pairs lie within kTrackSortChunk keys run on a shared-memory copy of that chunk. O(n log^2 n) work.
__device__ void track_sort(unsigned long long* g, int n, unsigned long long* sh) {
  if (n <= 1) return;
  int P = 2;
  while (P < n) P <<= 1;
  const int tid = threadIdx.x;
  for (int i = n + tid; i < P; i += kTrackThreads) g[i] = ~0ull;
  __syncthreads();
  const int C = min(P, kTrackSortChunk);
  for (int c0 = 0; c0 < P; c0 += C) {  // merges of up to C keys: each chunk in shared memory
    for (int i = tid; i < C; i += kTrackThreads) sh[i] = g[c0 + i];
    __syncthreads();
    for (int k = 2; k <= C; k <<= 1) {
      for (int j = k >> 1; j > 0; j >>= 1) {
        track_bitonic_step(sh, c0, C / 2, k, j);
        __syncthreads();
      }
    }
    for (int i = tid; i < C; i += kTrackThreads) g[c0 + i] = sh[i];
    __syncthreads();
  }
  for (int k = 2 * C; k <= P; k <<= 1) {  // larger merges: the steps across chunks in global memory, the rest per chunk
    for (int j = k >> 1; j >= C; j >>= 1) {
      track_bitonic_step(g, 0, P / 2, k, j);
      __syncthreads();
    }
    for (int c0 = 0; c0 < P; c0 += C) {
      for (int i = tid; i < C; i += kTrackThreads) sh[i] = g[c0 + i];
      __syncthreads();
      for (int j = C >> 1; j > 0; j >>= 1) {
        track_bitonic_step(sh, c0, C / 2, k, j);
        __syncthreads();
      }
      for (int i = tid; i < C; i += kTrackThreads) g[c0 + i] = sh[i];
      __syncthreads();
    }
  }
}

// Exclusive prefix of `flag` over the CTA; *total = the number of set flags. Ends with the flags of every warp in `warp_sum`:
// the caller synchronises before the next call.
__device__ __forceinline__ int track_block_scan(bool flag, int* warp_sum, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned b = __ballot_sync(0xffffffffu, flag);
  if (lane == 0) warp_sum[warp] = __popc(b);
  __syncthreads();
  int before = 0, all = 0;
  for (int w = 0; w < kTrackThreads / 32; ++w) {
    const int c = warp_sum[w];
    before += w < warp ? c : 0;
    all += c;
  }
  *total = all;
  return before + __popc(b & ((1u << lane) - 1u));
}

template <int LEN_BITS>
__global__ void __launch_bounds__(kTrackThreads, 1) k_track_wide(const TrackArgs a) {
  static_assert(LEN_BITS == 12 || LEN_BITS == 14, "run_len_bits");
  if (!a.result->handoff) return;  // k_track ran this push
  constexpr int kRunLenBits = LEN_BITS;
  extern __shared__ __align__(16) unsigned char track_smem[];
  TrackWideShared& s = *reinterpret_cast<TrackWideShared*>(track_smem);
  const TrackParams& p = a.p;
  int* const key = a.state.key;
  long long* const first = a.state.first;
  long long* const last = a.state.last;
  unsigned int* const hit = a.hit;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int T = a.n_frames;
  const int gh = p.group_size / 2, margin = track_margin(p.group_size);
  int n_evals = 0, n_events = 0, n_best = 0;

  if (tid == 0) {
    s.n = *a.state.n;
    s.n_log = 0;
  }
  __syncthreads();

  for (int bs = 0; bs < T; bs += kTrackFrames) {  // k_track's block walk
    const int be = min(T, bs + kTrackFrames);
    const int t = bs + tid;
    const bool in_block = t < be;
    int n_stop = 0, n_start = 0;
    s.time[tid] = track_frame_time(a.t0_ms, a.period_ms, a.frame_offset + t);
    bool long_run = false;
    if (in_block) {
      n_stop = a.run_count[t];
      n_start = a.run_count[T + t];
#pragma unroll
      for (int L = 0; L < 2; ++L) {
        const int cnt = min(L == 0 ? n_stop : n_start, kRunCap);
#pragma unroll
        for (int r = 0; r < kRunCap; ++r) {
          if (r < cnt) {
            const int lo = a.run_lo[static_cast<size_t>(L * kRunCap + r) * T + t], hi = a.run_hi[static_cast<size_t>(L * kRunCap + r) * T + t];
            long_run = long_run || hi - lo >= (1 << kRunLenBits);
            s.runs[L][r][tid] = (static_cast<unsigned>(lo) << kRunLenBits) | static_cast<unsigned>(min(hi - lo, (1 << kRunLenBits) - 1));
          }
        }
      }
    }
    if (long_run) n_stop = kRunCap + 1;
    const long long now = s.time[tid];
    const bool complex_frame = n_stop > kRunCap || n_start > kRunCap;
    __syncthreads();
    int ts = bs;
    while (ts < be) {
      // ================= evaluation =================
      ++n_evals;
      const bool mine = in_block && t >= ts;
      const int K = s.n;
      bool event = mine && complex_frame;
      if (mine && !event) {
        for (int r = 0; r < n_start && !event; ++r) {
          const unsigned run = s.runs[1][r][tid];
          int pos = static_cast<int>(run >> kRunLenBits);
          const int end = pos + static_cast<int>(run & ((1u << kRunLenBits) - 1u));
          int i = track_lower_bound(key, K, pos - margin);
          while (pos <= end) {
            if (i >= K || key[i] - margin > pos) {
              event = true;
              break;
            }
            pos = key[i] + margin + 1;
            ++i;
          }
        }
      }
      for (int q = 0; q < K; ++q) {
        const int lo = max(0, key[q] - gh), hi = min(p.n - 1, key[q] + gh);
        bool h = false;
        if (mine) {
          for (int r = 0; r < min(n_stop, kRunCap); ++r) {
            const unsigned run = s.runs[0][r][tid];
            const int rl = static_cast<int>(run >> kRunLenBits);
            h = h || (rl <= hi && rl + static_cast<int>(run & ((1u << kRunLenBits) - 1u)) >= lo);
          }
        }
        const unsigned m = __ballot_sync(0xffffffffu, h);
        if (lane == 0) hit[static_cast<size_t>(q) * kTrackWords + warp] = m;
      }
      __syncthreads();
      if (mine && !event) {
        for (int q = 0; q < K; ++q) {
          const unsigned int* hq = hit + static_cast<size_t>(q) * kTrackWords;
          long long lt = last[q];
          unsigned m = hq[warp] & (0xffffffffu >> (31 - lane));
          int w = warp;
          while (m == 0u && w > 0) m = hq[--w];
          if (m != 0u) lt = s.time[32 * w + (31 - __clz(m))];
          if (lt + p.timeout <= now || first[q] + p.max_time <= now) {
            event = true;
            break;
          }
        }
      }
      {
        const unsigned m = __ballot_sync(0xffffffffu, event);
        if (lane == 0) s.evmask[warp] = m;
      }
      if (tid == 0) s.changed = 0;
      __syncthreads();
      // ================= the event frames in order =================
      int cur = ts;
      while (true) {
        int te = be;
        {
          int w = (cur - bs) >> 5;
          unsigned m = w < kTrackWords ? (s.evmask[w] & (0xffffffffu << ((cur - bs) & 31))) : 0u;
          while (m == 0u && ++w < kTrackWords) m = s.evmask[w];
          if (m != 0u) te = min(be, bs + 32 * w + (__ffs(m) - 1));
        }
        if (te > cur) {
          const int last_f = te - 1 - bs, w_min = (cur - bs) >> 5;
          for (int q = tid; q < K; q += kTrackThreads) {
            const unsigned int* hq = hit + static_cast<size_t>(q) * kTrackWords;
            int w = last_f >> 5;
            unsigned m = hq[w] & (0xffffffffu >> (31 - (last_f & 31)));
            while (m == 0u && w > w_min) m = hq[--w];
            if (w == w_min) m &= 0xffffffffu << ((cur - bs) & 31);
            if (m != 0u) last[q] = s.time[32 * w + (31 - __clz(m))];
          }
        }
        __syncthreads();
        if (te >= be) {
          ts = be;
          break;
        }
        // ---- the event frame te (transmission.cpp:57-68) ----
        ++n_events;
        const long long ev_now = s.time[te - bs];
        const int e0 = a.offsets[te], e1 = a.offsets[te + 1];
        if (tid == 0) s.n_open = 0;
        __syncthreads();
        // addSignals: only the candidates no key covers when the frame begins can add a key (containsWithMargin,
        // transmission.cpp:99); sorting them alone gives them the order they hold among all candidates
        for (int e = e0 + tid; e < e1; e += kTrackThreads) {
          const DetectEntry d = a.entries[e];
          if (p.start_level <= d.value && track_candidate_bin(p, d.bin) && !track_within_margin(key, s.n, d.bin, margin)) {
            a.sort_keys[atomicAdd(&s.n_open, 1)] = track_sort_key(d.value, d.bin);
          }
        }
        __syncthreads();
        const int n_open = s.n_open;
        track_sort(a.sort_keys, n_open, s.sort);  // (value desc, bin asc)
        for (int u = 0; u < n_open; ++u) {
          const int idx = static_cast<int>(static_cast<unsigned>(a.sort_keys[u]));
          if (track_within_margin(key, s.n, idx, margin)) continue;  // uniform
          ++n_best;
          track_best_index(a, s, idx, te);
          const int nk = s.n, bk = s.best_key;
          const int pos = track_lower_bound(key, nk, bk);
          const bool insert = !(pos < nk && key[pos] == bk);  // std::map::insert keeps an existing element
          __syncthreads();
          if (insert) {
            for (int top = nk; top > pos; top -= kTrackThreads) {  // [pos, nk) up by one, from the top down
              const int i = top - 1 - tid;
              int k = 0;
              long long f = 0, l = 0;
              if (i >= pos) {
                k = key[i];
                f = first[i];
                l = last[i];
              }
              __syncthreads();
              if (i >= pos) {
                key[i + 1] = k;
                first[i + 1] = f;
                last[i + 1] = l;
              }
              __syncthreads();
            }
            if (tid == 0) {
              key[pos] = bk;
              first[pos] = ev_now;  // Signal(now)
              last[pos] = ev_now;
              s.n = nk + 1;
              s.changed = 1;
              if (a.log) track_log(a, s.n_log++, B2S_EV_START, bk, te, ev_now, ev_now, ev_now);
            }
          }
          __syncthreads();
        }
        // updateSignals
        for (int i = tid; i < s.n; i += kTrackThreads) {
          const int lo = max(0, key[i] - gh), hi = min(p.n - 1, key[i] + gh);
          int x = e0, y = e1;
          while (x < y) {
            const int m = (x + y) >> 1;
            if (a.entries[m].bin < lo) x = m + 1; else y = m;
          }
          bool h = false;
          for (int e = x; e < e1 && a.entries[e].bin <= hi; ++e) h = h || (p.stop_level <= a.entries[e].value);
          if (h) last[i] = ev_now;
        }
        __syncthreads();
        // clearSignals: a stable compaction in place, 1024 keys at a time (a kept key only moves down, past keys already read).
        // Key i is the (i - at)-th erased one when `at` kept keys precede it: its place among the frame's STOP records.
        {
          const int nk = s.n, log_base = s.n_log;
          int w = 0;
          for (int c = 0; c < nk; c += kTrackThreads) {
            const int i = c + tid;
            int k = 0;
            long long f = 0, l = 0;
            bool keep = false;
            if (i < nk) {
              k = key[i];
              f = first[i];
              l = last[i];
              keep = !(l + p.timeout <= ev_now || f + p.max_time <= ev_now);
            }
            int total;
            const int at = w + track_block_scan(keep, s.warp_sum, &total);
            if (keep) {
              key[at] = k;
              first[at] = f;
              last[at] = l;
            } else if (a.log && i < nk) {
              track_log(a, log_base + i - at, B2S_EV_STOP, k, te, ev_now, f, l);
            }
            w += total;
            __syncthreads();
          }
          if (tid == 0 && w != nk) {
            s.n = w;
            s.changed = 1;
            s.n_log = log_base + nk - w;
          }
        }
        __syncthreads();
        cur = te + 1;
        if (s.changed) {
          ts = cur;
          break;
        }
        if (cur >= be) {
          ts = be;
          break;
        }
      }
      __syncthreads();
    }
  }

  // ---- after the last frame: m_power, getSortedTransmissions ----
  const int K = s.n;
  const long long last_now = T > 0 ? track_frame_time(a.t0_ms, a.period_ms, a.frame_offset + T - 1) : 0;
  for (int i = tid; i < K; i += kTrackThreads) {
    const int lo = max(0, key[i] - gh), hi = min(p.n - 1, key[i] + gh);
    float pw = a.box_last[lo];
    for (int b = lo + 1; b <= hi; ++b) pw = fmaxf(pw, a.box_last[b]);
    a.state.power[i] = pw;
    a.sort_keys[i] = track_sort_key(pw, i);
  }
  __syncthreads();
  track_sort(a.sort_keys, K, s.sort);  // power descending, equal powers by ascending key
  for (int r = tid; r < K; r += kTrackThreads) {
    const int i = static_cast<int>(static_cast<unsigned>(a.sort_keys[r]));
    b2s_transmission tx;
    tx.shift_hz = track_tuned(track_index_to_shift(p, key[i]), p.tuning_step);
    tx.flush = (last[i] == last_now && first[i] + p.min_time <= last_now) ? 1 : 0;
    tx.key = key[i];
    tx.power = a.state.power[i];
    a.tx[r] = tx;
    if (r < B2S_MAX_TX) a.result->tx[r] = tx;
  }
  if (tid == 0) {
    *a.state.n = K;
    track_write_header(a, K, last_now, 1, n_evals, n_events, n_best, s.n_log);
  }
}

}  // namespace b2s
