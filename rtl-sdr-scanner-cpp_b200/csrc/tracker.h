// Host-side signal bookkeeping: the std::map<Index, Signal> logic of the reference's Transmission block
//   addSignals / getBestIndex        sources/radio/blocks/transmission.cpp:88-111,132-154
//   updateSignals / Signal::newData  sources/radio/blocks/transmission.cpp:113-130, sources/radio/signal.cpp:16-24
//   clearSignals / isTimeout ...     sources/radio/blocks/transmission.cpp:70-86, sources/radio/signal.cpp:26-32
//   getSortedTransmissions           sources/radio/blocks/transmission.cpp:166-176
// driven by the GPU's compact detection entries (every bin whose boxcar power reached min(start, stop)) instead of
// dense rows. It is O(#entries + #signals) per frame, time-based and ordered like std::map — host work by design
// (SURVEY.md §2 row 3). Two things it cannot derive from the entries are fetched from the device on demand through
// DeviceQueries: ring windows for getBestIndex (new signal) and window maxima of frames where the whole window sits
// below the detection level (only needed to order the output list).
//
// Tie rules the reference leaves to an unstable std::sort are fixed as: candidates by (power desc, index asc),
// transmissions by (power desc, key asc) — the oracle uses the same rules.
#pragma once
#include <cmath>
#include <cstdint>
#include <map>
#include <vector>

#include "../../include/b2s.h"
#include "detect.cuh"
#include "host_utils.h"

namespace b2s {

struct TrackerParams {
  int n = 0;
  int32_t sample_rate = 0;
  int32_t center = 0, range_lo = 0, range_hi = 0;
  int n_ignored = 0;
  int32_t ignored_lo[B2S_MAX_IGNORED] = {0}, ignored_hi[B2S_MAX_IGNORED] = {0};
  int group_size = 0;  // m_groupSize (bins)
  int group_y = 21;
  float start_level = 8.0f, stop_level = 5.0f;
  int32_t tuning_step = 2500;
  int64_t min_time = 2000, timeout = 2000, max_time = 600000;
};

struct TrackedSignal {
  int64_t first = 0, last = 0;  // Signal::m_firstDataTime / m_lastDataTime
  float power = 0.0f;           // Signal::m_power
  int watch = -1;               // slot of this key in the current chunk's watch list (refreshed by Tracker::run), -1 = none
};

// what the tracker may ask the device for (implemented by the band)
struct DeviceQueries {
  virtual ~DeviceQueries() {}
  // noise-subtracted rows for in-push frames [frame_first, frame_first + rows) (negative = before this push, i.e. the
  // Averager ring as it was when the push began), bins [bin_lo, bin_lo + width); out[rows][width]
  virtual int fetch_ring_window(int frame_first, int rows, int bin_lo, int width, float* out) = 0;
  // max / first-argmax of the boxcar row over [bin_lo, bin_hi] for each frame of [frame_lo, frame_hi)
  struct Window {
    int bin_lo, bin_hi, frame_lo, frame_hi;
  };
  virtual int query_windows(const std::vector<Window>& w, std::vector<std::vector<float>>& values, std::vector<std::vector<int>>& indices) = 0;
};

class Tracker {
 public:
  TrackerParams p;
  std::map<int, TrackedSignal> signals;  // transmission.h:49

  // The signal event log (b2s_signal_event): where run() inserts a key it appends a START, where it erases one a STOP, in that
  // order within a frame (Transmission::process, transmission.cpp:57-68). Frame t of a run is stamped log_frame_base + t.
  std::vector<b2s_signal_event>* log = nullptr;  // null = off
  int64_t log_frame_base = 0;

  void reset() { signals.clear(); }  // first half of Transmission::resetBuffers, transmission.cpp:42-55 (logs nothing, like the reference)

  // sdr_device.cpp:150,153-158
  double step() const { return static_cast<double>(p.sample_rate) / p.n; }
  int32_t index_to_shift(int i) const { return static_cast<int32_t>(step() * (i + 0.5)) - p.sample_rate / 2; }
  int32_t index_to_frequency(int i) const { return p.center + index_to_shift(i); }
  bool in_range(int i) const {
    const int32_t f = index_to_frequency(i);
    return p.range_lo <= f && f <= p.range_hi;
  }
  bool ignored(int i) const {  // transmission.cpp:156-164
    const int32_t f = index_to_frequency(i);
    for (int r = 0; r < p.n_ignored; ++r) {
      if (p.ignored_lo[r] <= f && f <= p.ignored_hi[r]) return true;
    }
    return false;
  }

  struct FrameState {  // the live signals after one frame, in map order
    int frame;
    int64_t now;
    std::vector<int> keys;
    std::vector<TrackedSignal> sig;
    std::vector<char> power_known;
  };

  // What K2 already reduced for the keys that were live when the chunk was enqueued (DetectArgs watch list):
  // max[t * kMaxWatch + i] = order-preserving image of max(boxcar row over key_i's window) in frame t (0 = nothing),
  // flag[t] != 0 when some bin >= start level lies outside every watched key's margin interval.
  struct Watch {
    int n = 0;
    const int* key = nullptr;
    const unsigned int* max = nullptr;
    const int* flag = nullptr;
  };

  // entries: the detection entries of the chunk ordered by (frame, bin); frame_begin[t]..frame_begin[t+1] index them.
  // Produces one FrameState per frame that ends with at least one live signal (only the last frame unless
  // need_every_frame). Frame t of this chunk is frame (frame_offset + t) of the caller's push and is stamped accordingly.
  int run(const DetectEntry* entries, const int* frame_begin, size_t n_frames, int64_t t0_ms, double period_ms, size_t frame_offset, DeviceQueries& dev,
          bool need_every_frame, const Watch& watch, std::vector<FrameState>& out) {
    out.clear();
    const int half_g = p.group_size / 2;
    // which watch slot (if any) covers a live key; how many watched keys are still alive. While ALL watched keys are
    // alive the current margins cover at least what K2 assumed, so flag[t] == 0 proves that addSignals cannot fire.
    auto watch_slot = [&](int key) {
      for (int i = 0; i < watch.n; ++i) {
        if (watch.key[i] == key) return i;
      }
      return -1;
    };
    int watched_alive = 0;
    for (auto& kv : signals) {
      kv.second.watch = watch_slot(kv.first);
      watched_alive += kv.second.watch >= 0 ? 1 : 0;
    }
    for (size_t t = 0; t < n_frames; ++t) {
      const int e0 = frame_begin[t], e1 = frame_begin[t + 1];
      const bool flags_valid = watch.flag != nullptr && watched_alive == watch.n;
      if (signals.empty() && (flags_valid ? watch.flag[t] == 0 : e0 == e1)) continue;
      const int64_t now = host::frame_time(t0_ms, period_ms, frame_offset + t);
      // ---- addSignals ----
      // A candidate only changes the map when no key lies within the margin; the power ordering of the candidates
      // (std::sort in the reference) matters only then, so the list is built and ordered lazily.
      bool any_new = false;
      if (!flags_valid || watch.flag[t] != 0) {
        for (int e = e0; e < e1 && !any_new; ++e) {
          const DetectEntry& d = entries[e];
          if (p.start_level <= d.value && !host::key_within_margin(signals, d.bin, p.group_size) && in_range(d.bin) && !ignored(d.bin)) any_new = true;
        }
      }
      if (any_new) {
        cand_.clear();
        for (int e = e0; e < e1; ++e) {
          const DetectEntry& d = entries[e];
          if (p.start_level <= d.value && in_range(d.bin) && !ignored(d.bin)) cand_.push_back(e);
        }
        std::stable_sort(cand_.begin(), cand_.end(), [&](int a, int b) { return entries[a].value > entries[b].value; });  // entries are bin-ascending
        for (int e : cand_) {
          const int idx = entries[e].bin;
          if (!host::key_within_margin(signals, idx, p.group_size)) {
            int key = idx;
            const int rc = best_index(idx, static_cast<int>(t), dev, &key);
            if (rc != 0) return rc;
            const int slot = watch_slot(key);
            if (signals.insert({key, TrackedSignal{now, now, 0.0f, slot}}).second) {
              if (slot >= 0) watched_alive++;
              log_event(B2S_EV_START, key, t, now, now, now);
            }
          }
        }
      }
      if (signals.empty()) continue;
      // ---- updateSignals: window maximum of the boxcar row around every key, then clearSignals ----
      for (auto it = signals.begin(); it != signals.end();) {
        TrackedSignal& s = it->second;
        const int ws = s.watch;
        const unsigned int image = (ws >= 0 && watch.max) ? watch.max[t * kMaxWatch + ws] : 0u;
        if (image != 0u) {
          const float best = ordered_to_float(image);  // exact window maximum, also below the detection level
          s.power = best;                              // Signal::newData: m_power = avgPower
          if (p.stop_level <= best) s.last = now;
        } else {
          const int lo = std::max(0, it->first - half_g), hi = std::min(p.n - 1, it->first + half_g);
          int a = e0, b = e1;
          while (a < b) {  // first entry of this frame with bin >= lo
            const int m = (a + b) / 2;
            if (entries[m].bin < lo) a = m + 1; else b = m;
          }
          bool found = false;
          float best = 0.0f;
          for (int e = a; e < e1 && entries[e].bin <= hi; ++e) {
            if (!found || entries[e].value > best) {
              best = entries[e].value;
              found = true;
            }
          }
          if (found) {
            s.power = best;
            if (p.stop_level <= best) s.last = now;
          } else {
            // every bin of the window is below min(start, stop): neither level test can pass; only m_power is unknown
            s.power = std::nanf("");
          }
        }
        if (s.last + p.timeout <= now || s.first + p.max_time <= now) {
          if (ws >= 0) watched_alive--;
          log_event(B2S_EV_STOP, it->first, t, now, s.first, s.last);
          it = signals.erase(it);
        } else {
          ++it;
        }
      }
      if (!signals.empty() && (need_every_frame || t + 1 == n_frames)) {
        out.emplace_back();
        FrameState& fs = out.back();
        fs.frame = static_cast<int>(t);
        fs.now = now;
        for (const auto& kv : signals) {
          fs.keys.push_back(kv.first);
          fs.sig.push_back(kv.second);
          fs.power_known.push_back(std::isnan(kv.second.power) ? 0 : 1);
        }
      }
    }
    return resolve_unknown_powers(dev, out);
  }

  // transmission.cpp:166-176 for one recorded frame
  int sorted_transmissions(const FrameState& fs, b2s_transmission* out, int cap) const {
    std::vector<int> order(fs.keys.size());
    for (size_t i = 0; i < order.size(); ++i) order[i] = static_cast<int>(i);
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return fs.sig[a].power > fs.sig[b].power; });  // keys ascend in map order
    int count = 0;
    for (int i : order) {
      if (count >= cap) break;
      const TrackedSignal& s = fs.sig[i];
      out[count].shift_hz = host::tuned_frequency(index_to_shift(fs.keys[i]), p.tuning_step);
      out[count].flush = ((s.last == fs.now) && (s.first + p.min_time <= fs.now)) ? 1 : 0;  // Signal::needFlush, signal.cpp:32
      out[count].key = fs.keys[i];
      out[count].power = s.power;
      ++count;
    }
    return static_cast<int>(fs.keys.size());
  }

 private:
  void log_event(int kind, int key, size_t t, int64_t now, int64_t first, int64_t last) {
    if (!log) return;
    log->push_back(b2s_signal_event{kind, key, host::tuned_frequency(index_to_shift(key), p.tuning_step), 0, log_frame_base + static_cast<int64_t>(t), now, first, last});
  }

  // getBestIndex, transmission.cpp:132-154: newest half of the ring rows, per row the first maximum around `index`
  int best_index(int index, int frame, DeviceQueries& dev, int* key) {
    const int total = p.group_y;
    const int rows = total - total / 2;  // rows [total/2, total)
    const int lo = std::max(0, index - p.group_size / 2), hi = std::min(p.n - 1, index + p.group_size / 2);
    const int width = hi - lo + 1;
    scratch_.resize(static_cast<size_t>(rows) * width);
    const int rc = dev.fetch_ring_window(frame - rows + 1, rows, lo, width, scratch_.data());
    if (rc != 0) return rc;
    std::vector<int> votes;
    for (int r = 0; r < rows; ++r) {
      const float* row = scratch_.data() + static_cast<size_t>(r) * width;
      int best = 0;
      for (int i = 1; i < width; ++i) {
        if (row[best] < row[i]) best = i;
      }
      if (p.start_level <= row[best]) votes.push_back(lo + best);
    }
    // the reference indexes an empty vector here (collection_utils.h:46-49); defined as "keep the candidate bin"
    *key = votes.empty() ? index : host::most_frequent(votes);
    return 0;
  }

  int resolve_unknown_powers(DeviceQueries& dev, std::vector<FrameState>& frames) {
    // group consecutive unknown frames per key into window queries
    struct Run {
      int key, frame_lo, frame_hi;
    };
    std::vector<Run> runs;
    std::map<int, size_t> open;  // key -> index into runs
    for (const FrameState& fs : frames) {
      for (size_t i = 0; i < fs.keys.size(); ++i) {
        if (fs.power_known[i]) continue;
        auto it = open.find(fs.keys[i]);
        if (it != open.end() && runs[it->second].frame_hi == fs.frame) {
          runs[it->second].frame_hi = fs.frame + 1;
        } else {
          open[fs.keys[i]] = runs.size();
          runs.push_back(Run{fs.keys[i], fs.frame, fs.frame + 1});
        }
      }
    }
    if (runs.empty()) return 0;
    std::vector<DeviceQueries::Window> w;
    for (const Run& r : runs) {
      w.push_back({std::max(0, r.key - p.group_size / 2), std::min(p.n - 1, r.key + p.group_size / 2), r.frame_lo, r.frame_hi});
    }
    std::vector<std::vector<float>> values;
    std::vector<std::vector<int>> indices;
    const int rc = dev.query_windows(w, values, indices);
    if (rc != 0) return rc;
    std::map<std::pair<int, int>, float> lut;  // (key, frame) -> power
    for (size_t q = 0; q < runs.size(); ++q) {
      for (int f = runs[q].frame_lo; f < runs[q].frame_hi; ++f) lut[{runs[q].key, f}] = values[q][f - runs[q].frame_lo];
    }
    for (FrameState& fs : frames) {
      for (size_t i = 0; i < fs.keys.size(); ++i) {
        if (!fs.power_known[i]) {
          fs.sig[i].power = lut[{fs.keys[i], fs.frame}];
          fs.power_known[i] = 1;
        }
      }
    }
    // the live map keeps the value of the last frame it was updated in
    if (!frames.empty()) {
      const FrameState& last = frames.back();
      for (size_t i = 0; i < last.keys.size(); ++i) {
        auto it = signals.find(last.keys[i]);
        if (it != signals.end() && std::isnan(it->second.power)) it->second.power = last.sig[i].power;
      }
    }
    return 0;
  }

  std::vector<float> scratch_;
  std::vector<int> cand_;
};

}  // namespace b2s
