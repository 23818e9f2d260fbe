// Scanner hop policy and recorder assignment (SURVEY.md §8(f)#3): the host logic that consumes the detection path's mailbox.
//   Scanner::worker                 reference sources/scanner.cpp:36-64      which range is scanned, and for how long
//   SdrDevice::updateRecordings     reference sources/radio/sdr_device.cpp:82-144   which Recorder follows which transmission
//   getRangeSplitSampleRate / splitRange(s)   reference sources/utils/radio_utils.cpp:162-199
// Plain state machines over the injected clock: one notification (the list the band's mailbox holds) in, the recorder actions and
// the hop decision out. The reference blocks inside Notification::wait(); here the caller owns the loop (b2s_band_push /
// b2s_band_sync produce the notifications), so the same decisions can be driven from any host loop or replayed in a test.
#pragma once
#include <algorithm>
#include <cstdint>
#include <limits>
#include <set>
#include <utility>
#include <vector>

#include "../../include/b2s.h"

namespace b2s {
namespace host {

inline int32_t round_down(int32_t v, int32_t m) { return v - v % m; }
// getRangeSplitSampleRate — radio_utils.cpp:162-172
inline int32_t range_split_sample_rate(int32_t fs) {
  if (10000000 <= fs) return round_down(fs, 1000000);
  if (1000000 <= fs) return round_down(fs, 500000);
  if (100000 <= fs) return round_down(fs, 100000);
  return fs;
}
// splitRange / splitRanges — radio_utils.cpp:174-199
inline void split_range(int32_t lo, int32_t hi, int32_t fs, std::vector<std::pair<int32_t, int32_t>>& out) {
  if (hi - lo <= fs) {
    out.emplace_back(lo, hi);
    return;
  }
  for (int64_t f = lo; f < hi; f += fs) out.emplace_back(static_cast<int32_t>(f), static_cast<int32_t>(f + fs));
}

class ScanPolicy {
 public:
  struct Recorder {  // Recorder::{m_shift, isRecording}, recorder.cpp:16-19,54-56
    bool recording = false;
    int32_t shift = std::numeric_limits<int32_t>::max();
    int64_t first = 0, last = 0;  // m_firstDataTime / m_lastDataTime
  };
  std::vector<std::pair<int32_t, int32_t>> ranges;  // Scanner::m_ranges
  std::vector<Recorder> recorders;
  std::set<int32_t> ignored;  // SdrDevice::ignoredTransmissions
  int64_t scanning_time = 500;  // RANGE_SCANNING_TIME, config.h:25
  size_t current = 0;
  int64_t start = 0;

  ScanPolicy(const int32_t* lo, const int32_t* hi, int n, int32_t sample_rate, int n_recorders, int64_t scanning_time_ms) : recorders(n_recorders), scanning_time(scanning_time_ms) {
    const int32_t split = range_split_sample_rate(sample_rate);  // Scanner::Scanner, scanner.cpp:10
    for (int i = 0; i < n; ++i) split_range(lo[i], hi[i], split, ranges);
  }

  // SdrDevice::updateRecordings (sdr_device.cpp:82-144) for one sorted list; appends the actions in the reference's order and, when
  // `source` is given, for each action the index of the list entry it acts on (-1 for a STOP: its shift left the list)
  void update_recordings(int64_t now, const b2s_transmission* list, int n, std::vector<b2s_recorder_action>& actions, std::vector<int>* source = nullptr) {
    auto waiting = [&](int32_t shift) {
      for (int i = 0; i < n; ++i) {
        if (list[i].shift_hz == shift) return true;
      }
      return false;
    };
    for (size_t r = 0; r < recorders.size(); ++r) {  // stop the recorders whose transmission left the list
      if (recorders[r].recording && !waiting(recorders[r].shift)) {
        actions.push_back({B2S_REC_STOP, static_cast<int32_t>(r), recorders[r].shift, recorders[r].last - recorders[r].first});
        if (source) source->push_back(-1);
        recorders[r] = Recorder{};
      }
    }
    for (int i = 0; i < n; ++i) {
      const int32_t shift = list[i].shift_hz;
      size_t r = 0;
      while (r < recorders.size() && recorders[r].shift != shift) ++r;
      if (r < recorders.size()) {
        if (list[i].flush) {  // Recorder::flush: publish what has been buffered
          recorders[r].last = now;
          actions.push_back({B2S_REC_FLUSH, static_cast<int32_t>(r), shift, 0});
          if (source) source->push_back(i);
        }
        continue;
      }
      size_t f = 0;
      while (f < recorders.size() && recorders[f].recording) ++f;
      if (f < recorders.size()) {  // Recorder::startRecording(getFrequency(), shift)
        recorders[f] = Recorder{true, shift, now, now};
        actions.push_back({B2S_REC_START, static_cast<int32_t>(f), shift, 0});
        if (source) source->push_back(i);
      } else if (!ignored.count(shift)) {
        ignored.insert(shift);
        actions.push_back({B2S_REC_NONE_FREE, -1, shift, 0});
        if (source) source->push_back(i);
      }
    }
    for (auto it = ignored.begin(); it != ignored.end();) {
      if (waiting(*it)) ++it; else it = ignored.erase(it);
    }
  }

  // Scanner::worker's inner loop for one notification: returns true when the scanner moves on to the next range
  // (the caller then retunes: b2s_band_set_center + b2s_band_reset, sdr_device.cpp:54-80)
  bool dwell_over(int64_t now, bool notification_empty) const {
    if (ranges.size() <= 1) return false;  // a single range is scanned forever (scanner.cpp:41-45)
    return !(now <= start + scanning_time || !notification_empty);
  }
  void hop(int64_t now) {
    current = (current + 1) % ranges.size();
    start = now;
  }
};

}  // namespace host
}  // namespace b2s
