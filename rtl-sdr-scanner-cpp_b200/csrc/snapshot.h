// Snapshots of a band or a recorder bank (b2s_*_save_state / b2s_*_load_state): the whole format, described in DESIGN.md §3.
// Included by b2s_api.cu after its helpers (fail, CU) and includes.
//   header   u32 magic "B2ST", u32 version, u32 kind, u64 total length
//   sections u32 tag, u64 payload length, payload; in a fixed order per kind, the config block first
//   trailer  u64 FNV-1a of every byte before it
// Every value is written field by field in the host's (little-endian) byte order, so a snapshot holds no padding.
// The sections of each kind are described once, by a function templated on the direction (band_sections, bank_sections). A save runs
// it with a Writer, which copies every device array straight into the snapshot. A load runs it with a Reader, which reads and checks
// every field and leaves every array where it lies in the snapshot, for the owner to upload once the whole snapshot is checked.
#pragma once

static_assert(__BYTE_ORDER__ == __ORDER_LITTLE_ENDIAN__, "snapshots are defined as little-endian");

namespace snapshot {

constexpr uint32_t kMagic = 0x54533242u;  // "B2ST"
constexpr uint32_t kVersion = 1;
constexpr uint32_t kBand = 1, kBank = 2;
constexpr size_t kHeader = 20;

constexpr uint32_t tag(const char (&s)[5]) {
  return static_cast<uint32_t>(s[0]) | static_cast<uint32_t>(s[1]) << 8 | static_cast<uint32_t>(s[2]) << 16 | static_cast<uint32_t>(s[3]) << 24;
}

inline uint64_t fnv1a64(const uint8_t* p, size_t n) {
  uint64_t h = 0xcbf29ce484222325ull;
  for (size_t i = 0; i < n; ++i) h = (h ^ p[i]) * 0x100000001b3ull;
  return h;
}

// ---- the three directions ----
struct Writer {
  static constexpr bool kLoad = false;
  cudaStream_t stream = nullptr;  // device arrays are copied on it
  int rc = 0;                     // the first failed device copy; the copies after it are skipped
  std::vector<uint8_t> out;
  size_t section_at = 0;
  template <typename T>
  void operator()(const T& v) {
    static_assert(std::is_arithmetic<T>::value, "fields are written one by one");
    bytes(&v, sizeof(T));
  }
  void flag(bool v) { (*this)(static_cast<uint8_t>(v)); }
  void bytes(const void* p, size_t n) { out.insert(out.end(), static_cast<const uint8_t*>(p), static_cast<const uint8_t*>(p) + n); }
  void bytes(const std::vector<int8_t>& v, size_t n) { bytes(v.data(), n); }
  void array(const void* dev, size_t n) {
    out.resize(out.size() + n);
    if (!rc) rc = download(out.data() + out.size() - n, dev, n);
  }
  int download(void* dst, const void* src, size_t n) {
    CU(cudaMemcpyAsync(dst, src, n, cudaMemcpyDeviceToHost, stream));
    CU(cudaStreamSynchronize(stream));  // `dst` lies in `out`, which the next field may move
    return 0;
  }
  void open(const char (&t)[5], const char*) {
    (*this)(tag(t));
    section_at = out.size();
    (*this)(uint64_t{0});
  }
  void close(const char*) {
    const uint64_t len = out.size() - section_at - sizeof(uint64_t);
    std::memcpy(out.data() + section_at, &len, sizeof(len));
  }
  void check(bool, const char*) {}
  bool fits(uint64_t, size_t) { return true; }
};

// Bounds-checked reads. A read past the current section reads zeros and, like a bool byte above 1, makes the next check refuse: it
// throws the reason, which `read` returns as B2S_E_INVALID.
struct Reader {
  static constexpr bool kLoad = true;
  const uint8_t* p = nullptr;
  size_t end = 0, at = 0, section_end = 0;
  bool bad = false;
  const uint8_t* span(size_t n) {
    bad = bad || n > section_end - at;
    if (bad) return nullptr;
    at += n;
    return p + at - n;
  }
  template <typename T>
  void operator()(T& v) {
    static_assert(std::is_arithmetic<T>::value, "fields are read one by one");
    v = T{};
    if (const uint8_t* s = span(sizeof(T))) std::memcpy(&v, s, sizeof(T));
  }
  void flag(bool& v) {
    uint8_t b;
    (*this)(b);
    bad = bad || b > 1;
    v = b != 0;
  }
  void bytes(const void*& s, size_t n) { s = span(n); }
  void bytes(std::vector<int8_t>& v, size_t n) {
    if (const int8_t* s = reinterpret_cast<const int8_t*>(span(n))) v.assign(s, s + n);
  }
  void array(const void*& s, size_t n) { s = span(n); }
  // the next section, which must have this tag and lie within the snapshot
  void open(const char (&t)[5], const char* why) {
    section_end = end;
    uint32_t got;
    uint64_t len;
    (*this)(got), (*this)(len);
    check(got == tag(t) && len <= end - at, why);
    section_end = at + len;
  }
  // the section was read to its last byte
  void close(const char* why) { check(at == section_end, why); }
  // refuses with `why` unless `cond` holds and every read since the last check was good
  void check(bool cond, const char* why) {
    if (bad || !cond) throw why;
  }
  // `count` items of `item` bytes fit in the rest of the section
  bool fits(uint64_t count, size_t item) { return count <= (section_end - at) / item; }
};

// the bytes a description writes: measures a list item, so that a load checks a count before the count sizes an allocation
struct Counter {
  static constexpr bool kLoad = false;
  size_t n = 0;
  template <typename T>
  void operator()(const T&) { n += sizeof(T); }
  void flag(bool) { n += 1; }
  template <class S>
  void bytes(const S&, size_t k) { n += k; }
  void array(const void*, size_t k) { n += k; }
};
template <class F>
size_t measure(F&& describe) {
  Counter c;
  describe(c);
  return c.n;
}

// A count of type Count, then that many items. A load refuses (`why`) a count above `most`, or one whose items cannot fit in the rest
// of the section, before the count sizes the list (a save's count is the list's size).
template <class Count, class IO, class List, class Item>
void list(IO& io, List& v, const char* why, Item&& item, uint64_t most = UINT64_MAX) {
  Count n = static_cast<Count>(v.size());
  io(n);
  io.check(n <= most && io.fits(n, measure([&](Counter& c) { typename List::value_type x{}; item(c, x); })), why);
  v.resize(n);
  for (auto& x : v) item(io, x);
}

// a save: the header, the sections that `describe(w)` writes, the trailer
template <class F>
int write(uint32_t kind, cudaStream_t stream, std::vector<uint8_t>& out, F&& describe) {
  Writer w;
  w.stream = stream;
  w(kMagic), w(kVersion), w(kind), w(uint64_t{0});  // the total length is filled in last
  describe(w);
  if (w.rc) return w.rc;
  const uint64_t total = w.out.size() + sizeof(uint64_t);
  std::memcpy(w.out.data() + kHeader - sizeof(total), &total, sizeof(total));
  w(fnv1a64(w.out.data(), w.out.size()));
  out.swap(w.out);
  return 0;
}

// a load: the header and the checksum, then `describe(r)` reads and checks every section; nothing may follow the last
template <class F>
int read(const void* buf, size_t len, uint32_t kind, const char* who, F&& describe) {
  if (len < kHeader + sizeof(uint64_t)) return fail(B2S_E_INVALID, "%s: %zu bytes are too short for a snapshot", who, len);
  Reader r;
  r.p = static_cast<const uint8_t*>(buf);
  r.end = r.section_end = len;
  uint32_t magic, version, k;
  uint64_t total, sum;
  r(magic), r(version), r(k), r(total);
  r.at = len - sizeof(uint64_t);
  r(sum);
  if (magic != kMagic) return fail(B2S_E_INVALID, "%s: not a b2s snapshot (magic %08x)", who, magic);
  if (version != kVersion) return fail(B2S_E_INVALID, "%s: snapshot format version %u, this library reads version %u", who, version, kVersion);
  if (k != kind) return fail(B2S_E_INVALID, "%s: the snapshot is of a %s, not of a %s", who, k == kBand ? "band" : k == kBank ? "recorder bank" : "unknown kind",
                             kind == kBand ? "band" : "recorder bank");
  if (total != len) return fail(B2S_E_INVALID, "%s: the snapshot is %llu bytes long, %zu were given", who, static_cast<unsigned long long>(total), len);
  if (fnv1a64(r.p, len - sizeof(uint64_t)) != sum) return fail(B2S_E_INVALID, "%s: checksum mismatch (the snapshot is damaged)", who);
  r.end = r.section_end = len - sizeof(uint64_t);
  r.at = kHeader;
  try {
    describe(r);
    r.check(r.at == r.end, "unexpected bytes after the last section");
  } catch (const char* why) {
    return fail(B2S_E_INVALID, "%s: %s", who, why);
  }
  return 0;
}

// ---- band: CONF SCAL NOIS SPEC AVGR SMAP MBOX EVNT ROWS, and LEAD with B2S_FLAG_SUBFRAME_OVERLAP ----
// every field of b2s_band_config except the window_taps pointer, in declaration order
template <typename F>
void band_config_fields(b2s_band_config& c, F&& f) {
  f(c.fft_size), f(c.sample_rate_hz), f(c.frame_stride_samples), f(c.iq_format), f(c.iq_scale), f(c.window_kind), f(c.grouping_x), f(c.grouping_y);
  f(c.group_size_bins), f(c.start_level), f(c.stop_level), f(c.learn_frames), f(c.center_hz), f(c.range_lo_hz), f(c.range_hi_hz), f(c.n_ignored);
  for (auto& v : c.ignored_lo_hz) f(v);
  for (auto& v : c.ignored_hi_hz) f(v);
  f(c.tuning_step_hz), f(c.min_time_ms), f(c.timeout_ms), f(c.max_time_ms), f(c.spectrogram_out_size), f(c.spectrogram_interval_ms), f(c.flags);
  f(c.max_frames_per_push), f(c.detect_capacity), f(c.noise_learning_ms);
}
// Two creation configs that a snapshot may move between: equal bit for bit except the centre and range (state), the flags other
// than the sub-frame bits (the learned noise depends on those, and the overlap bit on whether the snapshot holds a lead-in) and the
// sizing fields.
inline bool same_band_config(b2s_band_config a, b2s_band_config b) {
  Writer x, y;
  for (auto* c : {&a, &b}) {
    c->center_hz = c->range_lo_hz = c->range_hi_hz = c->max_frames_per_push = c->detect_capacity = 0;
    c->flags &= kSubframeFlags | B2S_FLAG_SUBFRAME_OVERLAP;
    c->window_taps = nullptr;
  }
  band_config_fields(a, x);
  band_config_fields(b, y);
  return x.out == y.out;
}

// The state of a band that a snapshot holds, but for the lists it keeps on the host. Each pointer is the array in device memory for a
// save, and its place in the snapshot after a load.
struct NoiseImage {
  int32_t center = 0, samples = 0;
  bool ready = false, started = false;
  int64_t start_ms = 0;
  const void* thr = nullptr;  // [N]
};
struct SpectroImage {
  int32_t center = 0, counter = 0;
  int64_t last_send = 0;
  const void* sum = nullptr;  // [M]
};
struct BandImage {
  int32_t center = 0, range_lo = 0, range_hi = 0;
  int64_t frames_pushed = 0;
  bool event_log = false;
  int32_t stat_entries = 0, stat_rows = 0, capacity = 0;
  std::vector<NoiseImage> noise;      // by ascending centre
  std::vector<SpectroImage> spectro;  // by ascending centre
  int32_t avg_frames = 0;
  const void *avg_sum = nullptr, *avg_last = nullptr, *ring = nullptr;  // [N], [N], [Y][N] oldest row first
  int32_t live = 0;  // the signal map: its live entries, then their keys, first, last and power
  const void *key = nullptr, *first = nullptr, *last = nullptr, *power = nullptr;
  bool has_lead = false;  // B2S_FLAG_SUBFRAME_OVERLAP: whether the next push's frame 0 has a lead-in, and its N / 2 samples
  const void* lead = nullptr;
};

template <class IO>
void map_arrays(IO& io, BandImage& m) {
  const size_t live = std::max(m.live, 0);
  io.array(m.key, sizeof(int32_t) * live), io.array(m.first, sizeof(int64_t) * live), io.array(m.last, sizeof(int64_t) * live);
  io.array(m.power, sizeof(float) * live);
}

// A band's snapshot. `own` and `own_taps` are the band's creation config and B2S_WINDOW_USER taps, which a load requires the snapshot
// to match; `rows` are the band's SentRows (time, centre, M bytes).
template <class IO, class Rows>
void band_sections(IO& io, BandImage& s, std::vector<b2s_transmission>& mailbox, std::deque<b2s_signal_event>& events, Rows& rows,
                   const b2s_band_config& own, const float* own_taps) {
  const int n = own.fft_size, Y = own.grouping_y;
  const size_t M = std::max(own.spectrogram_out_size, 0), taps_bytes = own.window_kind == B2S_WINDOW_USER ? sizeof(float) * n : 0;

  io.open("CONF", "the config block is missing or truncated");
  b2s_band_config c = own;
  band_config_fields(c, io);
  io.check(true, "the config block is truncated");
  if (IO::kLoad)
    io.check(same_band_config(c, own), "the snapshot was made with another configuration (every field but center_hz, range_lo_hz, range_hi_hz, the "
                                       "flags other than B2S_FLAG_SUBFRAME_*, max_frames_per_push and detect_capacity must match)");
  const void* taps = own_taps;
  io.bytes(taps, taps_bytes);
  io.check(true, "the config block is truncated");
  if (IO::kLoad) io.check(taps_bytes == 0 || std::memcmp(taps, own_taps, taps_bytes) == 0, "the snapshot was made with other user window taps");
  io.close("the config block has the wrong length");

  io.open("SCAL", "the scalar section is missing or truncated");
  io(s.center), io(s.range_lo), io(s.range_hi), io(s.frames_pushed), io.flag(s.event_log), io(s.stat_entries), io(s.stat_rows), io(s.capacity);
  io.close("the scalar section is malformed");
  io.check(s.frames_pushed >= 0 && s.stat_entries >= 0 && s.stat_rows >= 0 && s.capacity >= 1 && s.capacity <= n, "the scalar section is malformed");

  io.open("NOIS", "the noise section is missing or truncated");
  list<uint32_t>(io, s.noise, "the noise section is truncated", [&](auto& io, NoiseImage& x) {
    io(x.center), io(x.samples), io.flag(x.ready), io.flag(x.started), io(x.start_ms), io.array(x.thr, sizeof(float) * n);
  });
  for (size_t i = 0; i < s.noise.size(); ++i)
    io.check(s.noise[i].samples >= 0 && (i == 0 || s.noise[i].center > s.noise[i - 1].center), "the noise section is malformed");
  io.close("the noise section has the wrong length");

  io.open("SPEC", "the spectrogram section is missing or truncated");
  list<uint32_t>(
      io, s.spectro, "the spectrogram section is malformed",
      [&](auto& io, SpectroImage& x) { io(x.center), io(x.counter), io(x.last_send), io.array(x.sum, sizeof(float) * M); }, M > 0 ? UINT64_MAX : 0);
  for (size_t i = 0; i < s.spectro.size(); ++i)
    io.check(s.spectro[i].counter >= 0 && (i == 0 || s.spectro[i].center > s.spectro[i - 1].center), "the spectrogram section is malformed");
  io.close("the spectrogram section has the wrong length");

  io.open("AVGR", "the Averager section is missing or truncated");
  io(s.avg_frames), io.array(s.avg_sum, sizeof(float) * n), io.array(s.avg_last, sizeof(float) * n), io.array(s.ring, sizeof(float) * n * Y);
  io.close("the Averager section is malformed");
  io.check(s.avg_frames >= 0 && s.avg_frames <= Y, "the Averager section is malformed");

  io.open("SMAP", "the signal map section is missing or truncated");
  io(s.live);
  BandImage one;
  one.live = 1;
  io.check(s.live >= 0 && s.live <= n && io.fits(s.live, measure([&](Counter& c) { map_arrays(c, one); })), "the signal map section is malformed");
  map_arrays(io, s);
  io.close("the signal map section has the wrong length");
  for (int32_t i = 0, key, prev = -1; IO::kLoad && i < s.live; ++i, prev = key) {
    std::memcpy(&key, static_cast<const uint8_t*>(s.key) + sizeof(key) * i, sizeof(key));
    io.check(key > prev && key < n, "the signal map's keys are not strictly ascending bins");
  }

  io.open("MBOX", "the mailbox section is missing or truncated");
  list<uint32_t>(
      io, mailbox, "the mailbox section is malformed", [](auto& io, b2s_transmission& t) { io(t.shift_hz), io(t.flush), io(t.key), io(t.power); }, n);
  io.close("the mailbox section has the wrong length");

  io.open("EVNT", "the event section is missing or truncated");
  list<uint64_t>(io, events, "the event section is truncated", [](auto& io, b2s_signal_event& e) {
    io(e.kind), io(e.key), io(e.shift_hz), io(e.reserved), io(e.frame), io(e.time_ms), io(e.first_ms), io(e.last_ms);
  });
  io.close("the event section has the wrong length");

  io.open("ROWS", "the spectrogram row section is missing or truncated");
  list<uint64_t>(
      io, rows, "the spectrogram row section is malformed", [&](auto& io, auto& r) { io(r.time), io(r.center), io.bytes(r.row, M); }, M > 0 ? UINT64_MAX : 0);
  io.close("the spectrogram row section has the wrong length");

  // only a band with overlapping sub-frames has this section; a load has checked that the snapshot's overlap bit is the band's
  if (own.flags & B2S_FLAG_SUBFRAME_OVERLAP) {
    io.open("LEAD", "the lead-in section is missing or truncated");
    io.flag(s.has_lead), io.array(s.lead, static_cast<size_t>(n / 2) * (own.iq_format == B2S_IQ_CS8 ? 2 : 8));
    io.close("the lead-in section has the wrong length");
  }
}

// ---- recorder bank: CONF RAWC, then one CHAN per channel ----
// A bank's config and sizes, which a load requires the snapshot to match, and its device arrays: each pointer is in device memory
// for a save, and its place in the snapshot after a load.
struct BankImage {
  int32_t sample_rate = 0, bandwidth = 0, iq_format = 0;
  float iq_scale = 0.0f;
  int32_t channels = 0;
  size_t raw_bytes = 0, chunk_bytes = 0;  // the raw-sample carry; a complete chunk
  std::vector<size_t> carry_bytes;        // a channel's carry in each stage after the first
  const void* raw = nullptr;
  std::vector<const void*> carry;  // [channel][stage after the first]
};

// A bank's snapshot. `channels` are the bank's Channels (their position, their complete chunks and their tail).
template <class IO, class Channels>
void bank_sections(IO& io, BankImage& s, Channels& channels) {
  io.open("CONF", "the config block is missing or truncated");
  int32_t rate = s.sample_rate, bandwidth = s.bandwidth, format = s.iq_format, n_ch = s.channels;
  float scale = s.iq_scale;
  io(rate), io(bandwidth), io(format), io(scale), io(n_ch);
  io.close("the config block has the wrong length");
  io.check(rate == s.sample_rate && bandwidth == s.bandwidth && format == s.iq_format && std::memcmp(&scale, &s.iq_scale, sizeof(float)) == 0 &&
               n_ch == s.channels,
           "the snapshot was made by a bank with another sample rate, bandwidth, iq_format, iq_scale or channel count");

  io.open("RAWC", "the raw carry is missing or truncated");
  io.array(s.raw, s.raw_bytes);
  io.close("the raw carry has the wrong length");

  s.carry.resize(channels.size() * s.carry_bytes.size());
  size_t j = 0;
  for (auto& ch : channels) {
    io.open("CHAN", "a channel section is missing or truncated");
    io.flag(ch.recording), io.flag(ch.timed), io(ch.phase_inc), io(ch.seen), io(ch.start_ms), io(ch.flushed);
    for (size_t bytes : s.carry_bytes) io.array(s.carry[j++], bytes);
    list<uint64_t>(io, ch.chunks, "a channel's chunks are truncated", [&](auto& io, std::vector<int8_t>& chunk) { io.bytes(chunk, s.chunk_bytes); });
    uint64_t tail = ch.tail.size();
    io(tail);
    io.check(tail < s.chunk_bytes && tail % 2 == 0, "a channel's incomplete chunk is malformed");
    io.bytes(ch.tail, tail);
    io.close("a channel section is malformed");
    io.check(ch.seen >= 0 && ch.flushed >= 0, "a channel section is malformed");
  }
}

}  // namespace snapshot
