// b2s C-ABI implementation (include/b2s.h): engine / band objects, kernel launches, host tracker glue.
// The compute path is CUDA only; there is deliberately no CPU fallback anywhere in this file.
#include <cuda.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <chrono>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <limits>
#include <map>
#include <memory>
#include <mutex>
#include <set>
#include <string>
#include <type_traits>
#include <utility>
#include <vector>

#include "../../include/b2s.h"
#include "detect.cuh"
#include "host_utils.h"
#include "occupancy.cuh"
#include "recorder.cuh"
#include "scan_policy.h"
#include "spectral3.cuh"
#include "track.cuh"
#include "tracker.h"

namespace {

thread_local std::string g_error;

int fail(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_error = buf;
  return code;
}

#define CU(call)                                                                                        \
  do {                                                                                                  \
    cudaError_t err__ = (call);                                                                         \
    if (err__ != cudaSuccess) return fail(B2S_E_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(err__), __FILE__, __LINE__); \
  } while (0)

// copies up to `cap` of the queued events (or actions) to `out`, reports how many there are and drops the copied ones when asked to
template <class Queue, class T>
static void hand_out_events(Queue& q, T* out, int cap, int consume, int* count) {
  const int total = static_cast<int>(q.size()), n = out ? std::max(0, std::min(cap, total)) : 0;
  std::copy(q.begin(), q.begin() + n, out);
  *count = total;
  if (consume) q.erase(q.begin(), q.begin() + n);
}

// The owners of the library's CUDA resources. Each frees what it holds when it is destroyed and can be moved but not copied, so an
// object's resources go with the object and an early return frees what a function had allocated.

// `count` elements of device memory (DevBuf) or pinned host memory (PinBuf)
template <typename T, bool kPinned>
struct CudaBuf {
  T* p = nullptr;
  size_t n = 0;
  CudaBuf() = default;
  CudaBuf(CudaBuf&& o) noexcept : p(std::exchange(o.p, nullptr)), n(std::exchange(o.n, 0)) {}
  CudaBuf& operator=(CudaBuf&& o) noexcept {
    std::swap(p, o.p);
    std::swap(n, o.n);
    return *this;
  }
  ~CudaBuf() { free(); }
  // grow-only; a reallocation does not keep the contents
  int alloc(size_t count) {
    if (count <= n) return 0;
    free();
    const size_t bytes = count * sizeof(T);
    if ((kPinned ? cudaMallocHost(&p, bytes) : cudaMalloc(&p, bytes)) != cudaSuccess)
      return fail(B2S_E_NOMEM, "%s of %zu bytes failed", kPinned ? "cudaMallocHost" : "cudaMalloc", bytes);
    n = count;
    return 0;
  }

 private:
  void free() {
    if (p && kPinned) cudaFreeHost(p);
    if (p && !kPinned) cudaFree(p);
    p = nullptr;
    n = 0;
  }
};
template <typename T>
using DevBuf = CudaBuf<T, false>;
template <typename T>
using PinBuf = CudaBuf<T, true>;
static_assert(!std::is_copy_constructible<DevBuf<float>>::value && !std::is_copy_assignable<DevBuf<float>>::value, "DevBuf owns its memory");
static_assert(!std::is_copy_constructible<PinBuf<float>>::value && !std::is_copy_assignable<PinBuf<float>>::value, "PinBuf owns its memory");

// a stream or an event; it is created into `h` by the cudaStreamCreate* / cudaEventCreate* call (and flags) its owner needs
template <typename H>
struct CudaHandle {
  H h = nullptr;
  CudaHandle() = default;
  CudaHandle(CudaHandle&& o) noexcept : h(std::exchange(o.h, nullptr)) {}
  CudaHandle& operator=(CudaHandle&& o) noexcept {
    std::swap(h, o.h);
    return *this;
  }
  ~CudaHandle() {
    if (h) destroy(h);
  }
  operator H() const { return h; }

 private:
  static void destroy(cudaStream_t s) { cudaStreamDestroy(s); }
  static void destroy(cudaEvent_t e) { cudaEventDestroy(e); }
};
using Stream = CudaHandle<cudaStream_t>;
using Event = CudaHandle<cudaEvent_t>;
static_assert(!std::is_copy_constructible<Stream>::value && !std::is_copy_assignable<Stream>::value, "Stream owns its stream");
static_assert(!std::is_copy_constructible<Event>::value && !std::is_copy_assignable<Event>::value, "Event owns its event");

bool is_pow2(int v) { return v > 0 && (v & (v - 1)) == 0; }

void make_window(const b2s_band_config& cfg, std::vector<float>& w) {
  const int n = cfg.fft_size;
  w.resize(n);
  if (cfg.window_kind == B2S_WINDOW_USER && cfg.window_taps) {
    std::memcpy(w.data(), cfg.window_taps, sizeof(float) * n);
  } else {
    // gr::fft::window::hamming(N) (reference call site sources/radio/sdr_device.cpp:164): symmetric, double -> f32
    const double m = static_cast<double>(n - 1);
    for (int i = 0; i < n; ++i) w[i] = (n == 1) ? 1.0f : static_cast<float>(0.54 - 0.46 * std::cos((2.0 * M_PI * i) / m));
  }
}

}  // namespace

using namespace b2s;

// ------------------------------------------------------------------------------------------------------------
// engine
// ------------------------------------------------------------------------------------------------------------
struct b2s_engine {
  int device = 0;
  cudaDeviceProp prop{};
  int sm_count = 0;
  // kernels whose function attributes have been set on THIS device -> resident CTAs per SM. Function attributes are per
  // device, so the cache lives in the engine (one engine per GPU; several engines may share a process).
  std::mutex attr_mutex;
  std::map<const void*, int> kernel_ctas;
};

namespace {

// Opt the kernel into `smem` bytes of dynamic shared memory on the engine's device (once per engine) and report how many
// CTAs of `threads` threads fit on an SM.
template <typename K>
int prepare_kernel(b2s_engine* e, K kernel, int threads, size_t smem, int* ctas_per_sm) {
  std::lock_guard<std::mutex> lk(e->attr_mutex);
  const void* key = reinterpret_cast<const void*>(kernel);
  auto it = e->kernel_ctas.find(key);
  if (it == e->kernel_ctas.end()) {
    int ctas = 0;
    CU(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas, kernel, threads, smem));
    if (ctas < 1) return fail(B2S_E_CUDA, "a kernel needing %zu bytes of shared memory and %d threads does not fit on an SM of this device", smem, threads);
    it = e->kernel_ctas.emplace(key, ctas).first;
  }
  if (ctas_per_sm) *ctas_per_sm = it->second;
  return 0;
}

// K1 launcher -------------------------------------------------------------------------------------------------
template <int N, int MODE, bool LIN, bool SUB>
int launch_spectrum_v(b2s_engine* e, const SpectralArgs& a, cudaStream_t stream) {
  using PL = FftPlanT<N>;
  constexpr int T = N / PL::E;
  const size_t smem = sizeof(float2) * (exchange_elems<N>() + TwiddleLayout<N>::SMEM) + (MODE == kModeCs8Tma ? 2 * N : 0);
  int ctas_per_sm = 1;
  int rc = prepare_kernel(e, k_spectrum<N, MODE, LIN, SUB>, T, smem, &ctas_per_sm);
  if (rc) return rc;
  const int grid = std::min(a.n_frames, e->sm_count * ctas_per_sm);
  k_spectrum<N, MODE, LIN, SUB><<<grid, T, smem, stream>>>(a);
  CU(cudaGetLastError());
  return 0;
}
// k_spectrum3: N = RA * 1024 directly (RA = 4, 8, 16), or N = S * 16384 through the split mode (S = a.split > 1)
template <int RA, int MODE, bool LIN, int S, bool SUB>
int launch_spectrum3_v(b2s_engine* e, const SpectralArgs& a, cudaStream_t stream) {
  constexpr int T = RA * 32;
  constexpr bool SPLIT = S > 1;
  const size_t smem = sizeof(float2) * (RA * kBlockPitch + 31 * 32) + (MODE == kModeCs8Tma ? (SPLIT ? 2 * kSplitStageBytes : 2 * RA * 1024) : 0);
  int ctas_per_sm = 1;
  int rc = prepare_kernel(e, k_spectrum3<RA, MODE, LIN, S, SUB>, T, smem, &ctas_per_sm);
  if (rc) return rc;
  if (!a.work_counter) return fail(B2S_E_INVALID, "k_spectrum3 needs a work counter");
  const int items = a.n_frames * S;
  if (a.split != S) return fail(B2S_E_INVALID, "split tables were built for another fft_size");
  const int grid = std::min(items, std::max(1, e->sm_count - a.reserve_sms) * ctas_per_sm);
  if (SPLIT) {
    if (!a.peak_packed || !a.split_tw || !a.split_ws) return fail(B2S_E_INVALID, "split-mode tables are missing");
    CU(cudaMemsetAsync(a.peak_packed, 0, sizeof(unsigned long long) * a.n_frames, stream));
  }
  k_spectrum3<RA, MODE, LIN, S, SUB><<<grid, T, smem, stream>>>(a);
  CU(cudaGetLastError());
  if (SPLIT) {
    k_peak_unpack<<<(a.n_frames + 255) / 256, 256, 0, stream>>>(a.peak_packed, a.n_frames, a.peak_index, a.peak_value);
    CU(cudaGetLastError());
  }
  return 0;
}

// Which K1 serves which FFT size: k_spectrum (Stockham, two barriers per pass) below 4096, k_spectrum3 (warp-local passes) for
// 4096 / 8192 / 16384, and k_spectrum3's split mode (S residue classes x 16384 points) for 32768 ... 1048576.
constexpr int kMaxFft = 64 * kSplitM;
constexpr bool k1_is_v3(int n) { return n >= 4096; }

// A band's per-push PSD slot holds max_frames_per_push rows of N floats. The default is 4096 rows up to N = 262144; above
// that, the default and the cap are 2^30 / N rows, so that no slot is larger than the 4 GiB of a default slot at 262144.
constexpr long long kMaxPushBins = 1LL << 30;
constexpr int default_max_frames(int n) { return n > 16 * kSplitM ? static_cast<int>(kMaxPushBins / n) : 4096; }

template <int N, int MODE, bool SUB>
int launch_spectrum_s(b2s_engine* e, const SpectralArgs& a, cudaStream_t stream) {
  // the |X|^2/fs debug rows come from a debug twin of each instantiation (parity tests); the product one stays lean
  if constexpr (N > kSplitM) {
    if (a.power_lin) return launch_spectrum3_v<16, MODE, true, N / kSplitM, SUB>(e, a, stream);
    return launch_spectrum3_v<16, MODE, false, N / kSplitM, SUB>(e, a, stream);
  } else if constexpr (k1_is_v3(N)) {
    if (a.power_lin) return launch_spectrum3_v<N / 1024, MODE, true, 1, SUB>(e, a, stream);
    return launch_spectrum3_v<N / 1024, MODE, false, 1, SUB>(e, a, stream);
  } else {
    if (a.power_lin) return launch_spectrum_v<N, MODE, true, SUB>(e, a, stream);
    return launch_spectrum_v<N, MODE, false, SUB>(e, a, stream);
  }
}
// a.sub_r > 1 (sub-frames) runs the SUB instantiations; r = 1 runs the kernels of a frame without sub-frames
template <int N, int MODE>
int launch_spectrum_t(b2s_engine* e, const SpectralArgs& a, cudaStream_t stream) {
  if (a.sub_r > 1) return launch_spectrum_s<N, MODE, true>(e, a, stream);
  return launch_spectrum_s<N, MODE, false>(e, a, stream);
}

template <int MODE>
int launch_spectrum_n(b2s_engine* e, int n, const SpectralArgs& a, cudaStream_t stream) {
  if (!a.peak_index || !a.peak_value) return fail(B2S_E_INVALID, "peak buffers are required");
  switch (n) {
    case 256: return launch_spectrum_t<256, MODE>(e, a, stream);
    case 512: return launch_spectrum_t<512, MODE>(e, a, stream);
    case 1024: return launch_spectrum_t<1024, MODE>(e, a, stream);
    case 2048: return launch_spectrum_t<2048, MODE>(e, a, stream);
    case 4096: return launch_spectrum_t<4096, MODE>(e, a, stream);
    case 8192: return launch_spectrum_t<8192, MODE>(e, a, stream);
    case 16384: return launch_spectrum_t<16384, MODE>(e, a, stream);
    case 32768: return launch_spectrum_t<32768, MODE>(e, a, stream);
    case 65536: return launch_spectrum_t<65536, MODE>(e, a, stream);
    case 131072: return launch_spectrum_t<131072, MODE>(e, a, stream);
    case 262144: return launch_spectrum_t<262144, MODE>(e, a, stream);
    case 524288: return launch_spectrum_t<524288, MODE>(e, a, stream);
    case 1048576: return launch_spectrum_t<1048576, MODE>(e, a, stream);
    default: return fail(B2S_E_INVALID, "fft_size %d is not supported (256..%d)", n, kMaxFft);
  }
}

int launch_spectrum(b2s_engine* e, int n, int iq_format, const SpectralArgs& a, cudaStream_t stream) {
  if (iq_format == B2S_IQ_CF32) return launch_spectrum_n<kModeCf32>(e, n, a, stream);
  const bool aligned = (reinterpret_cast<uintptr_t>(a.iq) % 16 == 0) && (a.frame_stride_bytes % 16 == 0);
  if (aligned) return launch_spectrum_n<kModeCs8Tma>(e, n, a, stream);
  return launch_spectrum_n<kModeCs8Direct>(e, n, a, stream);
}

template <int N>
void plan_radices_t(int* r) {
  r[0] = FftPlanT<N>::R0;
  r[1] = FftPlanT<N>::R1;
  r[2] = FftPlanT<N>::R2;
  r[3] = FftPlanT<N>::R3;
}
void plan_radices(int n, int* r) {
  switch (n) {
    case 256: plan_radices_t<256>(r); break;
    case 512: plan_radices_t<512>(r); break;
    case 1024: plan_radices_t<1024>(r); break;
    case 2048: plan_radices_t<2048>(r); break;
    case 4096: plan_radices_t<4096>(r); break;
    case 8192: plan_radices_t<8192>(r); break;
    default: plan_radices_t<2048>(r); break;  // larger sizes run k_spectrum3, which has its own tables
  }
}

// Sub-frames a frame's PSD row is made of: floor(stride / N) with B2S_FLAG_SUBFRAME_MEAN or _MAX, stride / (N / 2) when they overlap
// by half (B2S_FLAG_SUBFRAME_OVERLAP), else 1.
constexpr int kSubframeFlags = B2S_FLAG_SUBFRAME_MEAN | B2S_FLAG_SUBFRAME_MAX;
bool overlapped(const b2s_band_config& c) { return (c.flags & B2S_FLAG_SUBFRAME_OVERLAP) != 0; }
int subframes(const b2s_band_config& c) {
  if (!(c.flags & kSubframeFlags)) return 1;
  return overlapped(c) ? c.frame_stride_samples / (c.fft_size / 2) : c.frame_stride_samples / c.fft_size;
}
// Samples a push of n >= 1 frames reads: its last frame needs its sub-frames only, unless they overlap (the last one ends with the
// stride) or `whole` (an attached bank reads the whole stream)
size_t push_samples(const b2s_band_config& c, size_t n, bool whole) {
  const size_t stride = static_cast<size_t>(c.frame_stride_samples);
  if (whole || overlapped(c)) return n * stride;
  return (n - 1) * stride + static_cast<size_t>(subframes(c)) * c.fft_size;
}

struct SpectralTables {
  DevBuf<float> wscale;
  DevBuf<float2> twiddle, split_tw, split_ws;
  DevBuf<int> work_counter;  // k_spectrum3's {next item, finished CTAs}; the kernel leaves both at zero
  int split = 1;
  int sub_r = 1, sub_max = 0;  // sub-frames per frame and their reduction (B2S_FLAG_SUBFRAME_*)
  long long sub_step = 0, sub_off = 0;  // where they lie (SpectralArgs::sub_step_bytes, sub_off_bytes)
  int build(const b2s_band_config& cfg) {
    const int n = cfg.fft_size;
    sub_r = subframes(cfg);
    sub_max = (cfg.flags & B2S_FLAG_SUBFRAME_MAX) != 0;
    const long long bps = cfg.iq_format == B2S_IQ_CS8 ? 2 : 8;
    sub_step = (overlapped(cfg) ? n / 2 : n) * bps;
    sub_off = overlapped(cfg) ? -(n / 2) * bps : 0;
    std::vector<float> w;
    make_window(cfg, w);
    if (cfg.iq_format == B2S_IQ_CS8) {
      // unpack scale folded into the window: x*scale*w -> x*(scale*w); differs from the two-step product by < 1 ulp
      for (int i = 0; i < n; ++i) w[i] = w[i] * cfg.iq_scale;
    }
    split = n > kSplitM ? n / kSplitM : 1;
    const int m = n / split;  // length of the transform the passes run (the whole FFT, or one residue class of it)
    std::vector<float2> tw;
    auto root = [](double num, double den) {
      const double ang = -2.0 * M_PI * num / den;
      return make_float2(static_cast<float>(std::cos(ang)), static_cast<float>(std::sin(ang)));
    };
    if (k1_is_v3(m)) {
      // k_spectrum3 (TwiddleLayout3): pass A  W_m^(b*k0) as [k0-1][b], b < 1024;  pass B  W_1024^(n2*k1) as [k1-1][n2]
      const int ra = m / 1024;
      for (int k0 = 1; k0 < ra; ++k0)
        for (int b = 0; b < 1024; ++b) tw.push_back(root(static_cast<double>(b) * k0, m));
      for (int k1 = 1; k1 < 32; ++k1)
        for (int n2 = 0; n2 < 32; ++n2) tw.push_back(root(static_cast<double>(n2) * k1, 1024.0));
    } else {
      // per-pass compact tables [m-1][k] = exp(-2 pi i k m / (P R)), interleaved (re, im), in the order of TwiddleLayout<N>
      int radix[4] = {0, 0, 0, 0};
      plan_radices(n, radix);
      int P = radix[0];
      for (int pass = 1; pass < 4 && radix[pass] > 1; ++pass) {
        const int R = radix[pass];
        for (int mm = 1; mm < R; ++mm)
          for (int k = 0; k < P; ++k) tw.push_back(root(static_cast<double>(k) * mm, static_cast<double>(P) * R));
        P *= R;
      }
    }
    int rc = wscale.alloc(n);
    if (rc) return rc;
    rc = twiddle.alloc(tw.size() + 1);
    if (rc) return rc;
    CU(cudaMemcpy(wscale.p, w.data(), sizeof(float) * n, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(twiddle.p, tw.data(), sizeof(float2) * tw.size(), cudaMemcpyHostToDevice));
    if ((rc = work_counter.alloc(2))) return rc;
    CU(cudaMemset(work_counter.p, 0, sizeof(int) * 2));
    if (split > 1) {
      // split mode: class twiddles W_N^(n' c) as [c][n'] (n' c < N^2 fits a double exactly), and the S-th roots of unity
      std::vector<float2> tc(static_cast<size_t>(split) * m), ws(split);
      for (int c = 0; c < split; ++c)
        for (int i = 0; i < m; ++i) tc[static_cast<size_t>(c) * m + i] = root(std::fmod(static_cast<double>(i) * c, static_cast<double>(n)), n);
      for (int j = 0; j < split; ++j) ws[j] = root(j, split);
      if ((rc = split_tw.alloc(tc.size()))) return rc;
      if ((rc = split_ws.alloc(ws.size()))) return rc;
      CU(cudaMemcpy(split_tw.p, tc.data(), sizeof(float2) * tc.size(), cudaMemcpyHostToDevice));
      CU(cudaMemcpy(split_ws.p, ws.data(), sizeof(float2) * ws.size(), cudaMemcpyHostToDevice));
    }
    return 0;
  }
  // the table pointers of a K1 launch
  void fill(SpectralArgs& sa) const {
    sa.wscale = wscale.p;
    sa.twiddle = twiddle.p;
    sa.work_counter = work_counter.p;
    sa.split = split;
    sa.split_tw = split_tw.p;
    sa.split_ws = split_ws.p;
    sa.sub_r = sub_r;
    sa.sub_max = sub_max;
    sa.sub_step_bytes = sub_step;
    sa.sub_off_bytes = sub_off;
  }
};

int validate_config(const b2s_band_config& c) {
  if (!is_pow2(c.fft_size) || c.fft_size < 256 || c.fft_size > kMaxFft) return fail(B2S_E_INVALID, "fft_size must be a power of two in 256..%d (got %d)", kMaxFft, c.fft_size);
  if (c.fft_size > 16 * kSplitM && static_cast<long long>(c.max_frames_per_push) * c.fft_size > kMaxPushBins)
    return fail(B2S_E_INVALID, "max_frames_per_push %d at fft_size %d exceeds %d: one push's PSD rows would take more than 4 GiB of device memory",
                c.max_frames_per_push, c.fft_size, default_max_frames(c.fft_size));
  if (c.sample_rate_hz <= 0) return fail(B2S_E_INVALID, "sample_rate_hz must be positive");
  if (c.frame_stride_samples < c.fft_size) return fail(B2S_E_INVALID, "frame_stride_samples (%d) < fft_size", c.frame_stride_samples);
  if (c.iq_format != B2S_IQ_CS8 && c.iq_format != B2S_IQ_CF32) return fail(B2S_E_INVALID, "unknown iq_format %d", c.iq_format);
  if ((c.flags & kSubframeFlags) == kSubframeFlags) return fail(B2S_E_INVALID, "B2S_FLAG_SUBFRAME_MEAN and B2S_FLAG_SUBFRAME_MAX exclude each other");
  if (overlapped(c) && !(c.flags & kSubframeFlags))
    return fail(B2S_E_INVALID, "B2S_FLAG_SUBFRAME_OVERLAP needs B2S_FLAG_SUBFRAME_MEAN or B2S_FLAG_SUBFRAME_MAX");
  if (overlapped(c) && c.frame_stride_samples % (c.fft_size / 2) != 0)
    return fail(B2S_E_INVALID, "B2S_FLAG_SUBFRAME_OVERLAP needs a frame_stride_samples (%d) that is a multiple of fft_size / 2", c.frame_stride_samples);
  if (c.window_kind == B2S_WINDOW_USER && !c.window_taps) return fail(B2S_E_INVALID, "window_taps is NULL");
  if (c.grouping_x < 1 || c.grouping_x > 65) return fail(B2S_E_INVALID, "grouping_x must be in 1..65");
  if (c.grouping_y < 1 || c.grouping_y > 256) return fail(B2S_E_INVALID, "grouping_y must be in 1..256");
  if (c.group_size_bins < 0 || c.group_size_bins > 4096) return fail(B2S_E_INVALID, "group_size_bins must be in 0..4096");
  if (c.learn_frames < 1) return fail(B2S_E_INVALID, "learn_frames must be >= 1");
  if (c.noise_learning_ms < 0) return fail(B2S_E_INVALID, "noise_learning_ms must be >= 0 (0 = count learn_frames frames)");
  if (c.n_ignored < 0 || c.n_ignored > B2S_MAX_IGNORED) return fail(B2S_E_INVALID, "n_ignored out of range");
  if (c.tuning_step_hz <= 0) return fail(B2S_E_INVALID, "tuning_step_hz must be positive");
  if (c.spectrogram_out_size < 0 || (c.spectrogram_out_size > 0 && (!is_pow2(c.spectrogram_out_size) || c.spectrogram_out_size > c.fft_size ||
                                                                   c.fft_size / c.spectrogram_out_size > kDetectBinsPerCta)))
    return fail(B2S_E_INVALID, "spectrogram_out_size must be 0 or a power of two with N/out <= %d", kDetectBinsPerCta);
  return 0;
}

}  // namespace

// 2-D tensor map over a row-major fp32 matrix [rows][cols] with box [box_rows][box_cols] (cuTensorMapEncodeTiled through the
// runtime's driver entry point: no link-time dependency on libcuda)
static int make_tile_map(CUtensorMap* out, const float* base, size_t cols, size_t rows, int box_cols, int box_rows) {
  using EncodeFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  static EncodeFn encode = nullptr;
  if (!encode) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    CU(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q));
    if (!fn || q != cudaDriverEntryPointSuccess) return fail(B2S_E_CUDA, "cuTensorMapEncodeTiled is not available in this driver");
    encode = reinterpret_cast<EncodeFn>(fn);
  }
  const cuuint64_t dims[2] = {cols, rows};
  const cuuint64_t strides[1] = {cols * sizeof(float)};
  const cuuint32_t box[2] = {static_cast<cuuint32_t>(box_cols), static_cast<cuuint32_t>(box_rows)};
  const cuuint32_t elem[2] = {1, 1};
  const CUresult r = encode(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), dims, strides, box, elem, CU_TENSOR_MAP_INTERLEAVE_NONE,
                            CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(B2S_E_CUDA, "cuTensorMapEncodeTiled failed (%d) for box %dx%d", static_cast<int>(r), box_cols, box_rows);
  return 0;
}

// Least float x with fl(x / divisor) >= level (IEEE single division is monotonic in x, so the bins whose quotient reaches a level
// are exactly those whose undivided sum reaches this x): lets K2 compare boxcar SUMS and divide only what leaves the kernel.
static float least_sum_reaching(float level, int divisor) {
  if (!std::isfinite(level)) return level;
  const float d = static_cast<float>(divisor);
  float x = level * d;
  for (int i = 0; i < 64 && !(x / d >= level); ++i) x = std::nextafterf(x, INFINITY);
  for (int i = 0; i < 64 && std::nextafterf(x, -INFINITY) / d >= level; ++i) x = std::nextafterf(x, -INFINITY);
  return x;
}

// ------------------------------------------------------------------------------------------------------------
// snapshots of a band or a recorder bank: the format
// ------------------------------------------------------------------------------------------------------------
#include "snapshot.h"

// ------------------------------------------------------------------------------------------------------------
// band
// ------------------------------------------------------------------------------------------------------------
#include "band.cuh"

// ------------------------------------------------------------------------------------------------------------
// recorder chain (recorder.cuh)
// ------------------------------------------------------------------------------------------------------------
// new carry = the last `hc` elements of (old carry ++ fresh[0 .. n_new)); one CTA, read everything before writing anything
template <typename T>
__global__ void k_shift_carry(T* carry, const T* fresh, int hc, long long n_new) {
  extern __shared__ unsigned char carry_smem[];
  T* tmp = reinterpret_cast<T*>(carry_smem);
  for (int i = threadIdx.x; i < hc; i += blockDim.x) {
    const long long j = i + n_new;  // position in (old carry ++ fresh)
    tmp[i] = j < hc ? carry[j] : fresh[j - hc];
  }
  __syncthreads();
  for (int i = threadIdx.x; i < hc; i += blockDim.x) carry[i] = tmp[i];
}
// the same for the per-channel buffers of a stage >= 1: CTA i shifts channel a.ch[i], whose row is [hc carried | n_in fresh]
__global__ void k_shift_carry_ch(const __grid_constant__ ResampleArgs a) {
  const StageChan& c = a.ch[blockIdx.x];
  double* row = static_cast<double*>(const_cast<void*>(a.carry)) + c.slot * a.in_stride;
  extern __shared__ unsigned char carry_smem[];
  double* tmp = reinterpret_cast<double*>(carry_smem);
  for (int i = threadIdx.x; i < a.hc; i += blockDim.x) {
    const long long j = i + static_cast<long long>(c.n_in);
    tmp[i] = row[j];  // j < hc: old carry, else fresh[j - hc]: the row is contiguous
  }
  __syncthreads();
  for (int i = threadIdx.x; i < a.hc; i += blockDim.x) row[i] = tmp[i];
}

// A bank of recorders on one IQ stream (SdrDevice::m_recorders, sdr_device.cpp:39-41): the stages, taps, stream, input staging and
// the raw-sample carry are shared; each channel has its shift, its start, its rows of the stage buffers and its chunk buffer.
struct b2s_recorder_bank {
  b2s_engine* engine = nullptr;
  int32_t sample_rate = 0, bandwidth = 0;
  int iq_format = B2S_IQ_CS8;
  float iq_scale = 1.0f;
  bool on_device = false;
  bool keep_chunks = true;  // false for a stand-alone b2s_recorder, whose caller takes the samples from every push
  size_t max_in = 0;
  int n_ch = 0;
  int chunk_samples = 0;  // roundUp(bandwidth * RECORDER_FLUSH_INTERVAL / 1000, 4096), recorder.cpp:35
  Stream stream;  // declared before the buffers, so it is destroyed after them
  struct Stage {
    int interp = 1, decim = 1, n_taps = 0, hc = 0;
    std::vector<float> h_taps;
    DevBuf<float> taps, taps_pq;  // taps_pq: [decim][kPolyQ] polyphase layout for k_decimate_poly (decimating stages), else empty
    DevBuf<float2> buf;           // stages >= 1: one row per channel, [hc carried samples | the previous stage's outputs of this push]
    size_t max_in = 0, stride = 0;  // stride: float2 per row
  };
  std::vector<Stage> stages;
  DevBuf<unsigned char> carry_raw, staging;  // stage 0: the stream's newest raw samples (shared); host input staging
  DevBuf<signed char> d_out;                 // [n_ch][out_stride] int8 pairs
  // h_out[slot]: the host copy of d_out. A push launched from an asynchronous band leaves its host side pending; the next push uses the
  // other slot, so its copy does not overwrite the output the pending push has not taken yet.
  PinBuf<signed char> h_out[2];
  Event out_ready[2];  // recorded after the device-to-host copy into h_out[slot] (pending pushes)
  size_t out_stride = 0;
  // One push between its launch and its host side: the channels it ran, what each produced, and whether the output was copied back
  struct Launched {
    std::vector<int> rec;
    std::vector<long long> produced;
    long long most = 0;
    int slot = 0;
    bool fetch = false;
  };
  Launched pending;
  bool has_pending = false;
  b2s_band* band = nullptr;  // the band whose pushes feed this bank (b2s_band_attach_recorder_bank), or none
  struct Channel {
    bool recording = false, timed = false;  // timed: start_ms is set (the first push after start)
    unsigned long long phase_inc = 0;
    long long seen = 0;        // stream samples pushed since startRecording
    int64_t start_ms = 0;
    long long flushed = 0;     // chunks consumed by flush since startRecording
    // int8 pairs not consumed by flush, like Buffer's items (buffer.h:22-55): complete chunks of chunk_samples, then the incomplete
    // tail. A push appends without moving what is already held, however long the caller waits to flush.
    std::deque<std::vector<int8_t>> chunks;
    std::vector<int8_t> tail;
    void hold(const int8_t* src, size_t bytes, size_t chunk_bytes) {
      while (bytes > 0) {
        if (tail.capacity() < chunk_bytes) tail.reserve(chunk_bytes);
        const size_t m = std::min(bytes, chunk_bytes - tail.size());
        tail.insert(tail.end(), src, src + m);
        src += m;
        bytes -= m;
        if (tail.size() == chunk_bytes) {
          chunks.push_back(std::move(tail));
          tail = std::vector<int8_t>();
        }
      }
    }
    void drop() {
      chunks.clear();
      tail = std::vector<int8_t>();
    }
  };
  std::vector<Channel> ch;
  // History (b2s_recorder_bank_set_history): the newest hist_cap raw samples of the stream, stream position p in ring slot
  // p % hist_cap. hist_end counts the samples pushed since the last set_history or load; hist_epoch changes whenever the history is
  // emptied, so that positions taken before are recognised as void.
  DevBuf<unsigned char> hist;
  size_t hist_cap = 0;
  long long hist_end = 0;
  uint64_t hist_epoch = 0;
  long long hist_oldest() const { return hist_end - std::min<long long>(hist_end, static_cast<long long>(hist_cap)); }
  size_t raw_bytes() const { return iq_format == B2S_IQ_CS8 ? 2 : 8; }
};

// one Recorder: a bank of one channel that keeps no chunks
struct b2s_recorder {
  std::unique_ptr<b2s_recorder_bank> bank;
};

namespace {

// outputs of a stage once it has seen g input samples: those whose newest input has arrived
long long stage_outputs(long long g, int interp, int decim) { return g > 0 ? (g * interp - 1) / decim + 1 : 0; }

// Recorder::startRecording (recorder.cpp:58-73): rotator phase increment per sample in turns, -shift / fs, as a 64-bit binary
// fraction (exact to 2^-65 turns)
unsigned long long rotator_phase_inc(int32_t shift_hz, int32_t sample_rate) {
  const long double turns = -static_cast<long double>(shift_hz) / static_cast<long double>(sample_rate);
  long double frac = turns - floorl(turns);  // [0, 1)
  unsigned long long inc = static_cast<unsigned long long>(frac * 18446744073709551616.0L + 0.5L);
  if (shift_hz != 0 && inc == 0) inc = 1;
  return inc;
}

void start_channel(b2s_recorder_bank::Channel& c, unsigned long long phase_inc) {
  c.recording = true;
  c.timed = false;
  c.phase_inc = phase_inc;
  c.seen = 0;
  c.start_ms = 0;
  c.flushed = 0;
  c.drop();
}

int bank_create(b2s_engine* e, int32_t sample_rate_hz, int32_t bandwidth_hz, int iq_format, float iq_scale, int flags, int n_channels, size_t max_samples_per_push,
                bool keep_chunks, std::unique_ptr<b2s_recorder_bank>& out) {
  CU(cudaSetDevice(e->device));
  auto k = std::make_unique<b2s_recorder_bank>();
  k->engine = e;
  k->sample_rate = sample_rate_hz;
  k->bandwidth = bandwidth_hz;
  k->iq_format = iq_format;
  k->iq_scale = iq_scale;
  k->on_device = (flags & B2S_FLAG_IQ_ON_DEVICE) != 0;
  k->keep_chunks = keep_chunks;
  k->max_in = max_samples_per_push ? max_samples_per_push : (size_t(1) << 22);
  k->n_ch = n_channels;
  k->chunk_samples = static_cast<int>((static_cast<long long>(bandwidth_hz) * 100 / 1000 + 4095) / 4096 * 4096);  // RECORDER_FLUSH_INTERVAL = 100 ms
  k->ch.resize(n_channels);
  const cudaError_t err = cudaStreamCreateWithFlags(&k->stream.h, cudaStreamNonBlocking);
  if (err != cudaSuccess) return fail(B2S_E_CUDA, "cudaStreamCreate: %s", cudaGetErrorString(err));
  int rc;
  size_t n_in = k->max_in;
  for (const auto& f : host::resamplers_factors(sample_rate_hz, bandwidth_hz, 125)) {  // RESAMPLER_THRESHOLD, config.h
    k->stages.emplace_back();
    auto& st = k->stages.back();
    st.interp = f.first;
    st.decim = f.second;
    st.h_taps = host::design_resampler_taps(st.interp, st.decim);
    st.n_taps = static_cast<int>(st.h_taps.size());
    st.hc = (st.n_taps - 1 + st.decim) / st.interp + 2;
    st.max_in = n_in;
    st.stride = st.hc + n_in + 2;
    if (st.hc > 4096) return fail(B2S_E_INVALID, "resampler stage %d/%d needs %d samples of history", st.interp, st.decim, st.hc);
    if ((rc = st.taps.alloc(st.n_taps))) return rc;
    if (cudaMemcpy(st.taps.p, st.h_taps.data(), sizeof(float) * st.n_taps, cudaMemcpyHostToDevice) != cudaSuccess) return fail(B2S_E_CUDA, "taps upload failed");
    if (st.interp == 1 && st.decim >= 2 && (st.n_taps + st.decim - 1) / st.decim <= kPolyQ) {
      std::vector<float> pq(static_cast<size_t>(st.decim) * kPolyQ, 0.0f);  // h[q D + p] at [p][q], zero padded
      for (int i = 0; i < st.n_taps; ++i) pq[static_cast<size_t>(i % st.decim) * kPolyQ + i / st.decim] = st.h_taps[i];
      if ((rc = st.taps_pq.alloc(pq.size()))) return rc;
      if (cudaMemcpy(st.taps_pq.p, pq.data(), sizeof(float) * pq.size(), cudaMemcpyHostToDevice) != cudaSuccess) return fail(B2S_E_CUDA, "taps upload failed");
    }
    if (k->stages.size() > 1 && (rc = st.buf.alloc(st.stride * n_channels))) return rc;
    n_in = (n_in * st.interp) / st.decim + 2;
  }
  k->out_stride = n_in;
  if ((rc = k->carry_raw.alloc(static_cast<size_t>(k->stages[0].hc) * k->raw_bytes()))) return rc;
  if ((rc = k->d_out.alloc(2 * k->out_stride * n_channels))) return rc;
  if ((rc = k->h_out[0].alloc(2 * k->out_stride * n_channels))) return rc;
  if (!k->on_device && (rc = k->staging.alloc(k->max_in * k->raw_bytes()))) return rc;
  out = std::move(k);
  return 0;
}

// Adds channel `channel`, fed its next n_samples stream samples, to the launch p: its geometry in every stage (appended to geo, which
// is [channel][stage]) and its output count (p.produced, p.most). Reads the channel's stream position and changes nothing.
void plan_channel(const b2s_recorder_bank* k, int channel, size_t n_samples, b2s_recorder_bank::Launched& p, std::vector<StageChan>& geo) {
  const auto& c = k->ch[channel];
  long long seen = c.seen, n_in = static_cast<long long>(n_samples);
  for (size_t si = 0; si < k->stages.size(); ++si) {
    const auto& st = k->stages[si];
    StageChan g{};
    g.g0 = seen;
    g.m0 = stage_outputs(seen, st.interp, st.decim);
    g.n_in = static_cast<int>(n_in);
    g.n_out = static_cast<int>(stage_outputs(seen + n_in, st.interp, st.decim) - g.m0);
    g.phase_inc = si == 0 ? c.phase_inc : 0ull;
    g.slot = channel;
    geo.push_back(g);
    seen = g.m0;
    n_in = g.n_out;
  }
  p.rec.push_back(channel);
  p.produced.push_back(n_in);
  p.most = std::max(p.most, n_in);
}

// What a push of n_samples does: every recording channel (p.rec), each one's geometry in every stage ([channel][stage], the return
// value) and output count (p.produced, p.most).
std::vector<StageChan> bank_plan(const b2s_recorder_bank* k, size_t n_samples, b2s_recorder_bank::Launched& p) {
  std::vector<StageChan> geo;
  p.rec.clear();
  p.produced.clear();
  p.most = 0;
  for (int i = 0; i < k->n_ch; ++i)
    if (k->ch[i].recording) plan_channel(k, i, n_samples, p, geo);
  return geo;
}

// One stage launch: the polyphase kernel for a decimating stage, the general one otherwise
template <class Args>
int launch_stage(b2s_recorder_bank* k, const b2s_recorder_bank::Stage& st, const Args& a, int most_out) {
  if (st.taps_pq.p) k_decimate_poly<<<((most_out + kPolyOut - 1) / kPolyOut) * a.n_ch, kPolyThreads, 0, k->stream>>>(a, st.taps_pq.p);
  else k_resample<<<((most_out + a.per_cta - 1) / a.per_cta) * a.n_ch, kResampleThreads, sizeof(float2) * kResampleTile, k->stream>>>(a);
  CU(cudaGetLastError());
  return 0;
}

// the history ring's slot of stream position pos >= 0
size_t hist_slot(const b2s_recorder_bank* k, long long pos) { return static_cast<size_t>(pos % static_cast<long long>(k->hist_cap)); }

// The device half of a push whose n_samples input samples are on the device at `in`: one launch per stage (per kLaunchChannels
// channels), the carries, and (p.fetch) the copy of the channels' int8 outputs into h_out[p.slot], all on the bank's stream. Advances the
// channels' stream positions by their stage-0 inputs.
// ring0 == nullptr: the stream's next n_samples samples. Stage 0 reads the shared raw carry and moves it on, and the samples are
// appended to the history; stage0_done (optional) is recorded once none of this reads `in` any more.
// Otherwise a catch-up piece (bank_catch_up): stage 0 reads the history ring in place, channel p.rec[i] from ring slot ring0[i], with
// the ring slots before it as its carry; `in` and n_samples are unused, and the shared raw carry and the history stay as they are.
int bank_launch(b2s_recorder_bank* k, const void* in, size_t n_samples, int64_t t0_ms, const std::vector<StageChan>& geo, const b2s_recorder_bank::Launched& p,
                cudaEvent_t stage0_done, const long long* ring0 = nullptr) {
  const int n_st = static_cast<int>(k->stages.size());
  const std::vector<int>& rec = p.rec;
  const int raw_kind = k->iq_format == B2S_IQ_CS8 ? 0 : 1;
  const bool stream_push = ring0 == nullptr;
  int rc;
  for (int si = 0; si < n_st; ++si) {
    auto& st = k->stages[si];
    const bool last = si + 1 == n_st;
    for (size_t c0 = 0; c0 < rec.size(); c0 += kLaunchChannels) {
      ResampleArgs a{};
      a.in = si == 0 ? in : static_cast<const void*>(st.buf.p + st.hc);
      a.carry = si > 0 ? static_cast<const void*>(st.buf.p) : stream_push ? static_cast<const void*>(k->carry_raw.p) : nullptr;
      a.in_stride = si == 0 ? 0 : static_cast<long long>(st.stride);
      a.kind = si == 0 ? raw_kind : 2;
      a.iq_scale = k->iq_scale;
      a.hc = st.hc;
      a.taps = st.taps.p;
      a.n_taps = st.n_taps;
      a.interp = st.interp;
      a.decim = st.decim;
      a.per_cta = std::max(1, std::min(kResampleThreads, static_cast<int>((static_cast<long long>(kResampleTile - 2) - st.n_taps / st.interp) * st.interp / st.decim)));
      if (last) {
        a.out_i8 = k->d_out.p;
        a.out_stride = static_cast<long long>(k->out_stride);
      } else {
        a.out_f = k->stages[si + 1].buf.p + k->stages[si + 1].hc;
        a.out_stride = static_cast<long long>(k->stages[si + 1].stride);
      }
      a.n_ch = static_cast<int>(std::min<size_t>(kLaunchChannels, rec.size() - c0));
      int most_out = 0;
      for (int j = 0; j < a.n_ch; ++j) {
        a.ch[j] = geo[(c0 + j) * n_st + si];
        most_out = std::max(most_out, a.ch[j].n_out);
      }
      if (most_out > 0 && si == 0 && !stream_push) {
        RingArgs r{};
        static_cast<ResampleArgs&>(r) = a;
        r.in = k->hist.p;
        r.ring_cap = static_cast<long long>(k->hist_cap);
        for (int j = 0; j < a.n_ch; ++j) r.ring0[j] = ring0[c0 + j];
        if ((rc = launch_stage(k, st, r, most_out))) return rc;
      } else if (most_out > 0 && (rc = launch_stage(k, st, a, most_out))) {
        return rc;
      }
      // carry the newest inputs of this stage over to the next push
      if (si > 0) {
        k_shift_carry_ch<<<a.n_ch, 1024, st.hc * 8, k->stream>>>(a);
        CU(cudaGetLastError());
      }
    }
    if (si == 0 && stream_push) {  // the raw stream's carry, shared by every channel, moves with every push
      if (raw_kind == 0) k_shift_carry<short><<<1, 1024, st.hc * 2, k->stream>>>(static_cast<short*>(static_cast<void*>(k->carry_raw.p)), static_cast<const short*>(in), st.hc, n_samples);
      else k_shift_carry<double><<<1, 1024, st.hc * 8, k->stream>>>(static_cast<double*>(static_cast<void*>(k->carry_raw.p)), static_cast<const double*>(in), st.hc, n_samples);
      CU(cudaGetLastError());
      if (k->hist_cap) {  // the push's newest hist_cap samples into the history ring, cut where the ring ends
        const size_t bps = k->raw_bytes(), keep = std::min(n_samples, k->hist_cap);
        const long long from = k->hist_end + static_cast<long long>(n_samples - keep);
        const unsigned char* src = static_cast<const unsigned char*>(in) + (n_samples - keep) * bps;
        for (size_t done = 0; done < keep;) {
          const size_t at = hist_slot(k, from + static_cast<long long>(done)), m = std::min(keep - done, k->hist_cap - at);
          CU(cudaMemcpyAsync(k->hist.p + at * bps, src + done * bps, m * bps, cudaMemcpyDeviceToDevice, k->stream));
          done += m;
        }
      }
      k->hist_end += static_cast<long long>(n_samples);
      if (stage0_done) CU(cudaEventRecord(stage0_done, k->stream));
    }
  }
  if (p.fetch) {
    const size_t rows = static_cast<size_t>(rec.back()) + 1, pitch = 2 * k->out_stride;
    CU(cudaMemcpy2DAsync(k->h_out[p.slot].p, pitch, k->d_out.p, pitch, 2 * static_cast<size_t>(p.most), rows, cudaMemcpyDeviceToHost, k->stream));
  }
  for (size_t i = 0; i < rec.size(); ++i) {
    auto& c = k->ch[rec[i]];
    if (!c.timed) {
      c.timed = true;
      c.start_ms = t0_ms;
    }
    c.seen += geo[i * n_st].n_in;
  }
  return 0;
}

// The host half of a launched push, once its output copy has completed: each channel keeps its samples as chunks, and a direct push
// also hands them to the caller (out_iq, n_out).
void bank_take(b2s_recorder_bank* k, const b2s_recorder_bank::Launched& p, int8_t* out_iq, size_t cap_samples, size_t* n_out) {
  for (size_t i = 0; i < p.rec.size(); ++i) {
    auto& c = k->ch[p.rec[i]];
    const size_t bytes = 2 * static_cast<size_t>(p.produced[i]);
    const int8_t* src = reinterpret_cast<const int8_t*>(k->h_out[p.slot].p) + 2 * k->out_stride * p.rec[i];
    if (p.fetch && out_iq) std::memcpy(out_iq + 2 * cap_samples * p.rec[i], src, bytes);
    if (p.fetch && k->keep_chunks) c.hold(src, bytes, 2 * static_cast<size_t>(k->chunk_samples));
    if (n_out) n_out[p.rec[i]] = static_cast<size_t>(p.produced[i]);
  }
}

// The host side of the push that a band left pending (an asynchronous band's latest piece), if there is one
int bank_settle(b2s_recorder_bank* k) {
  if (!k->has_pending) return 0;
  CU(cudaSetDevice(k->engine->device));
  CU(cudaEventSynchronize(k->out_ready[k->pending.slot]));
  k->has_pending = false;
  bank_take(k, k->pending, nullptr, 0, nullptr);
  return 0;
}

// The stream's next n_samples through every recording channel: one launch per stage (per kLaunchChannels channels), the channels'
// int8 outputs back in one copy, one synchronise. Every check comes before the first copy or launch, so a refused push changes
// nothing. n_out (optional): [n_ch] samples per channel; out_iq (optional): [n_ch][cap_samples] int8 pairs.
int bank_push(b2s_recorder_bank* k, const void* iq, size_t n_samples, int64_t t0_ms, int8_t* out_iq, size_t cap_samples, bool check_cap, size_t* n_out,
              const char* who) {
  int rc = bank_settle(k);
  if (rc) return rc;
  if (n_samples > k->max_in) return fail(B2S_E_INVALID, "%s: %zu samples exceed max_samples_per_push %zu", who, n_samples, k->max_in);
  b2s_recorder_bank::Launched p;
  const std::vector<StageChan> geo = bank_plan(k, n_samples, p);
  if (check_cap && static_cast<size_t>(p.most) > cap_samples) return fail(B2S_E_INVALID, "%s: %lld output samples, the buffer holds %zu", who, p.most, cap_samples);
  if (n_out)
    for (int i = 0; i < k->n_ch; ++i) n_out[i] = 0;
  if (n_samples == 0) return 0;
  CU(cudaSetDevice(k->engine->device));
  const void* in = iq;
  if (!k->on_device) {
    CU(cudaMemcpyAsync(k->staging.p, iq, n_samples * k->raw_bytes(), cudaMemcpyHostToDevice, k->stream));
    in = k->staging.p;
  }
  p.fetch = p.most > 0 && (out_iq || k->keep_chunks);
  if ((rc = bank_launch(k, in, n_samples, t0_ms, geo, p, nullptr))) return rc;
  CU(cudaStreamSynchronize(k->stream));
  bank_take(k, p, out_iq, cap_samples, n_out);
  return 0;
}

// One piece of an attached band's push through the bank: the n_samples already on the device at `in`, read once `ready` (an event of
// the band's) has fired. The piece stays pending (its host side is done by bank_settle); the push pending before it is settled here,
// after this one is launched into the other output slot, so that the bank's kernels of consecutive pieces follow each other without a
// host wait in between.
int bank_feed(b2s_recorder_bank* k, const void* in, size_t n_samples, int64_t t0_ms, cudaEvent_t ready, cudaEvent_t stage0_done) {
  int rc = 0;
  // with one output slot (a bank that has only fed synchronous bands) the pending piece, left by a push that failed, is settled first
  if (k->has_pending && !k->h_out[1].p && (rc = bank_settle(k))) return rc;
  b2s_recorder_bank::Launched p;
  const std::vector<StageChan> geo = bank_plan(k, n_samples, p);
  p.slot = k->has_pending ? k->pending.slot ^ 1 : 0;
  p.fetch = p.most > 0;
  CU(cudaStreamWaitEvent(k->stream, ready, 0));
  rc = bank_launch(k, in, n_samples, t0_ms, geo, p, stage0_done);
  if (rc) return rc;
  CU(cudaEventRecord(k->out_ready[p.slot], k->stream));
  if ((rc = bank_settle(k))) return rc;
  k->pending = std::move(p);
  k->has_pending = true;
  return 0;
}

// A channel to start from the history: b2s_recorder_bank_start_from's arguments
struct CatchUp {
  int channel;
  int32_t shift_hz;
  long long position;
  int64_t start_ms;
};

// Start the channels `starts` (idle, distinct, positions inside the history) at their positions: each channel's samples [position, end)
// run at once, cut every max_in samples from its own position as a fresh bank's pushes would be, with seen counting from that position.
// Piece j of every channel goes into one launch per stage (per kLaunchChannels channels), each channel with its own geometry; channels
// with fewer pieces drop out of the later launches. Stage 0 reads each piece in the history ring in place, with the ring slots before it
// as its carry (the first piece reads none: they precede the channel's start). One synchronise per piece index. Synchronous on the
// bank's stream, which also orders it after every piece a band has fed; the caller has settled the bank's pending piece.
int bank_catch_up(b2s_recorder_bank* k, std::vector<CatchUp> starts) {
  std::sort(starts.begin(), starts.end(), [](const CatchUp& a, const CatchUp& b) { return a.channel < b.channel; });  // rows of one copy
  for (const CatchUp& s : starts) {
    auto& c = k->ch[s.channel];
    start_channel(c, rotator_phase_inc(s.shift_hz, k->sample_rate));
    if (s.position < k->hist_end) {  // stamped from start_ms by its first piece (at the end of the history: by the next push)
      c.timed = true;
      c.start_ms = s.start_ms;
    }
  }
  CU(cudaSetDevice(k->engine->device));
  const long long step = static_cast<long long>(k->max_in);
  for (long long j = 0;; ++j) {
    b2s_recorder_bank::Launched p;
    std::vector<StageChan> geo;
    std::vector<long long> ring0;
    for (const CatchUp& s : starts) {
      const long long a = s.position + j * step;
      if (a >= k->hist_end) continue;
      plan_channel(k, s.channel, static_cast<size_t>(std::min(step, k->hist_end - a)), p, geo);
      ring0.push_back(static_cast<long long>(hist_slot(k, a)));
    }
    if (p.rec.empty()) return 0;
    p.fetch = p.most > 0;
    int rc = bank_launch(k, nullptr, 0, 0, geo, p, nullptr, ring0.data());
    if (rc) return rc;
    CU(cudaStreamSynchronize(k->stream));
    bank_take(k, p, nullptr, 0, nullptr);
  }
}

// b2s_recorder_bank_start_from: the checks, then the catch-up of the one channel
int bank_start_from(b2s_recorder_bank* k, int channel, int32_t shift_hz, long long position, int64_t start_ms, const char* who) {
  int rc = bank_settle(k);
  if (rc) return rc;
  if (k->ch[channel].recording) return fail(B2S_E_STATE, "%s: channel %d is already recording", who, channel);
  if (!k->hist_cap || position < k->hist_oldest() || position > k->hist_end)
    return fail(B2S_E_INVALID, "%s: position %lld is outside the history [%lld, %lld)", who, position, k->hist_oldest(), k->hist_end);
  return bank_catch_up(k, {CatchUp{channel, shift_hz, position, start_ms}});
}

// Detach the band's bank (b->mutex held): the band's outstanding pushes are drained and the bank's last push settled, so that neither
// object refers to the other afterwards. The bank keeps its stream position. Detaches even when draining reports an earlier error,
// which it then returns.
int band_detach(b2s_band* b) {
  if (!b->bank) return 0;
  int rc = b->drain();
  const int rc2 = bank_settle(b->bank);
  b->bank->band = nullptr;
  b->bank = nullptr;
  b->autorec = b2s_band::AutoRecord{};
  b->d_whole = DevBuf<unsigned char>();
  return rc ? rc : rc2;
}

// bank_feed of the piece of a band push that starts at frame `first` of the push, band frame `frame`, `frames` frames long. While the
// bank keeps history the band notes where the piece sits in the bank's stream, for b2s_band_record_from.
int band_feed(b2s_band* b, const void* in, int64_t frame, size_t first, size_t frames, int64_t t0_ms, double period_ms, cudaEvent_t ready,
              cudaEvent_t stage0_done) {
  b2s_recorder_bank* k = b->bank;
  const long long position = k->hist_end;
  const int rc = bank_feed(k, in, frames * static_cast<size_t>(b->cfg.frame_stride_samples), host::frame_time(t0_ms, period_ms, first), ready, stage0_done);
  if (rc || !k->hist_cap) return rc;
  if (b->hist_epoch != k->hist_epoch) {
    b->hist_pieces.clear();
    b->hist_epoch = k->hist_epoch;
  }
  b->hist_pieces.push_back({frame, static_cast<int64_t>(frames), position, t0_ms, period_ms, first});
  const long long stride = b->cfg.frame_stride_samples;
  while (!b->hist_pieces.empty() && b->hist_pieces.front().position + b->hist_pieces.front().n_frames * stride <= k->hist_oldest()) b->hist_pieces.pop_front();
  return 0;
}

// Band frame `frame`'s position in the attached bank's stream and its clock, when the bank's history holds it: b2s_band_record_from's rule
bool band_frame_in_history(const b2s_band* b, int64_t frame, long long* position, int64_t* time_ms) {
  const b2s_recorder_bank* k = b->bank;
  if (!k || !k->hist_cap || b->hist_epoch != k->hist_epoch) return false;
  const b2s_band::HistPiece* piece = nullptr;  // the newest piece that starts at or before `frame`
  for (auto it = b->hist_pieces.rbegin(); it != b->hist_pieces.rend() && !piece; ++it)
    if (it->frame <= frame) piece = &*it;
  if (!piece || frame >= piece->frame + piece->n_frames) return false;
  *position = piece->position + (frame - piece->frame) * static_cast<long long>(b->cfg.frame_stride_samples);
  *time_ms = host::frame_time(piece->t0_ms, piece->period_ms, piece->first + static_cast<size_t>(frame - piece->frame));
  return *position >= k->hist_oldest();
}

// The oldest band frame band_frame_in_history accepts, or -1 when it accepts none
int64_t band_oldest_frame(const b2s_band* b) {
  const b2s_recorder_bank* k = b->bank;
  if (!k || !k->hist_cap || b->hist_epoch != k->hist_epoch) return -1;
  const long long stride = b->cfg.frame_stride_samples;
  for (const auto& p : b->hist_pieces) {
    const long long skip = std::max(0LL, (k->hist_oldest() - p.position + stride - 1) / stride);  // frames of the piece that left
    if (skip < p.n_frames) return p.frame + skip;
  }
  return -1;
}

bool bank_auto_recorded(const b2s_recorder_bank* k) { return k->band && k->band->autorec.on; }

// Auto-record's decision for the push that finished last (b->autorec.due): ScanPolicy::update_recordings on the mailbox, then the bank's
// stops, the starts without usable history, and one catch-up for the starts from history, in that order of effect on the bank (each
// action touches another channel, so the order does not show in the output).
int band_auto_decide(b2s_band* b) {
  auto& a = b->autorec;
  if (!a.on || !a.due) return 0;
  a.due = false;
  b2s_recorder_bank* k = b->bank;
  std::vector<b2s_transmission> list;
  {
    std::lock_guard<std::mutex> lk(b->qmutex);
    list = b->mailbox;
  }
  std::vector<b2s_recorder_action> acts;
  std::vector<int> source;
  a.policy->update_recordings(a.time_ms, list.data(), static_cast<int>(list.size()), acts, &source);
  int rc = bank_settle(k);
  if (rc) return rc;
  const int64_t oldest = band_oldest_frame(b);
  std::vector<CatchUp> catch_up;
  for (size_t i = 0; i < acts.size(); ++i) {
    const b2s_recorder_action& act = acts[i];
    b2s_auto_record_action out{act.kind, act.recorder, act.shift_hz, source[i] >= 0 ? list[source[i]].key : 0, a.frame, -1, a.time_ms, 0};
    if (act.kind == B2S_REC_STOP) {
      out.key = a.key[act.recorder];
      out.duration_ms = act.duration_ms;
      auto& c = k->ch[act.recorder];
      c.recording = false;
      c.drop();
    } else if (act.kind == B2S_REC_START) {
      a.key[act.recorder] = out.key;
      bool found = false;
      std::pair<int64_t, int64_t> start{0, 0};
      {
        std::lock_guard<std::mutex> lk(b->qmutex);
        auto it = b->start_of.find(out.key);
        found = it != b->start_of.end() && it->second.first > b->start_lost_through;
        if (found) start = it->second;
      }
      long long position = 0;
      int64_t time_ms = 0;
      found = found && start.first >= a.enabled_at && start.first <= a.frame && oldest >= 0 && start.first >= oldest &&
              band_frame_in_history(b, start.first, &position, &time_ms);
      if (found) {
        out.from_frame = std::max(start.first - a.preroll, oldest);
        band_frame_in_history(b, out.from_frame, &position, &out.time_ms);
        catch_up.push_back(CatchUp{act.recorder, act.shift_hz, position, out.time_ms});
      } else {
        start_channel(k->ch[act.recorder], rotator_phase_inc(act.shift_hz, k->sample_rate));
      }
    }
    b->auto_actions.push_back(out);
  }
  return bank_catch_up(k, std::move(catch_up));
}

// ---- recorder bank snapshot (snapshot.h) ----
// channel i's row of stage si >= 1, whose first hc samples are its carry
float2* stage_row(b2s_recorder_bank* k, size_t si, int i) { return k->stages[si].buf.p + k->stages[si].stride * i; }
// Finishes the bank's work, then describes it: its config and sizes, and for a save its device arrays
int bank_image(b2s_recorder_bank* k, snapshot::BankImage& s) {
  int rc = bank_settle(k);
  if (rc) return rc;
  CU(cudaSetDevice(k->engine->device));
  CU(cudaStreamSynchronize(k->stream));
  s.sample_rate = k->sample_rate, s.bandwidth = k->bandwidth, s.iq_format = k->iq_format, s.iq_scale = k->iq_scale, s.channels = k->n_ch;
  s.raw_bytes = static_cast<size_t>(k->stages[0].hc) * k->raw_bytes();
  s.chunk_bytes = 2 * static_cast<size_t>(k->chunk_samples);
  for (size_t si = 1; si < k->stages.size(); ++si) s.carry_bytes.push_back(sizeof(float2) * k->stages[si].hc);
  s.raw = k->carry_raw.p;
  for (int i = 0; i < k->n_ch; ++i)
    for (size_t si = 1; si < k->stages.size(); ++si) s.carry.push_back(stage_row(k, si, i));
  return 0;
}

int bank_save(b2s_recorder_bank* k, std::vector<uint8_t>& out) {
  snapshot::BankImage s;
  const int rc = bank_image(k, s);
  return rc ? rc : snapshot::write(snapshot::kBank, k->stream, out, [&](snapshot::Writer& w) { snapshot::bank_sections(w, s, k->ch); });
}

int bank_load(b2s_recorder_bank* k, const void* buf, size_t len) {
  snapshot::BankImage s;
  std::vector<b2s_recorder_bank::Channel> s_ch(k->n_ch);
  int rc = bank_image(k, s);
  if (rc || (rc = snapshot::read(buf, len, snapshot::kBank, "b2s_recorder_bank_load_state", [&](snapshot::Reader& r) { snapshot::bank_sections(r, s, s_ch); })))
    return rc;
  CU(cudaMemcpyAsync(k->carry_raw.p, s.raw, s.raw_bytes, cudaMemcpyHostToDevice, k->stream));
  size_t j = 0;
  for (int i = 0; i < k->n_ch; ++i)
    for (size_t si = 1; si < k->stages.size(); ++si, ++j) CU(cudaMemcpyAsync(stage_row(k, si, i), s.carry[j], s.carry_bytes[si - 1], cudaMemcpyHostToDevice, k->stream));
  CU(cudaStreamSynchronize(k->stream));
  k->ch.swap(s_ch);
  k->hist_end = 0;  // the history, which a snapshot does not hold, is of another stream
  ++k->hist_epoch;
  return 0;
}

// the C-ABI half of a save: the snapshot if it fits `cap`, its size in any case
int hand_out_state(const std::vector<uint8_t>& blob, void* buf, size_t cap, size_t* written, const char* who) {
  *written = blob.size();
  if (!buf || cap < blob.size()) return fail(B2S_E_INVALID, "%s: the snapshot needs %zu bytes, the buffer holds %zu", who, blob.size(), buf ? cap : 0);
  std::memcpy(buf, blob.data(), blob.size());
  return 0;
}

}  // namespace

// ------------------------------------------------------------------------------------------------------------
// stand-alone device Averager
// ------------------------------------------------------------------------------------------------------------
struct b2s_averager {
  b2s_engine* engine = nullptr;
  int size = 0, group = 0, frames = 0, cur = 0;
  DevBuf<float> sum, ring[2], avg, rows;
  int reset() {
    CU(cudaMemset(sum.p, 0, sizeof(float) * size));
    CU(cudaMemset(ring[0].p, 0, sizeof(float) * size * group));
    CU(cudaMemset(ring[1].p, 0, sizeof(float) * size * group));
    std::vector<float> nd(size, kNoData);
    CU(cudaMemcpy(avg.p, nd.data(), sizeof(float) * size, cudaMemcpyHostToDevice));
    frames = 0;
    cur = 0;
    return 0;
  }
};

// ---- self-test of the exact constant division used on the Averager / boxcar fast paths (detect.cuh: div_const) ----
template <int D>
static int run_div_check(const b2s_engine* e, unsigned long long* d_bad) {
  k_check_div_const<D><<<e->sm_count * 8, 256>>>(d_bad);
  CU(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------------------------
// C-ABI
// ------------------------------------------------------------------------------------------------------------
extern "C" {

const char* b2s_last_error(void) { return g_error.c_str(); }
int b2s_version(void) { return B2S_VERSION; }

int b2s_engine_create(int cuda_device, b2s_engine** out) {
  if (!out) return fail(B2S_E_INVALID, "out is NULL");
  *out = nullptr;
  int count = 0;
  cudaError_t err = cudaGetDeviceCount(&count);
  if (err != cudaSuccess || count == 0) return fail(B2S_E_CUDA, "no usable CUDA device (%s); this engine has no CPU fallback", cudaGetErrorString(err));
  if (cuda_device < 0 || cuda_device >= count) return fail(B2S_E_INVALID, "cuda_device %d out of range (0..%d)", cuda_device, count - 1);
  auto e = std::make_unique<b2s_engine>();
  e->device = cuda_device;
  CU(cudaSetDevice(cuda_device));
  CU(cudaGetDeviceProperties(&e->prop, cuda_device));
  if (e->prop.major != 9 || e->prop.minor != 0)  // sm_90a code runs on compute capability 9.0 and nothing else
    return fail(B2S_E_CUDA, "device is sm_%d%d; this build targets sm_90a (H100) only", e->prop.major, e->prop.minor);
  e->sm_count = e->prop.multiProcessorCount;
  *out = e.release();
  return 0;
}
int b2s_engine_destroy(b2s_engine* e) {
  delete e;
  return 0;
}
int b2s_engine_device_name(b2s_engine* e, char* buf, size_t cap) {
  if (!e || !buf || cap == 0) return fail(B2S_E_INVALID, "bad argument");
  snprintf(buf, cap, "%s (%d SMs)", e->prop.name, e->sm_count);
  return 0;
}

void b2s_default_config(b2s_band_config* cfg, int32_t sample_rate_hz, int32_t center_hz, int32_t recording_bandwidth_hz) {
  std::memset(cfg, 0, sizeof(*cfg));
  const int n = host::fft_size_for(sample_rate_hz, 250);  // SIGNAL_DETECTION_MAX_STEP, config.h:33
  const double step = static_cast<double>(sample_rate_hz) / n;
  cfg->fft_size = n;
  cfg->sample_rate_hz = sample_rate_hz;
  cfg->frame_stride_samples = n * host::decimator_factor(sample_rate_hz, n);
  cfg->iq_format = B2S_IQ_CS8;
  cfg->iq_scale = 1.0f / 127.0f;
  cfg->window_kind = B2S_WINDOW_HAMMING;
  cfg->grouping_x = 21;
  cfg->grouping_y = 21;
  cfg->group_size_bins = static_cast<int32_t>(std::ceil(recording_bandwidth_hz / step));  // sdr_device.cpp:151
  cfg->start_level = 8.0f;
  cfg->stop_level = 5.0f;
  const double period = static_cast<double>(cfg->frame_stride_samples) * 1000.0 / sample_rate_hz;
  cfg->learn_frames = b2s_learn_frames_from_ms(2000, period);
  cfg->noise_learning_ms = 2000;  // NOISE_LEARNING_TIME (config.h:24): the reference's wall-clock rule on the frame clock
  cfg->center_hz = center_hz;
  cfg->range_lo_hz = center_hz - sample_rate_hz / 2;
  cfg->range_hi_hz = center_hz + sample_rate_hz / 2;
  cfg->tuning_step_hz = 2500;
  cfg->min_time_ms = 2000;
  cfg->timeout_ms = 2000;
  cfg->max_time_ms = 600000;
  cfg->spectrogram_out_size = std::min(n, std::min(16384, host::fft_size_for(sample_rate_hz, 1000)));
  cfg->spectrogram_interval_ms = 1000;
}

int b2s_band_create(b2s_engine* e, const b2s_band_config* cfg, b2s_band** out) {
  if (!e || !cfg || !out) return fail(B2S_E_INVALID, "NULL argument");
  *out = nullptr;
  int rc = validate_config(*cfg);
  if (rc) return rc;
  auto b = std::make_unique<b2s_band>();
  if ((rc = b->init(e, *cfg))) return rc;
  *out = b.release();
  return 0;
}
int b2s_band_destroy(b2s_band* b) {
  if (b) {
    cudaSetDevice(b->engine->device);
    {
      std::lock_guard<std::mutex> lock(b->mutex);
      band_detach(b);  // the bank continues on its own
    }
    delete b;
  }
  return 0;
}

int b2s_band_attach_recorder_bank(b2s_band* b, b2s_recorder_bank* k) {
  if (!b) return fail(B2S_E_INVALID, "NULL band");
  std::lock_guard<std::mutex> lock(b->mutex);
  CU(cudaSetDevice(b->engine->device));
  if (!k) return band_detach(b);
  if (b->bank) return fail(B2S_E_INVALID, "b2s_band_attach_recorder_bank: the band already has a recorder bank (detach it first)");
  if (k->band) return fail(B2S_E_INVALID, "b2s_band_attach_recorder_bank: the recorder bank is attached to a band");
  if (k->engine != b->engine) return fail(B2S_E_INVALID, "b2s_band_attach_recorder_bank: the recorder bank belongs to another engine");
  if (k->sample_rate != b->cfg.sample_rate_hz || k->iq_format != b->cfg.iq_format || k->iq_scale != b->cfg.iq_scale)
    return fail(B2S_E_INVALID, "b2s_band_attach_recorder_bank: the recorder bank's sample rate, iq_format or iq_scale differs from the band's");
  const size_t stride = static_cast<size_t>(b->cfg.frame_stride_samples), need = static_cast<size_t>(b->max_frames) * stride;
  if (k->max_in < need)
    return fail(B2S_E_INVALID, "b2s_band_attach_recorder_bank: max_samples_per_push %zu is below max_frames_per_push x frame_stride_samples = %zu", k->max_in, need);
  // everything the attachment needs is allocated before either object changes
  DevBuf<unsigned char> whole;
  int rc = 0;
  if (!(b->cfg.flags & B2S_FLAG_IQ_ON_DEVICE) && !b->async_mode && (rc = whole.alloc(need * k->raw_bytes()))) return rc;
  if (b->async_mode && (rc = k->h_out[1].alloc(k->h_out[0].n))) return rc;  // its latest piece is still pending when the next one launches
  for (auto* e : {&b->bank_prev_use[0], &b->bank_prev_use[1], &b->push_ready, &b->bank_read, &k->out_ready[0], &k->out_ready[1]}) {
    if (!*e) CU(cudaEventCreateWithFlags(&e->h, cudaEventDisableTiming));
  }
  b->d_whole = std::move(whole);
  b->bank = k;
  k->band = b;
  b->hist_pieces.clear();  // frames pushed before the attachment are not in the bank's history
  return 0;
}
int b2s_band_set_stream(b2s_band* b, void* cuda_stream) {
  if (!b) return fail(B2S_E_INVALID, "NULL band");
  std::lock_guard<std::mutex> lock(b->mutex);
  int rc = b->drain();
  if (rc) return rc;
  b->stream = cuda_stream ? static_cast<cudaStream_t>(cuda_stream) : b->own_stream;
  return 0;
}

static int band_push(b2s_band* b, const void* iq, size_t n_frames, int64_t t0_ms, double frame_period_ms, b2s_result* out) {
  if (out) {
    out->n_transmissions = 0;
    out->n_transmissions_total = 0;
    out->n_detect_entries = 0;
    out->n_spectrogram_rows = 0;
  }
  b->prof.pushes += 1;
  {
    int rc = b->grow_capacity();  // a previous push overflowed its per-frame entry lists
    if (rc) return rc;
  }
  const size_t bytes_per_sample = b->cfg.iq_format == B2S_IQ_CS8 ? 2 : 8;
  const size_t stride_bytes = static_cast<size_t>(b->cfg.frame_stride_samples) * bytes_per_sample;
  const bool on_device = (b->cfg.flags & B2S_FLAG_IQ_ON_DEVICE) != 0;
  const int64_t frame0 = b->frames_pushed;  // the band frame of the push's first frame
  // An attached bank reads the push as pieces of up to max_frames frames (frame_stride_samples each), piece j stamped like frame
  // j * max_frames. A synchronous band settles each piece before it moves on; an asynchronous one leaves the newest piece pending.
  auto settle_if_sync = [&]() { return b->bank && !b->async_mode ? bank_settle(b->bank) : 0; };
  if (b->bank && n_frames == 0) {
    const int rc = bank_settle(b->bank);
    if (rc) return rc;
  }
  if (on_device) {
    if (b->bank) CU(cudaEventRecord(b->push_ready, b->stream));  // the bank reads the caller's buffer no earlier than K1 could
    int rc = 0;
    for (size_t done = 0; done < n_frames && !rc;) {
      const size_t chunk = std::min(n_frames - done, static_cast<size_t>(b->max_frames));
      const char* piece = static_cast<const char*>(iq) + done * stride_bytes;
      rc = b->bank ? band_feed(b, piece, frame0 + done, done, chunk, t0_ms, frame_period_ms, b->push_ready, b->bank_read) : 0;
      if (!rc) rc = b->push_chunk(piece, chunk, t0_ms, frame_period_ms, done, out);
      if (!rc) rc = settle_if_sync();
      done += chunk;
    }
    // The caller may reuse `iq` in the band's stream order once the call returns, also when it failed: what follows on `stream` waits
    // for the bank's reads of it (the bank's stream is in order, so its last piece's stage 0 comes after every earlier one's), as it
    // follows K1. The wait comes after the push's own kernels, which therefore never wait for the bank.
    if (b->bank) CU(cudaStreamWaitEvent(b->stream, b->bank_read, 0));
    return rc;
  }
  // Host input: the push is cut into pipeline chunks; the host->device copy of chunk i+1 runs on a second stream
  // while chunk i is in the kernels / tracker (double-buffered staging), so PCIe time hides behind compute (or vice versa).
  // In async mode one chunk per push is enough: the copy of push k+1 already overlaps the work of push k.
  const size_t pipe = b->async_mode ? std::min<size_t>(b->max_frames, std::max<size_t>(n_frames, 1))
                                    : std::max<size_t>(1, std::min<size_t>(b->max_frames, n_frames >= 512 ? (n_frames + 3) / 4 : n_frames));
  if (!b->copy_stream) {
    CU(cudaStreamCreateWithFlags(&b->copy_stream.h, cudaStreamNonBlocking));
    CU(cudaEventCreateWithFlags(&b->copy_done[0].h, cudaEventDisableTiming));
    CU(cudaEventCreateWithFlags(&b->copy_done[1].h, cudaEventDisableTiming));
  }
  if (b->bank && !b->async_mode) {
    // Each piece is staged whole in d_whole: its pipeline chunks are copied to their offsets, and the bank is launched on the piece as
    // soon as the copy of its last chunk has been issued, so that its kernels run beside the band's chunks.
    unsigned char* whole = b->d_whole.p;
    for (size_t p0 = 0; p0 < n_frames; p0 += b->max_frames) {
      const size_t piece = std::min(n_frames - p0, static_cast<size_t>(b->max_frames));
      const size_t part = piece >= 512 ? (piece + 3) / 4 : piece;
      auto copy_part = [&](size_t off, int slot) -> int {
        const size_t bytes = std::min(part, piece - off) * stride_bytes;
        CU(cudaMemcpyAsync(whole + off * stride_bytes, static_cast<const char*>(iq) + (p0 + off) * stride_bytes, bytes, cudaMemcpyHostToDevice, b->copy_stream));
        CU(cudaEventRecord(b->copy_done[slot], b->copy_stream));
        b->prof.h2d_bytes += bytes;
        if (off + part < piece) return 0;
        return band_feed(b, whole, frame0 + p0, p0, piece, t0_ms, frame_period_ms, b->copy_done[slot], b->bank_read);
      };
      // d_whole is overwritten only after the bank has read the previous piece (still pending if the push that fed it failed)
      CU(cudaStreamWaitEvent(b->copy_stream, b->bank_read, 0));
      int rc = copy_part(0, 0);
      if (rc) return rc;
      int slot = 0;
      for (size_t off = 0; off < piece; off += part, slot ^= 1) {
        CU(cudaStreamWaitEvent(b->stream, b->copy_done[slot], 0));
        if (off + part < piece && (rc = copy_part(off + part, slot ^ 1))) return rc;
        if ((rc = b->push_chunk(whole + off * stride_bytes, std::min(part, piece - off), t0_ms, frame_period_ms, p0 + off, out))) return rc;
      }
      if ((rc = bank_settle(b->bank))) return rc;
    }
    return 0;
  }
  const size_t buf_bytes = pipe * stride_bytes;
  for (int i = 0; i < 2; ++i) {
    int rc = b->d_iq[i].alloc(buf_bytes);
    if (rc) return rc;
  }
  auto chunk_len = [&](size_t done) { return std::min(n_frames - done, pipe); };
  auto start_copy = [&](size_t done, int slot) -> int {
    const size_t chunk = chunk_len(done);
    const size_t bytes = push_samples(b->cfg, chunk, b->bank != nullptr) * bytes_per_sample;
    CU(cudaMemcpyAsync(b->d_iq[slot].p, static_cast<const char*>(iq) + done * stride_bytes, bytes, cudaMemcpyHostToDevice, b->copy_stream));
    CU(cudaEventRecord(b->copy_done[slot], b->copy_stream));
    b->prof.h2d_bytes += bytes;
    return 0;
  };
  if (b->async_mode) {
    // staging buffer iq_slot was last read by the K1 of the chunk two chunks ago; iq_prev_use[slot] marks the end of that
    // chunk's kernels on b->stream, and the copy stream waits for it before overwriting the buffer
    for (size_t done = 0; done < n_frames;) {
      const size_t chunk = chunk_len(done);
      const int slot = b->iq_slot;
      CU(cudaStreamWaitEvent(b->copy_stream, b->iq_prev_use[slot], 0));
      if (b->bank) CU(cudaStreamWaitEvent(b->copy_stream, b->bank_prev_use[slot], 0));  // and the bank's stage 0 that read it
      int rc = start_copy(done, slot);
      if (rc) return rc;
      CU(cudaStreamWaitEvent(b->stream, b->copy_done[slot], 0));
      // a chunk is a whole piece here (pipe = max_frames when the push is longer)
      if (b->bank && (rc = band_feed(b, b->d_iq[slot].p, frame0 + done, done, chunk, t0_ms, frame_period_ms, b->copy_done[slot], b->bank_prev_use[slot])))
        return rc;
      rc = b->push_chunk(b->d_iq[slot].p, chunk, t0_ms, frame_period_ms, done, nullptr);
      if (rc) return rc;
      CU(cudaEventRecord(b->iq_prev_use[slot], b->stream));  // K1 (and the rest) of this chunk: the buffer may be overwritten after it
      CU(cudaStreamSynchronize(b->copy_stream));             // the caller may reuse `iq` as soon as the call returns
      b->iq_slot ^= 1;
      done += chunk;
    }
    return 0;
  }
  int slot = 0;
  if (n_frames > 0) {
    int rc = start_copy(0, 0);
    if (rc) return rc;
  }
  for (size_t done = 0; done < n_frames;) {
    const size_t chunk = chunk_len(done);
    CU(cudaStreamWaitEvent(b->stream, b->copy_done[slot], 0));
    if (done + chunk < n_frames) {  // the other staging buffer was released when the previous chunk finished (push_chunk is synchronous)
      int rc = start_copy(done + chunk, slot ^ 1);
      if (rc) return rc;
    }
    int rc = b->push_chunk(b->d_iq[slot].p, chunk, t0_ms, frame_period_ms, done, out);
    if (rc) return rc;
    done += chunk;
    slot ^= 1;
  }
  return 0;
}

int b2s_band_push(b2s_band* b, const void* iq, size_t n_frames, int64_t t0_ms, double frame_period_ms, b2s_result* out) {
  if (!b || (!iq && n_frames)) return fail(B2S_E_INVALID, "NULL argument");
  std::lock_guard<std::mutex> lock(b->mutex);
  CU(cudaSetDevice(b->engine->device));
  if (b->async_mode && out) return fail(B2S_E_INVALID, "with B2S_FLAG_ASYNC results are collected by b2s_band_sync; pass out = NULL to b2s_band_push");
  int rc = 0;
  if (b->autorec.due) {  // an asynchronous band's previous push: decided before this push feeds the bank
    if ((rc = b->drain()) || (rc = band_auto_decide(b))) return rc;
  }
  const int64_t frame0 = b->frames_pushed;
  if ((rc = band_push(b, iq, n_frames, t0_ms, frame_period_ms, out))) return rc;
  if (!b->autorec.on || n_frames == 0) return 0;
  b->autorec.due = true;
  b->autorec.frame = frame0 + static_cast<int64_t>(n_frames) - 1;
  b->autorec.time_ms = host::frame_time(t0_ms, frame_period_ms, n_frames - 1);
  return b->async_mode ? 0 : band_auto_decide(b);
}

int b2s_band_sync(b2s_band* b, b2s_result* out) {
  if (!b) return fail(B2S_E_INVALID, "NULL band");
  std::lock_guard<std::mutex> lock(b->mutex);
  CU(cudaSetDevice(b->engine->device));
  int rc = b->drain();
  if (rc) return rc;
  if ((rc = band_auto_decide(b))) return rc;
  if (b->bank && (rc = bank_settle(b->bank))) return rc;
  if (out) {
    out->n_transmissions_total = static_cast<int32_t>(b->mailbox.size());
    out->n_transmissions = std::min<int32_t>(out->n_transmissions_total, B2S_MAX_TX);
    std::memcpy(out->transmissions, b->mailbox.data(), sizeof(b2s_transmission) * out->n_transmissions);
    out->n_detect_entries = b->stat_entries;
    out->n_spectrogram_rows = b->stat_rows;
  }
  b->stat_entries = 0;
  b->stat_rows = 0;
  return 0;
}

int b2s_band_set_profiling(b2s_band* b, int enable) {
  if (!b) return fail(B2S_E_INVALID, "NULL band");
  std::lock_guard<std::mutex> lock(b->mutex);
  CU(cudaSetDevice(b->engine->device));
  int rc = b->drain();
  if (rc) return rc;
  b->profiling = enable != 0;
  b->profile_ctas = enable >= 2;
  return 0;
}
int b2s_band_get_profile(b2s_band* b, b2s_profile* out, int reset) {
  if (!b || !out) return fail(B2S_E_INVALID, "NULL argument");
  std::lock_guard<std::mutex> lock(b->mutex);
  int rc = b->drain();
  if (rc) return rc;
  *out = b->prof;
  if (reset) b->prof = b2s_profile{};
  return 0;
}

int b2s_band_reset(b2s_band* b) {
  if (!b) return fail(B2S_E_INVALID, "NULL band");
  std::lock_guard<std::mutex> lock(b->mutex);
  CU(cudaSetDevice(b->engine->device));
  return b->reset_buffers();
}

int b2s_band_set_center(b2s_band* b, int32_t center_hz, int32_t lo, int32_t hi) {
  if (!b) return fail(B2S_E_INVALID, "NULL band");
  std::lock_guard<std::mutex> lock(b->mutex);
  int rc = b->drain();
  if (rc) return rc;
  if (center_hz != b->center) {
    b->hist_pieces.clear();  // the history's IQ belongs to the old centre
    b->has_lead = false;     // and so do the samples before the next push
  }
  b->center = center_hz;
  b->tracker.p.center = center_hz;
  b->tracker.p.range_lo = lo;
  b->tracker.p.range_hi = hi;
  return 0;
}

int b2s_band_get_averager(b2s_band* b, float* sum, float* avg, float* ring, int32_t* frames) {
  if (!b) return fail(B2S_E_INVALID, "NULL band");
  std::lock_guard<std::mutex> lock(b->mutex);
  CU(cudaSetDevice(b->engine->device));
  int rc = b->drain();
  if (rc) return rc;
  CU(cudaStreamSynchronize(b->stream));
  const size_t n = b->cfg.fft_size, Y = b->cfg.grouping_y;
  if (sum) CU(cudaMemcpy(sum, b->d_sum[b->sum_cur].p, sizeof(float) * n, cudaMemcpyDeviceToHost));
  if (avg) CU(cudaMemcpy(avg, b->d_avg_last.p, sizeof(float) * n, cudaMemcpyDeviceToHost));
  if (ring) CU(cudaMemcpy(ring, b->d_ring[b->ring_cur].p, sizeof(float) * n * Y, cudaMemcpyDeviceToHost));
  if (frames) *frames = b->avg_frames;
  return 0;
}

int b2s_band_get_noise(b2s_band* b, float* threshold, int32_t* samples, int32_t* ready) {
  if (!b) return fail(B2S_E_INVALID, "NULL band");
  std::lock_guard<std::mutex> lock(b->mutex);
  CU(cudaSetDevice(b->engine->device));
  int rc = b->drain();
  if (rc) return rc;
  CU(cudaStreamSynchronize(b->stream));
  auto it = b->noise.find(b->center);
  if (it == b->noise.end()) {
    if (samples) *samples = 0;
    if (ready) *ready = 0;
    if (threshold) {
      for (int i = 0; i < b->cfg.fft_size; ++i) threshold[i] = -std::numeric_limits<float>::max();
    }
    return 0;
  }
  if (threshold) CU(cudaMemcpy(threshold, it->second.now(), sizeof(float) * b->cfg.fft_size, cudaMemcpyDeviceToHost));
  if (samples) *samples = it->second.samples;
  if (ready) *ready = it->second.ready ? 1 : 0;
  return 0;
}

int b2s_band_get_spectrogram(b2s_band* b, int64_t* times, int32_t* centers, int8_t* rows, int cap, int consume, int* count) {
  if (!b || !count) return fail(B2S_E_INVALID, "NULL argument");
  std::lock_guard<std::mutex> lock(b->mutex);
  int rc = b->drain();
  if (rc) return rc;
  const int M = b->cfg.spectrogram_out_size;
  const int total = static_cast<int>(b->sent.size());
  for (int i = 0; i < total && i < cap; ++i) {
    if (times) times[i] = b->sent[i].time;
    if (centers) centers[i] = b->sent[i].center;
    if (rows) std::memcpy(rows + static_cast<size_t>(i) * M, b->sent[i].row.data(), M);
  }
  *count = total;
  if (consume) b->sent.erase(b->sent.begin(), b->sent.begin() + std::min(total, std::max(cap, 0)));  // only the rows handed out
  return 0;
}

int b2s_band_get_transmissions(b2s_band* b, b2s_transmission* out, int cap, int* count) {
  if (!b || !count) return fail(B2S_E_INVALID, "NULL argument");
  std::lock_guard<std::mutex> lock(b->mutex);
  int rc = b->drain();
  if (rc) return rc;
  const int total = static_cast<int>(b->mailbox.size());
  if (out) std::memcpy(out, b->mailbox.data(), sizeof(b2s_transmission) * std::max(0, std::min(cap, total)));
  *count = total;
  return 0;
}

int b2s_band_get_signals(b2s_band* b, int32_t* keys, int64_t* first, int64_t* last, float* power, int cap, int* count) {
  if (!b || !count) return fail(B2S_E_INVALID, "NULL argument");
  std::lock_guard<std::mutex> lock(b->mutex);
  CU(cudaSetDevice(b->engine->device));
  int rc = b->drain();
  if (rc) return rc;
  b2s_band::HostMap h;  // the map is device resident (K4)
  if ((rc = b->download_state(h))) return rc;
  const int n = static_cast<int>(h.key.size());
  for (int i = 0; i < n && i < cap; ++i) {
    if (keys) keys[i] = h.key[i];
    if (first) first[i] = h.first[i];
    if (last) last[i] = h.last[i];
    if (power) power[i] = h.power[i];
  }
  *count = n;
  return 0;
}

int b2s_band_save_state(b2s_band* b, void* buf, size_t cap, size_t* written) {
  if (!b || !written) return fail(B2S_E_INVALID, "b2s_band_save_state: NULL argument");
  std::lock_guard<std::mutex> lock(b->mutex);
  CU(cudaSetDevice(b->engine->device));
  std::vector<uint8_t> blob;
  const int rc = b->save_state(blob);
  if (rc) return rc;
  return hand_out_state(blob, buf, cap, written, "b2s_band_save_state");
}
int b2s_band_load_state(b2s_band* b, const void* buf, size_t len) {
  if (!b || !buf) return fail(B2S_E_INVALID, "b2s_band_load_state: NULL argument");
  std::lock_guard<std::mutex> lock(b->mutex);
  CU(cudaSetDevice(b->engine->device));
  return b->load_state(buf, len);
}

int b2s_band_record_from(b2s_band* b, int channel, int32_t shift_hz, int64_t frame) {
  const char* who = "b2s_band_record_from";
  if (!b) return fail(B2S_E_INVALID, "%s: NULL band", who);
  std::lock_guard<std::mutex> lock(b->mutex);
  b2s_recorder_bank* k = b->bank;
  if (!k || !k->hist_cap) return fail(B2S_E_INVALID, "%s: the band has no recorder bank that keeps history", who);
  if (channel < 0 || channel >= k->n_ch) return fail(B2S_E_INVALID, "%s: bad channel", who);
  if (b->autorec.on) return fail(B2S_E_STATE, "%s: the band records automatically (b2s_band_set_auto_record)", who);
  long long position = 0;
  int64_t time_ms = 0;
  if (!band_frame_in_history(b, frame, &position, &time_ms))
    return fail(B2S_E_INVALID, "%s: frame %lld is not in the recorder bank's history", who, static_cast<long long>(frame));
  return bank_start_from(k, channel, shift_hz, position, time_ms, who);
}

int b2s_band_set_auto_record(b2s_band* b, int enable, int32_t preroll_frames) {
  const char* who = "b2s_band_set_auto_record";
  if (!b || preroll_frames < 0) return fail(B2S_E_INVALID, "%s: bad argument", who);
  std::lock_guard<std::mutex> lock(b->mutex);
  auto& a = b->autorec;
  if (!enable) {
    a = b2s_band::AutoRecord{};
    return 0;
  }
  b2s_recorder_bank* k = b->bank;
  if (!k) return fail(B2S_E_INVALID, "%s: the band has no recorder bank", who);
  if (a.on) {
    a.preroll = preroll_frames;
    return 0;
  }
  CU(cudaSetDevice(b->engine->device));
  const int rc = bank_settle(k);
  if (rc) return rc;
  for (int i = 0; i < k->n_ch; ++i)
    if (k->ch[i].recording) return fail(B2S_E_STATE, "%s: channel %d of the bank is recording", who, i);
  a.policy = std::make_unique<host::ScanPolicy>(nullptr, nullptr, 0, k->sample_rate, k->n_ch, 0);
  a.key.assign(k->n_ch, 0);
  a.preroll = preroll_frames;
  a.enabled_at = b->frames_pushed;
  a.on = true;
  std::lock_guard<std::mutex> lk(b->qmutex);
  b->start_of.clear();
  b->start_lost_through = -1;
  return 0;
}

int b2s_band_get_auto_record_actions(b2s_band* b, b2s_auto_record_action* out, int cap, int consume, int* count) {
  if (!b || !count) return fail(B2S_E_INVALID, "b2s_band_get_auto_record_actions: NULL argument");
  std::lock_guard<std::mutex> lock(b->mutex);
  hand_out_events(b->auto_actions, out, cap, consume, count);
  return 0;
}

int b2s_band_set_event_log(b2s_band* b, int enable) {
  if (!b) return fail(B2S_E_INVALID, "NULL band");
  std::lock_guard<std::mutex> lock(b->mutex);
  b->event_log = enable != 0;
  if (!b->event_log && !b->autorec.on) {  // the slots' record buffers go once no chunk in flight writes them
    CU(cudaSetDevice(b->engine->device));
    int rc = b->drain();
    if (rc) return rc;
    CU(cudaStreamSynchronize(b->track_stream));
    for (auto& s : b->slots) s.d_log = DevBuf<TrackEvent>();
  }
  return 0;
}

int b2s_band_get_events(b2s_band* b, b2s_signal_event* out, int cap, int consume, int* count) {
  if (!b || !count) return fail(B2S_E_INVALID, "NULL argument");
  std::lock_guard<std::mutex> lock(b->mutex);
  int rc = b->drain();
  if (rc) return rc;
  std::lock_guard<std::mutex> lk(b->qmutex);
  hand_out_events(b->events, out, cap, consume, count);
  return 0;
}

int b2s_band_set_occupancy(b2s_band* b, int enable) {
  if (!b) return fail(B2S_E_INVALID, "b2s_band_set_occupancy: NULL band");
  std::lock_guard<std::mutex> lock(b->mutex);
  b->occupancy = enable != 0;  // read at enqueue time: the pushes after this call
  return 0;
}

int b2s_band_occupancy_centers(b2s_band* b, int32_t* centers_hz, int cap, int* count) {
  if (!b || !count || (!centers_hz && cap > 0)) return fail(B2S_E_INVALID, "b2s_band_occupancy_centers: NULL argument");
  std::lock_guard<std::mutex> lock(b->mutex);
  int i = 0;
  for (const auto& kv : b->occ) {
    if (i < cap) centers_hz[i] = kv.first;
    ++i;
  }
  *count = i;
  return 0;
}

int b2s_band_get_occupancy(b2s_band* b, int32_t center_hz, uint32_t* above_start, uint32_t* above_stop, float* max_db, int64_t* frames,
                           int64_t* detect_frames, int64_t* truncated, int reset) {
  const char* who = "b2s_band_get_occupancy";
  if (!b || !above_start || !above_stop || !max_db || !frames || !detect_frames || !truncated) return fail(B2S_E_INVALID, "%s: NULL argument", who);
  std::lock_guard<std::mutex> lock(b->mutex);
  auto it = b->occ.find(center_hz);
  if (it == b->occ.end()) return fail(B2S_E_INVALID, "%s: no occupancy was counted at centre %d Hz", who, center_hz);
  CU(cudaSetDevice(b->engine->device));
  int rc = b->drain();
  if (rc) return rc;
  CU(cudaStreamSynchronize(b->stream));
  OccupancySlot& o = it->second;
  const size_t n = b->cfg.fft_size;
  CU(cudaMemcpy(above_start, o.above_start.p, sizeof(uint32_t) * n, cudaMemcpyDeviceToHost));
  CU(cudaMemcpy(above_stop, o.above_stop.p, sizeof(uint32_t) * n, cudaMemcpyDeviceToHost));
  CU(cudaMemcpy(max_db, o.max_db.p, sizeof(float) * n, cudaMemcpyDeviceToHost));
  *frames = o.frames;
  *detect_frames = o.detect_frames;
  *truncated = o.truncated;
  if (reset) {
    if ((rc = b->clear_occupancy(o))) return rc;
    CU(cudaStreamSynchronize(b->stream));  // cleared before the call returns, whichever stream the next push uses
  }
  return 0;
}

// ---- stand-alone operators ----
int b2s_averager_create(b2s_engine* e, int size, int group_size, b2s_averager** out) {
  if (!e || !out || size < 1 || group_size < 1) return fail(B2S_E_INVALID, "bad argument");
  CU(cudaSetDevice(e->device));
  auto a = std::make_unique<b2s_averager>();
  a->engine = e;
  a->size = size;
  a->group = group_size;
  int rc = a->sum.alloc(size);
  if (!rc) rc = a->ring[0].alloc(static_cast<size_t>(size) * group_size);
  if (!rc) rc = a->ring[1].alloc(static_cast<size_t>(size) * group_size);
  if (!rc) rc = a->avg.alloc(size);
  if (!rc) rc = a->reset();
  if (rc) return rc;
  *out = a.release();
  return 0;
}
int b2s_averager_destroy(b2s_averager* a) {
  delete a;
  return 0;
}
int b2s_averager_push_many(b2s_averager* a, const float* rows, int count) {
  if (!a || !rows || count < 0) return fail(B2S_E_INVALID, "bad argument");
  if (count == 0) return 0;
  CU(cudaSetDevice(a->engine->device));
  int rc = a->rows.alloc(static_cast<size_t>(count) * a->size);
  if (rc) return rc;
  CU(cudaMemcpy(a->rows.p, rows, sizeof(float) * count * a->size, cudaMemcpyHostToDevice));
  k_averager_push<<<(a->size + 127) / 128, 128>>>(a->rows.p, count, a->size, a->group, a->sum.p, a->ring[a->cur].p, a->ring[a->cur ^ 1].p, a->frames, a->avg.p);
  CU(cudaGetLastError());
  CU(cudaDeviceSynchronize());
  a->cur ^= 1;
  a->frames = std::min(a->frames + count, a->group);
  return 0;
}
int b2s_averager_push(b2s_averager* a, const float* data) { return b2s_averager_push_many(a, data, 1); }
int b2s_averager_reset(b2s_averager* a) {
  if (!a) return fail(B2S_E_INVALID, "NULL averager");
  CU(cudaSetDevice(a->engine->device));
  return a->reset();
}
int b2s_averager_average(b2s_averager* a, float* out) {
  if (!a || !out) return fail(B2S_E_INVALID, "bad argument");
  CU(cudaMemcpy(out, a->avg.p, sizeof(float) * a->size, cudaMemcpyDeviceToHost));
  return 0;
}
int b2s_averager_data(b2s_averager* a, float* out) {
  if (!a || !out) return fail(B2S_E_INVALID, "bad argument");
  CU(cudaMemcpy(out, a->ring[a->cur].p, sizeof(float) * a->size * a->group, cudaMemcpyDeviceToHost));
  return 0;
}
int b2s_averager_sum(b2s_averager* a, float* out, int32_t* frames) {
  if (!a) return fail(B2S_E_INVALID, "bad argument");
  if (out) CU(cudaMemcpy(out, a->sum.p, sizeof(float) * a->size, cudaMemcpyDeviceToHost));
  if (frames) *frames = a->frames;
  return 0;
}

int b2s_average(b2s_engine* e, const float* in, float* out, int size, int group_size, int rows, int exact) {
  if (!e || !in || !out || size < 1 || group_size < 1 || rows < 1) return fail(B2S_E_INVALID, "bad argument");
  CU(cudaSetDevice(e->device));
  DevBuf<float> din, dout;
  int rc = din.alloc(static_cast<size_t>(size) * rows);
  if (!rc) rc = dout.alloc(static_cast<size_t>(size) * rows);
  if (rc) return rc;
  CU(cudaMemcpy(din.p, in, sizeof(float) * size * rows, cudaMemcpyHostToDevice));
  if (exact) {
    k_boxcar_serial<<<(rows + 31) / 32, 32>>>(din.p, dout.p, size, group_size, rows);
  } else {
    dim3 grid((size + 127) / 128, rows);
    k_boxcar<<<grid, 128>>>(din.p, dout.p, size, group_size, rows);
  }
  CU(cudaGetLastError());
  CU(cudaMemcpy(out, dout.p, sizeof(float) * size * rows, cudaMemcpyDeviceToHost));
  return 0;
}

int b2s_psd(b2s_engine* e, const b2s_band_config* cfg, const void* iq, size_t n_frames, float* psd_db, float* power_lin) {
  if (!e || !cfg || !iq || !psd_db || n_frames == 0) return fail(B2S_E_INVALID, "bad argument");
  b2s_band_config c = *cfg;
  if (c.learn_frames < 1) c.learn_frames = 1;
  if (c.grouping_x < 1) c.grouping_x = 1;
  if (c.grouping_y < 1) c.grouping_y = 1;
  if (c.tuning_step_hz < 1) c.tuning_step_hz = 1;
  int rc = validate_config(c);
  if (rc) return rc;
  CU(cudaSetDevice(e->device));
  SpectralTables tables;
  DevBuf<unsigned char> diq;
  DevBuf<float> dpsd, dlin, dpv;
  DevBuf<int> dpi;
  DevBuf<unsigned long long> dpacked;
  const size_t n = c.fft_size;
  const size_t bps = c.iq_format == B2S_IQ_CS8 ? 2 : 8;
  const size_t stride = static_cast<size_t>(c.frame_stride_samples) * bps;
  // overlapping sub-frames: `iq` starts with frame 0's lead-in of N / 2 samples, which K1 reads as frame 0's sub-frame 0 along with
  // the first N / 2 samples of the frame
  const size_t lead = overlapped(c) ? n / 2 * bps : 0;
  const size_t bytes = lead + push_samples(c, n_frames, false) * bps;
  rc = tables.build(c);
  if (!rc) rc = diq.alloc(bytes);
  if (!rc) rc = dpsd.alloc(n_frames * n);
  if (!rc && power_lin) rc = dlin.alloc(n_frames * n);
  if (!rc) rc = dpv.alloc(n_frames);
  if (!rc) rc = dpi.alloc(n_frames);
  if (!rc && tables.split > 1) rc = dpacked.alloc(n_frames);
  if (rc) return rc;
  CU(cudaMemcpy(diq.p, iq, bytes, cudaMemcpyHostToDevice));
  SpectralArgs sa{};
  sa.iq = diq.p + lead;
  sa.frame_stride_bytes = static_cast<long long>(stride);
  sa.n_frames = static_cast<int>(n_frames);
  tables.fill(sa);
  if (lead) sa.sub_lead = diq.p;
  sa.inv_fs = 1.0f / static_cast<float>(c.sample_rate_hz);
  sa.psd_db = dpsd.p;
  sa.power_lin = power_lin ? dlin.p : nullptr;
  sa.peak_index = dpi.p;
  sa.peak_value = dpv.p;
  sa.peak_packed = dpacked.p;
  if ((rc = launch_spectrum(e, c.fft_size, c.iq_format, sa, nullptr))) return rc;
  CU(cudaDeviceSynchronize());
  CU(cudaMemcpy(psd_db, dpsd.p, sizeof(float) * n_frames * n, cudaMemcpyDeviceToHost));
  if (power_lin) CU(cudaMemcpy(power_lin, dlin.p, sizeof(float) * n_frames * n, cudaMemcpyDeviceToHost));
  return 0;
}

// ---- scan policy: Scanner's hop rule + SdrDevice::updateRecordings (scan_policy.h) ----
struct b2s_scan_policy {
  host::ScanPolicy policy;
  b2s_scan_policy(const int32_t* lo, const int32_t* hi, int n, int32_t fs, int rec, int64_t t) : policy(lo, hi, n, fs, rec, t) {}
};
int32_t b2s_get_range_split_sample_rate(int32_t sample_rate_hz) { return host::range_split_sample_rate(sample_rate_hz); }
int b2s_scan_policy_create(const int32_t* lo, const int32_t* hi, int n_ranges, int32_t sample_rate_hz, int n_recorders, int64_t scanning_time_ms, b2s_scan_policy** out) {
  if (!out || n_ranges < 0 || (n_ranges && (!lo || !hi)) || sample_rate_hz <= 0 || n_recorders < 0) return fail(B2S_E_INVALID, "b2s_scan_policy_create: bad argument");
  *out = new b2s_scan_policy(lo, hi, n_ranges, sample_rate_hz, n_recorders, scanning_time_ms > 0 ? scanning_time_ms : 500);
  return 0;
}
int b2s_scan_policy_destroy(b2s_scan_policy* p) {
  delete p;
  return 0;
}
int b2s_scan_policy_ranges(b2s_scan_policy* p, int32_t* lo, int32_t* hi, int cap) {
  if (!p) return fail(B2S_E_INVALID, "NULL policy");
  const auto& r = p->policy.ranges;
  for (size_t i = 0; i < r.size() && static_cast<int>(i) < cap; ++i) {
    if (lo) lo[i] = r[i].first;
    if (hi) hi[i] = r[i].second;
  }
  return static_cast<int>(r.size());
}
int b2s_scan_policy_begin(b2s_scan_policy* p, int64_t now_ms, int32_t* lo, int32_t* hi) {
  if (!p || p->policy.ranges.empty()) return fail(B2S_E_INVALID, "b2s_scan_policy_begin: no ranges to scan");
  p->policy.current = 0;
  p->policy.start = now_ms;
  if (lo) *lo = p->policy.ranges[0].first;
  if (hi) *hi = p->policy.ranges[0].second;
  return 0;
}
int b2s_scan_policy_notify(b2s_scan_policy* p, int64_t now_ms, const b2s_transmission* list, int n, b2s_recorder_action* actions, int cap, int* n_actions, int* hop,
                           int32_t* next_lo, int32_t* next_hi) {
  if (!p || n < 0 || (n && !list) || !n_actions || !hop) return fail(B2S_E_INVALID, "b2s_scan_policy_notify: bad argument");
  std::vector<b2s_recorder_action> acts;
  p->policy.update_recordings(now_ms, list, n, acts);
  for (size_t i = 0; i < acts.size() && static_cast<int>(i) < cap; ++i) actions[i] = acts[i];
  *n_actions = static_cast<int>(acts.size());
  *hop = p->policy.dwell_over(now_ms, n == 0) ? 1 : 0;
  if (*hop) {
    p->policy.hop(now_ms);
    if (next_lo) *next_lo = p->policy.ranges[p->policy.current].first;
    if (next_hi) *next_hi = p->policy.ranges[p->policy.current].second;
  }
  return 0;
}

// ---- recorder chain: rotate -> rational resamplers -> int8 (sources/radio/recorder.cpp:22-40,58-73) ----
int b2s_get_resamplers_factors(int32_t sample_rate_hz, int32_t bandwidth_hz, int threshold, int32_t* interp, int32_t* decim, int cap) {
  if (sample_rate_hz <= 0 || bandwidth_hz <= 0 || threshold < 1) return fail(B2S_E_INVALID, "b2s_get_resamplers_factors: bad argument");
  const auto f = host::resamplers_factors(sample_rate_hz, bandwidth_hz, threshold);
  for (size_t i = 0; i < f.size() && static_cast<int>(i) < cap; ++i) {
    if (interp) interp[i] = f[i].first;
    if (decim) decim[i] = f[i].second;
  }
  return static_cast<int>(f.size());
}
int b2s_recorder_create(b2s_engine* e, int32_t sample_rate_hz, int32_t bandwidth_hz, int iq_format, float iq_scale, int flags, size_t max_samples_per_push, b2s_recorder** out) {
  if (!e || !out || sample_rate_hz <= 0 || bandwidth_hz <= 0 || bandwidth_hz > sample_rate_hz) return fail(B2S_E_INVALID, "b2s_recorder_create: bad argument");
  if (iq_format != B2S_IQ_CS8 && iq_format != B2S_IQ_CF32) return fail(B2S_E_INVALID, "unknown iq_format %d", iq_format);
  *out = nullptr;
  auto r = std::make_unique<b2s_recorder>();
  const int rc = bank_create(e, sample_rate_hz, bandwidth_hz, iq_format, iq_scale, flags, 1, max_samples_per_push, false, r->bank);
  if (rc) return rc;
  *out = r.release();
  return 0;
}
int b2s_recorder_destroy(b2s_recorder* r) {
  if (r) {
    cudaSetDevice(r->bank->engine->device);
    delete r;
  }
  return 0;
}
int b2s_recorder_stages(b2s_recorder* r, int32_t* interp, int32_t* decim, int32_t* n_taps, int cap) {
  if (!r) return fail(B2S_E_INVALID, "NULL recorder");
  const auto& stages = r->bank->stages;
  for (size_t i = 0; i < stages.size() && static_cast<int>(i) < cap; ++i) {
    if (interp) interp[i] = stages[i].interp;
    if (decim) decim[i] = stages[i].decim;
    if (n_taps) n_taps[i] = stages[i].n_taps;
  }
  return static_cast<int>(stages.size());
}
int b2s_recorder_taps(b2s_recorder* r, int stage, float* taps, int cap) {
  if (!r || stage < 0 || stage >= static_cast<int>(r->bank->stages.size()) || !taps) return fail(B2S_E_INVALID, "b2s_recorder_taps: bad argument");
  const auto& h = r->bank->stages[stage].h_taps;
  std::memcpy(taps, h.data(), sizeof(float) * std::min<size_t>(h.size(), std::max(cap, 0)));
  return static_cast<int>(h.size());
}
// Recorder::startRecording (recorder.cpp:58-73): set the rotator to -shift, start from empty buffers (also when already recording)
int b2s_recorder_start(b2s_recorder* r, int32_t shift_hz) {
  if (!r) return fail(B2S_E_INVALID, "NULL recorder");
  start_channel(r->bank->ch[0], rotator_phase_inc(shift_hz, r->bank->sample_rate));
  return 0;
}
int b2s_recorder_stop(b2s_recorder* r) {
  if (!r) return fail(B2S_E_INVALID, "NULL recorder");
  r->bank->ch[0].recording = false;
  return 0;
}
int b2s_recorder_push(b2s_recorder* r, const void* iq, size_t n_samples, int8_t* out_iq, size_t cap_samples, size_t* n_out) {
  if (!r || (!iq && n_samples) || !n_out) return fail(B2S_E_INVALID, "b2s_recorder_push: NULL argument");
  *n_out = 0;
  if (!r->bank->ch[0].recording) return fail(B2S_E_STATE, "b2s_recorder_push: the recorder is not recording (b2s_recorder_start)");
  return bank_push(r->bank.get(), iq, n_samples, 0, out_iq, cap_samples, true, n_out, "b2s_recorder_push");
}

// ---- recorder bank: SdrDevice's recorders on one stream (sdr_device.cpp:39-41,82-144) ----
int b2s_recorder_bank_create(b2s_engine* e, int32_t sample_rate_hz, int32_t bandwidth_hz, int iq_format, float iq_scale, int flags, int n_channels,
                             size_t max_samples_per_push, b2s_recorder_bank** out) {
  if (!e || !out || sample_rate_hz <= 0 || bandwidth_hz <= 0 || bandwidth_hz > sample_rate_hz || n_channels <= 0)
    return fail(B2S_E_INVALID, "b2s_recorder_bank_create: bad argument");
  if (iq_format != B2S_IQ_CS8 && iq_format != B2S_IQ_CF32) return fail(B2S_E_INVALID, "unknown iq_format %d", iq_format);
  *out = nullptr;
  std::unique_ptr<b2s_recorder_bank> k;
  const int rc = bank_create(e, sample_rate_hz, bandwidth_hz, iq_format, iq_scale, flags, n_channels, max_samples_per_push, true, k);
  if (rc) return rc;
  *out = k.release();
  return 0;
}
int b2s_recorder_bank_destroy(b2s_recorder_bank* k) {
  if (k) {
    cudaSetDevice(k->engine->device);
    if (k->band) {  // detach first: the band goes on without the bank
      std::lock_guard<std::mutex> lock(k->band->mutex);
      band_detach(k->band);
    }
    delete k;
  }
  return 0;
}
int b2s_recorder_bank_start(b2s_recorder_bank* k, int channel, int32_t shift_hz) {
  if (!k || channel < 0 || channel >= k->n_ch) return fail(B2S_E_INVALID, "b2s_recorder_bank_start: bad channel");
  if (bank_auto_recorded(k)) return fail(B2S_E_STATE, "b2s_recorder_bank_start: the bank's band records automatically (b2s_band_set_auto_record)");
  const int rc = bank_settle(k);  // a push an asynchronous band left pending belongs to the recording as it was
  if (rc) return rc;
  if (k->ch[channel].recording) return fail(B2S_E_STATE, "b2s_recorder_bank_start: channel %d is already recording", channel);
  start_channel(k->ch[channel], rotator_phase_inc(shift_hz, k->sample_rate));
  return 0;
}
int b2s_recorder_bank_stop(b2s_recorder_bank* k, int channel) {
  if (!k || channel < 0 || channel >= k->n_ch) return fail(B2S_E_INVALID, "b2s_recorder_bank_stop: bad channel");
  if (bank_auto_recorded(k)) return fail(B2S_E_STATE, "b2s_recorder_bank_stop: the bank's band records automatically (b2s_band_set_auto_record)");
  const int rc = bank_settle(k);
  if (rc) return rc;
  auto& c = k->ch[channel];
  if (!c.recording) return fail(B2S_E_STATE, "b2s_recorder_bank_stop: channel %d is not recording", channel);
  c.recording = false;
  c.drop();
  return 0;
}
int b2s_recorder_bank_push(b2s_recorder_bank* k, const void* iq, size_t n_samples, int64_t t0_ms, int8_t* out_iq, size_t cap_samples, size_t* n_out) {
  if (!k || (!iq && n_samples)) return fail(B2S_E_INVALID, "b2s_recorder_bank_push: NULL argument");
  return bank_push(k, iq, n_samples, t0_ms, out_iq, cap_samples, out_iq != nullptr, n_out, "b2s_recorder_bank_push");
}
// Recorder::flush (recorder.cpp:89-97, buffer.h:22-55): the complete chunks, oldest first. Chunk j of a recording is stamped when its
// last sample arrives on the injected clock: start_ms + floor((j + 1) * chunk_samples * 1000 / bandwidth + 0.5)
int b2s_recorder_bank_flush(b2s_recorder_bank* k, int channel, int8_t* chunks, int64_t* times_ms, int cap, int consume, int* count, int* chunk_samples) {
  if (!k || channel < 0 || channel >= k->n_ch || cap < 0) return fail(B2S_E_INVALID, "b2s_recorder_bank_flush: bad argument");
  const int rc = bank_settle(k);
  if (rc) return rc;
  auto& c = k->ch[channel];
  const size_t chunk_bytes = 2 * static_cast<size_t>(k->chunk_samples);
  const int avail = static_cast<int>(std::min<size_t>(c.chunks.size(), std::numeric_limits<int>::max()));
  const int n = std::min(cap, avail);
  if (count) *count = avail;
  if (chunk_samples) *chunk_samples = k->chunk_samples;
  for (int i = 0; i < n; ++i) {
    if (chunks) std::memcpy(chunks + chunk_bytes * i, c.chunks[i].data(), chunk_bytes);
    if (times_ms) {
      const long long num = (c.flushed + i + 1) * static_cast<long long>(k->chunk_samples) * 1000;
      times_ms[i] = c.start_ms + (2 * num + k->bandwidth) / (2 * static_cast<long long>(k->bandwidth));
    }
  }
  if (consume && n > 0) {
    c.chunks.erase(c.chunks.begin(), c.chunks.begin() + n);
    c.flushed += n;
  }
  return 0;
}

int b2s_recorder_bank_save_state(b2s_recorder_bank* k, void* buf, size_t cap, size_t* written) {
  if (!k || !written) return fail(B2S_E_INVALID, "b2s_recorder_bank_save_state: NULL argument");
  std::vector<uint8_t> blob;
  const int rc = bank_save(k, blob);
  if (rc) return rc;
  return hand_out_state(blob, buf, cap, written, "b2s_recorder_bank_save_state");
}
int b2s_recorder_bank_load_state(b2s_recorder_bank* k, const void* buf, size_t len) {
  if (!k || !buf) return fail(B2S_E_INVALID, "b2s_recorder_bank_load_state: NULL argument");
  return bank_load(k, buf, len);
}

int b2s_recorder_bank_set_history(b2s_recorder_bank* k, size_t samples) {
  if (!k) return fail(B2S_E_INVALID, "b2s_recorder_bank_set_history: NULL bank");
  int rc = bank_settle(k);
  if (rc) return rc;
  CU(cudaSetDevice(k->engine->device));
  CU(cudaStreamSynchronize(k->stream));
  const size_t bps = k->raw_bytes();
  if (samples > SIZE_MAX / bps) return fail(B2S_E_NOMEM, "b2s_recorder_bank_set_history: %zu samples do not fit in memory", samples);
  DevBuf<unsigned char> ring;  // allocated before anything changes: a refusal keeps the previous history
  if (samples && (rc = ring.alloc(samples * bps))) {
    cudaGetLastError();  // the failed allocation is not an error of later calls
    return rc;
  }
  k->hist = std::move(ring);
  k->hist_cap = samples;
  k->hist_end = 0;
  ++k->hist_epoch;
  return 0;
}
int b2s_recorder_bank_history(b2s_recorder_bank* k, int64_t* oldest, int64_t* end) {
  if (!k || !oldest || !end) return fail(B2S_E_INVALID, "b2s_recorder_bank_history: NULL argument");
  *oldest = k->hist_oldest();
  *end = k->hist_end;
  return 0;
}
int b2s_recorder_bank_start_from(b2s_recorder_bank* k, int channel, int32_t shift_hz, int64_t position, int64_t start_ms) {
  if (!k || channel < 0 || channel >= k->n_ch) return fail(B2S_E_INVALID, "b2s_recorder_bank_start_from: bad channel");
  if (bank_auto_recorded(k)) return fail(B2S_E_STATE, "b2s_recorder_bank_start_from: the bank's band records automatically (b2s_band_set_auto_record)");
  return bank_start_from(k, channel, shift_hz, position, start_ms, "b2s_recorder_bank_start_from");
}

// self-test of the exact constant division (k_check_div_const above)
int b2s_selftest_div_const(b2s_engine* e, int divisor, uint64_t* mismatches) {
  if (!e || !mismatches) return fail(B2S_E_INVALID, "NULL argument");
  CU(cudaSetDevice(e->device));
  DevBuf<unsigned long long> bad;
  int rc = bad.alloc(1);
  if (rc) return rc;
  CU(cudaMemset(bad.p, 0, sizeof(unsigned long long)));
  switch (divisor) {
    case 2: rc = run_div_check<2>(e, bad.p); break;
    case 3: rc = run_div_check<3>(e, bad.p); break;
    case 5: rc = run_div_check<5>(e, bad.p); break;
    case 7: rc = run_div_check<7>(e, bad.p); break;
    case 9: rc = run_div_check<9>(e, bad.p); break;
    case 11: rc = run_div_check<11>(e, bad.p); break;
    case 13: rc = run_div_check<13>(e, bad.p); break;
    case 15: rc = run_div_check<15>(e, bad.p); break;
    case 17: rc = run_div_check<17>(e, bad.p); break;
    case 19: rc = run_div_check<19>(e, bad.p); break;
    case 21: rc = run_div_check<21>(e, bad.p); break;
    default: rc = fail(B2S_E_INVALID, "no div_const instantiation for divisor %d", divisor);
  }
  if (rc) return rc;
  unsigned long long h = 0;
  CU(cudaMemcpy(&h, bad.p, sizeof(h), cudaMemcpyDeviceToHost));
  *mismatches = h;
  return 0;
}

// ---- host helpers ----
int b2s_get_fft(int32_t sample_rate_hz, int32_t max_step_hz) { return host::fft_size_for(sample_rate_hz, max_step_hz); }
int32_t b2s_get_tuned_frequency(int32_t f, int32_t step) { return host::tuned_frequency(f, step); }
int b2s_get_max_index(const float* data, int size, int index, int group_size) { return host::max_index(data, size, index, group_size); }
int b2s_contains_with_margin(const int* keys, int n_keys, int index, int margin, int* found) {
  std::map<int, char> m;
  for (int i = 0; i < n_keys; ++i) m[keys[i]] = 0;
  return host::key_within_margin(m, index, margin, found) ? 1 : 0;
}
int b2s_most_frequent_value(const int* data, int n) {
  if (!data || n <= 0) return -1;
  return host::most_frequent(std::vector<int>(data, data + n));
}
int b2s_learn_frames_from_ms(int64_t learning_ms, double frame_period_ms) {
  // Noise::add (noise_learner.cpp:23): learning completes on the first frame k with t_k >= t_0 + learning_ms
  size_t k = 0;
  while (host::frame_time(0, frame_period_ms, k) < learning_ms) ++k;
  return static_cast<int>(k + 1);
}
int b2s_decimator_factor(int32_t sample_rate_hz, int32_t fft_size) { return host::decimator_factor(sample_rate_hz, fft_size); }

}  // extern "C"

// ------------------------------------------------------------------------------------------------------------
// Transmission bookkeeping on host rows: the band's tracker behind a DeviceQueries that reads dense host arrays
// ------------------------------------------------------------------------------------------------------------
struct b2s_host_transmission : DeviceQueries {
  b2s_band_config cfg{};
  Tracker tracker;
  std::vector<float> history;  // the last Y rows of q before the current call, oldest -> newest (zeros before any data)
  std::vector<b2s_signal_event> events;  // the tracker's signal event log
  int64_t frames_pushed = 0;
  // current call
  const float* box = nullptr;
  const float* q = nullptr;
  int frames = 0;
  double last_run_ms = 0.0;  // wall time of the last Tracker::run (the bookkeeping alone, without building its inputs)

  int fetch_ring_window(int frame_first, int rows, int bin_lo, int width, float* out) override {
    const int n = cfg.fft_size, Y = cfg.grouping_y;
    for (int r = 0; r < rows; ++r) {
      const int f = frame_first + r;
      float* dst = out + static_cast<size_t>(r) * width;
      const float* src = nullptr;
      if (f >= 0) {
        src = q + static_cast<size_t>(f) * n;
      } else if (Y + f >= 0) {
        src = history.data() + static_cast<size_t>(Y + f) * n;  // f = -1 is the newest row of the previous call
      }
      for (int i = 0; i < width; ++i) dst[i] = src ? src[bin_lo + i] : 0.0f;
    }
    return 0;
  }
  int query_windows(const std::vector<Window>& w, std::vector<std::vector<float>>& values, std::vector<std::vector<int>>& indices) override {
    const int n = cfg.fft_size;
    values.assign(w.size(), {});
    indices.assign(w.size(), {});
    for (size_t i = 0; i < w.size(); ++i) {
      for (int f = w[i].frame_lo; f < w[i].frame_hi; ++f) {
        const float* row = box + static_cast<size_t>(f) * n;
        int best = w[i].bin_lo;
        for (int b = w[i].bin_lo + 1; b <= w[i].bin_hi; ++b) {
          if (row[best] < row[b]) best = b;  // first maximum, collection_utils.h:9-14
        }
        values[i].push_back(row[best]);
        indices[i].push_back(best);
      }
    }
    return 0;
  }
};

extern "C" {

int b2s_host_transmission_create(const b2s_band_config* cfg, b2s_host_transmission** out) {
  if (!cfg || !out) return fail(B2S_E_INVALID, "NULL argument");
  int rc = validate_config(*cfg);
  if (rc) return rc;
  auto h = std::make_unique<b2s_host_transmission>();
  h->cfg = *cfg;
  h->cfg.window_taps = nullptr;
  TrackerParams& p = h->tracker.p;
  p.n = cfg->fft_size;
  p.sample_rate = cfg->sample_rate_hz;
  p.center = cfg->center_hz;
  p.range_lo = cfg->range_lo_hz;
  p.range_hi = cfg->range_hi_hz;
  p.n_ignored = cfg->n_ignored;
  for (int i = 0; i < cfg->n_ignored; ++i) {
    p.ignored_lo[i] = cfg->ignored_lo_hz[i];
    p.ignored_hi[i] = cfg->ignored_hi_hz[i];
  }
  p.group_size = cfg->group_size_bins;
  p.group_y = cfg->grouping_y;
  p.start_level = cfg->start_level;
  p.stop_level = cfg->stop_level;
  p.tuning_step = cfg->tuning_step_hz;
  p.min_time = cfg->min_time_ms;
  p.timeout = cfg->timeout_ms;
  p.max_time = cfg->max_time_ms;
  h->history.assign(static_cast<size_t>(cfg->grouping_y) * cfg->fft_size, 0.0f);  // Averager::reset fills the ring with zeros
  h->tracker.log = &h->events;
  *out = h.release();
  return 0;
}
int b2s_host_transmission_get_events(b2s_host_transmission* h, b2s_signal_event* out, int cap, int consume, int* count) {
  if (!h || !count) return fail(B2S_E_INVALID, "NULL argument");
  hand_out_events(h->events, out, cap, consume, count);
  return 0;
}
int b2s_host_transmission_destroy(b2s_host_transmission* h) {
  delete h;
  return 0;
}
double b2s_host_transmission_last_run_ms(b2s_host_transmission* h) { return h ? h->last_run_ms : 0.0; }
int b2s_host_transmission_reset(b2s_host_transmission* h) {
  if (!h) return fail(B2S_E_INVALID, "NULL handle");
  h->tracker.reset();
  std::fill(h->history.begin(), h->history.end(), 0.0f);
  return 0;
}
int b2s_host_transmission_push(b2s_host_transmission* h, const float* box_rows, const float* q_rows, int n_frames, int64_t t0_ms,
                               double frame_period_ms, int use_watch, int32_t* tx_count, b2s_transmission* tx) {
  if (!h || !box_rows || !q_rows || n_frames < 0) return fail(B2S_E_INVALID, "b2s_host_transmission_push: bad argument");
  const int n = h->cfg.fft_size, Y = h->cfg.grouping_y, T = n_frames;
  const TrackerParams& p = h->tracker.p;
  h->box = box_rows;
  h->q = q_rows;
  h->frames = T;
  // what K2 hands to the tracker: per frame the bins at or above min(start, stop), ascending
  const float level = std::min(p.start_level, p.stop_level);
  std::vector<DetectEntry> entries;
  std::vector<int> begin(T + 1, 0);
  for (int t = 0; t < T; ++t) {
    const float* row = box_rows + static_cast<size_t>(t) * n;
    begin[t] = static_cast<int>(entries.size());
    for (int b = 0; b < n; ++b) {
      if (row[b] >= level) entries.push_back(DetectEntry{b, row[b]});
    }
  }
  begin[T] = static_cast<int>(entries.size());
  // ... and, for the keys alive when the call starts, the window maxima and the "uncovered candidate" flags (k_detect's box warps)
  Tracker::Watch watch;
  std::vector<int> keys, flags;
  std::vector<unsigned int> maxima;
  if (use_watch) {
    for (const auto& kv : h->tracker.signals) {
      if (static_cast<int>(keys.size()) < kMaxWatch) keys.push_back(kv.first);
    }
    const int gh = p.group_size / 2, margin = (p.group_size % 2 == 0) ? gh : gh + 1;
    maxima.assign(static_cast<size_t>(T) * kMaxWatch, 0u);
    flags.assign(T, 0);
    for (int t = 0; t < T; ++t) {
      const float* row = box_rows + static_cast<size_t>(t) * n;
      for (size_t i = 0; i < keys.size(); ++i) {
        float m = -INFINITY;
        for (int b = std::max(0, keys[i] - gh); b <= std::min(n - 1, keys[i] + gh); ++b) m = std::max(m, row[b]);
        maxima[static_cast<size_t>(t) * kMaxWatch + i] = float_to_ordered(m);
      }
      for (int b = 0; b < n && !flags[t]; ++b) {
        if (row[b] < p.start_level) continue;
        bool covered = false;
        for (int key : keys) covered = covered || (b >= key - margin && b <= key + margin);
        if (!covered) flags[t] = 1;
      }
    }
    watch = Tracker::Watch{static_cast<int>(keys.size()), keys.data(), maxima.data(), flags.data()};
  }
  std::vector<Tracker::FrameState> states;
  const DetectEntry* ep = entries.empty() ? nullptr : entries.data();
  h->tracker.log_frame_base = h->frames_pushed;
  h->frames_pushed += T;
  const auto run_t0 = std::chrono::steady_clock::now();
  int rc = h->tracker.run(ep, begin.data(), static_cast<size_t>(T), t0_ms, frame_period_ms, 0, *h, tx_count != nullptr || tx != nullptr, watch, states);
  h->last_run_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - run_t0).count();
  if (rc) return rc;
  if (tx_count) std::fill(tx_count, tx_count + T, 0);
  for (const auto& fs : states) {
    const int total = h->tracker.sorted_transmissions(fs, tx ? tx + static_cast<size_t>(fs.frame) * B2S_MAX_TX : nullptr, tx ? B2S_MAX_TX : 0);
    if (tx_count) tx_count[fs.frame] = total;
  }
  // keep the newest Y rows of q for the next call's getBestIndex look-back
  std::vector<float> next(static_cast<size_t>(Y) * n);
  for (int i = 0; i < Y; ++i) {
    const int f = T - Y + i;
    const float* src = f >= 0 ? q_rows + static_cast<size_t>(f) * n : h->history.data() + static_cast<size_t>(T + i) * n;
    std::memcpy(next.data() + static_cast<size_t>(i) * n, src, sizeof(float) * n);
  }
  h->history.swap(next);
  h->box = h->q = nullptr;
  return 0;
}

// append the object representation of a field (the reference writes through reinterpret_cast on a little-endian host)
static void put_bytes(uint8_t* out, size_t& at, const void* v, size_t n) {
  std::memcpy(out + at, v, n);
  at += n;
}
#define B2S_PUT(type, expr)          \
  do {                               \
    const type field_ = (expr);      \
    put_bytes(out, at, &field_, sizeof(type)); \
  } while (0)

int b2s_pack_spectrogram_message(int64_t time_ms, int32_t center_hz, int32_t sample_rate_hz, const int8_t* row, int size, uint8_t* out, size_t cap,
                                 size_t* written) {
  if (!row || !out || !written || size <= 0) return fail(B2S_E_INVALID, "b2s_pack_spectrogram_message: NULL argument or size <= 0");
  const size_t need = sizeof(uint64_t) + 3 * sizeof(int32_t) + sizeof(uint32_t) + static_cast<size_t>(size);
  *written = need;
  if (cap < need) return fail(B2S_E_INVALID, "spectrogram message needs %zu bytes, buffer holds %zu", need, cap);
  size_t at = 0;
  B2S_PUT(uint64_t, time_ms);
  B2S_PUT(int32_t, center_hz - sample_rate_hz / 2);  // start
  B2S_PUT(int32_t, center_hz + sample_rate_hz / 2);  // stop
  B2S_PUT(int32_t, sample_rate_hz / size);           // step
  B2S_PUT(uint32_t, size);
  std::memcpy(out + at, row, static_cast<size_t>(size));
  return 0;
}

int b2s_pack_transmission_message(int64_t time_ms, int32_t frequency_hz, int32_t sample_rate_hz, const int8_t* iq, int n_samples, uint8_t* out,
                                  size_t cap, size_t* written) {
  if (!out || !written || n_samples < 0 || (n_samples > 0 && !iq)) return fail(B2S_E_INVALID, "b2s_pack_transmission_message: bad argument");
  const size_t header = sizeof(uint64_t) + 2 * sizeof(int32_t) + sizeof(uint32_t), body = 2 * static_cast<size_t>(n_samples);
  *written = header + body;
  if (cap < header + body) return fail(B2S_E_INVALID, "transmission message needs %zu bytes, buffer holds %zu", header + body, cap);
  size_t at = 0;
  B2S_PUT(uint64_t, time_ms);
  B2S_PUT(int32_t, frequency_hz - sample_rate_hz / 2);
  B2S_PUT(int32_t, frequency_hz + sample_rate_hz / 2);
  B2S_PUT(uint32_t, sample_rate_hz);
  for (size_t i = 0; i < body; ++i) out[at + i] = static_cast<uint8_t>(iq[i]) ^ 0x80u;  // offset-binary bytes, data_controller.cpp:38-40
  return 0;
}
#undef B2S_PUT

}  // extern "C"
