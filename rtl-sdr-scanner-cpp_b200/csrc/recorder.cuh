// Recorder DSP chain on the device (SURVEY.md §8(f)#1): what the reference builds per Recorder in sources/radio/recorder.cpp:22-40
//     source -> Blocker -> rotator_cc(phase_inc = 2 pi (-shift) / fs)            recorder.cpp:64
//            -> rational_resampler(f1, f2) for every pair of getResamplersFactors recorder.cpp:29-33, radio_utils.cpp:129-152
//            -> complex_to_interleaved_char(vector, scale 127)                    recorder.cpp:36
// The resampler is GNU Radio's (out of tree): with no taps given it designs a Kaiser low-pass (beta 7, fractional bandwidth 0.4)
// through firdes::low_pass — restated in design_resampler_taps() from GNU Radio 3.10's gr-filter (rational_resampler.cc,
// firdes.cc, window.cc); parity for this part is against a numpy restatement of the same published algorithm (oracle/
// recorder_oracle.py), not against GNU Radio itself (absent here): "parity unpinned" for the taps and the FIR, pinned for the
// factor pairs (the reference's own gtest vectors and its compiled getResamplersFactors).
//
// One stage = one launch of k_resample: y[m] = sum_k h[k] u[m D - k], u = the input upsampled by I with zeros, zero history at
// startRecording. A CTA produces a block of consecutive outputs from one shared-memory tile of inputs; the first stage unpacks the
// int8 / float IQ and applies the rotation while it fills the tile (phase from a 64-bit fixed-point accumulator: exact to 2^-65
// turns per sample, so no drift however long the recording), the last stage packs to int8 (round to nearest even, saturate:
// volk_32f_s32f_convert_8i).
//
// A launch serves up to kLaunchChannels recording channels of a recorder bank (SdrDevice's pool of Recorders on one source,
// sdr_device.cpp:39-41): every channel runs the same stages on the same stream, each with its own shift, start and buffers. CTA b
// works for channel b % n_ch, so the CTAs of all channels that cover the same span of the stream are adjacent in launch order. In
// the first stage they read the same raw samples: one read from HBM, the others from L2. A stand-alone recorder is a bank of one.
// A catch-up (a recording started from the bank's history) runs the same kernels with RingArgs: stage 0 reads the history ring in place.
#pragma once
#include <cmath>
#include <vector>

#include "b2s_device.cuh"

namespace b2s {

constexpr int kResampleThreads = 128;
constexpr int kResampleTile = 6000;  // input samples held in shared memory per CTA (48 KB of float2)
constexpr int kLaunchChannels = 64;  // channels per stage launch (their geometry travels in the kernel parameters)

// one channel's part of a stage launch; indices count from the channel's startRecording
struct StageChan {
  long long g0;                  // index of the first new input sample
  long long m0;                  // index of the first output of this launch
  unsigned long long phase_inc;  // rotation per input sample in turns * 2^64 (first stage; 0 = none)
  int n_in, n_out;
  int slot;                      // the channel's row in the per-channel buffers
};

struct ResampleArgs {
  // input of this launch, per channel: `n_in` new samples at `in`, preceded by `hc` carried samples at `carry`, both offset by
  // slot * in_stride elements (0 for the raw stream, which every channel shares)
  const void* in;
  const void* carry;
  long long in_stride;
  int kind;        // 0: int8 pairs, 1: float pairs (raw IQ); 2: float2 (output of the previous stage)
  float iq_scale;  // int8 only
  int hc;
  const float* taps;
  int n_taps, interp, decim, per_cta;
  float2* out_f;         // next stage's input, or ...
  signed char* out_i8;   // ... the int8 pairs of the last stage; row `slot` starts at slot * out_stride samples
  long long out_stride;
  int n_ch;
  StageChan ch[kLaunchChannels];
};

// Stage 0 of a catch-up: the raw samples come from the bank's history ring. `in` is the ring's base; the carry is the ring itself (the hc
// samples before a piece are the ring slots before it), so `carry` and `in_stride` are unused. Launch channel j's sample g0 sits in ring
// slot ring0[j]. Kept out of ResampleArgs so that the stream pushes' launches and kernels stay as they are.
struct RingArgs : ResampleArgs {
  long long ring_cap;  // capacity in samples
  long long ring0[kLaunchChannels];
};

// what one CTA reads: its channel's view of the stage input
struct StageView {
  const void* in;
  const void* carry;
  long long g0;
  int n_in, hc, kind;
  float iq_scale;
};
__device__ __forceinline__ StageView stage_view(const ResampleArgs& a, const StageChan& c, int) {
  const long long off = static_cast<long long>(c.slot) * a.in_stride * (a.kind == 0 ? 2 : 8);
  return StageView{static_cast<const char*>(a.in) + off, static_cast<const char*>(a.carry) + off, c.g0, c.n_in, a.hc, a.kind, a.iq_scale};
}
struct RingView {
  const void* ring;
  long long cap, at0;  // at0: the ring slot of sample g0
  long long g0;
  int n_in, kind;
  float iq_scale;
};
__device__ __forceinline__ RingView stage_view(const RingArgs& a, const StageChan& c, int j) {
  return RingView{a.in, a.ring_cap, a.ring0[j], c.g0, c.n_in, a.kind, a.iq_scale};
}

// sample g of this stage's input stream, before the rotator (zero before startRecording)
__device__ __forceinline__ float2 resample_raw(const StageView& a, long long g) {
  if (g < 0) return make_float2(0.0f, 0.0f);
  const long long rel = g - a.g0;
  if (rel >= a.n_in) return make_float2(0.0f, 0.0f);  // past the newest sample (the last CTA of k_decimate_poly stages a whole tile; only unused outputs see these)
  if (a.kind == 0) {
    const char2* p = rel >= 0 ? static_cast<const char2*>(a.in) + rel : static_cast<const char2*>(a.carry) + (a.hc + rel);
    const char2 s = *p;
    return make_float2(static_cast<float>(s.x) * a.iq_scale, static_cast<float>(s.y) * a.iq_scale);
  }
  const float2* p = rel >= 0 ? static_cast<const float2*>(a.in) + rel : static_cast<const float2*>(a.carry) + (a.hc + rel);
  return *p;
}
// The same from the ring: every sample read is at [piece start - hc, end of the history), inside the history's window of ring_cap samples
// that also holds the piece's start, so rel lies in (-cap, cap) and one wrap in either direction takes the slot modulo the capacity.
__device__ __forceinline__ float2 resample_raw(const RingView& a, long long g) {
  if (g < 0) return make_float2(0.0f, 0.0f);
  const long long rel = g - a.g0;
  if (rel >= a.n_in) return make_float2(0.0f, 0.0f);
  long long i = a.at0 + rel;
  if (i < 0) i += a.cap;
  else if (i >= a.cap) i -= a.cap;
  if (a.kind == 0) {
    const char2 s = static_cast<const char2*>(a.ring)[i];
    return make_float2(static_cast<float>(s.x) * a.iq_scale, static_cast<float>(s.y) * a.iq_scale);
  }
  return static_cast<const float2*>(a.ring)[i];
}
// exp(i * 2 pi * turns), turns as a 64-bit binary fraction
__device__ __forceinline__ float2 rotor_of(unsigned long long turns64) {
  float sn, cs;
  sincospif(static_cast<float>(static_cast<unsigned int>(turns64 >> 32)) * (2.0f / 4294967296.0f), &sn, &cs);
  return make_float2(cs, sn);
}

template <class View>
__device__ __forceinline__ float2 resample_input(const View& a, unsigned long long phase_inc, long long g) {
  if (g < 0) return make_float2(0.0f, 0.0f);  // before startRecording: zero history
  float2 v = resample_raw(a, g);
  if (a.kind == 2) return v;
  if (phase_inc) {  // rotator_cc: x[n] * exp(i * phase_inc * n)
    const unsigned long long ph = static_cast<unsigned long long>(g) * phase_inc;  // turns * 2^64, modulo 1 turn by overflow
    float sn, cs;
    sincospif(static_cast<float>(static_cast<unsigned int>(ph >> 32)) * (2.0f / 4294967296.0f), &sn, &cs);
    v = make_float2(fmaf(v.x, cs, -v.y * sn), fmaf(v.x, sn, v.y * cs));
  }
  return v;
}

// Args: ResampleArgs, or RingArgs for stage 0 of a catch-up
template <class Args>
__global__ void __launch_bounds__(kResampleThreads) k_resample(const __grid_constant__ Args a) {
  extern __shared__ float2 tile[];
  const int tid = threadIdx.x;
  const int j = blockIdx.x % a.n_ch;
  const StageChan& c = a.ch[j];
  const int cta = blockIdx.x / a.n_ch;
  const auto v = stage_view(a, c, j);
  const long long mb = c.m0 + static_cast<long long>(cta) * a.per_cta;  // first output of this CTA
  const int count = min(a.per_cta, c.n_out - cta * a.per_cta);
  if (count <= 0) return;
  // inputs needed: u indices [mb D - (n_taps - 1), (mb + count - 1) D]  ->  x indices [floor(lo / I) .. floor(hi / I)]
  const long long u_lo = mb * a.decim - (a.n_taps - 1), u_hi = (mb + count - 1) * a.decim;
  const long long x_lo = u_lo >= 0 ? u_lo / a.interp : -((-u_lo + a.interp - 1) / a.interp), x_hi = u_hi / a.interp;
  const int span = static_cast<int>(x_hi - x_lo + 1);
  for (int i = tid; i < span; i += kResampleThreads) tile[i] = resample_input(v, c.phase_inc, x_lo + i);
  __syncthreads();
  for (int o = tid; o < count; o += kResampleThreads) {
    const long long m = mb + o;
    const long long j0 = m * a.decim;  // u index of tap 0
    // taps k with (j0 - k) % I == 0: k = k0 + I q
    const int k0 = static_cast<int>(j0 % a.interp);
    long long x = (j0 - k0) / a.interp - x_lo;  // tile index of the sample under tap k0
    float re = 0.0f, im = 0.0f;
    for (int k = k0; k < a.n_taps; k += a.interp, --x) {
      const float h = __ldg(a.taps + k);
      const float2 v = tile[x];
      re = fmaf(h, v.x, re);
      im = fmaf(h, v.y, im);
    }
    const long long oi = c.slot * a.out_stride + (m - c.m0);
    if (a.out_i8) {  // complex_to_interleaved_char(vector, 127): rint, saturate
      const int r = max(-128, min(127, __float2int_rn(re * 127.0f))), q = max(-128, min(127, __float2int_rn(im * 127.0f)));
      a.out_i8[2 * oi] = static_cast<signed char>(r);
      a.out_i8[2 * oi + 1] = static_cast<signed char>(q);
    } else {
      a.out_f[oi] = make_float2(re, im);
    }
  }
}

// Decimating stages (interpolation 1 — every stage the reference's factor pairs produce for a recorder below the device rate) in
// polyphase form: k = q D + p,   y[m] = sum_p sum_q h[q D + p] x[(m - q) D - p].
// A CTA produces kPolyOut consecutive outputs. It walks the D phases; for phase p it stages x_p[n] = x[(m0 - (Q - 1) + n) D - p]
// (rotated on the way in: one sincospif per thread and phase, then a constant rotor per step — the 64-bit phase accumulator still
// anchors every phase of every CTA, so there is no drift) into one of two shared tiles, and every thread accumulates kPolyR
// consecutive outputs from a register window of kPolyR + Q - 1 samples of that phase: 33 x 9 complex multiply-adds per 41 shared
// loads and 33 broadcast tap loads, against one shared load and one global tap load per multiply-add in k_resample. The lane stride
// of the window (9 samples = 18 words) is conflict-free for 8-byte accesses.
constexpr int kPolyQ = 33;        // taps per phase: GNU Radio's default design has ceil(n_taps / D) = 33 for every D
constexpr int kPolyR = 9;         // outputs per thread
constexpr int kPolyThreads = 128;
constexpr int kPolyOut = kPolyThreads * kPolyR;   // outputs per CTA
constexpr int kPolyTile = kPolyOut + kPolyQ - 1;  // samples of one phase a CTA needs

template <class Args>
__global__ void __launch_bounds__(kPolyThreads) k_decimate_poly(const __grid_constant__ Args a, const float* __restrict__ taps_pq /* [D][kPolyQ]: h[q D + p], zero padded */) {
  __shared__ float2 tile[2][kPolyTile];
  __shared__ float htap[2][kPolyQ];
  const int tid = threadIdx.x;
  const int D = a.decim;
  const int j = blockIdx.x % a.n_ch;
  const StageChan& c = a.ch[j];
  const int cta = blockIdx.x / a.n_ch;
  const auto sv = stage_view(a, c, j);
  const long long mb = c.m0 + static_cast<long long>(cta) * kPolyOut;  // first output of this CTA
  const int count = min(kPolyOut, c.n_out - cta * kPolyOut);
  if (count <= 0) return;
  const unsigned long long phase_inc = c.phase_inc;
  const bool rotate = a.kind != 2 && phase_inc != 0;
  // rotor of kPolyThreads tile steps = kPolyThreads * D input samples
  const float2 rstep = rotate ? rotor_of(static_cast<unsigned long long>(kPolyThreads) * static_cast<unsigned long long>(D) * phase_inc) : make_float2(1.0f, 0.0f);
  auto fill = [&](int p, int buf) {
    long long g = (mb - (kPolyQ - 1) + tid) * D - p;  // input sample under tile element n = tid
    float2 r = rotate ? rotor_of(static_cast<unsigned long long>(g) * phase_inc) : make_float2(1.0f, 0.0f);
    for (int n = tid; n < kPolyTile; n += kPolyThreads, g += static_cast<long long>(kPolyThreads) * D) {
      float2 v = resample_raw(sv, g);
      if (rotate) {
        v = make_float2(fmaf(v.x, r.x, -v.y * r.y), fmaf(v.x, r.y, v.y * r.x));
        r = make_float2(fmaf(r.x, rstep.x, -r.y * rstep.y), fmaf(r.x, rstep.y, r.y * rstep.x));
      }
      tile[buf][n] = v;
    }
    if (tid < kPolyQ) htap[buf][tid] = taps_pq[p * kPolyQ + tid];
  };
  float2 acc[kPolyR];
#pragma unroll
  for (int r = 0; r < kPolyR; ++r) acc[r] = make_float2(0.0f, 0.0f);
  fill(0, 0);
  __syncthreads();
  for (int p = 0; p < D; ++p) {
    if (p + 1 < D) fill(p + 1, (p + 1) & 1);
    const float2* w = tile[p & 1] + tid * kPolyR;  // w[j] = x_p[tid R + j]; output r, tap q reads j = r + (Q - 1) - q
    float2 win[kPolyR + kPolyQ - 1];
#pragma unroll
    for (int j = 0; j < kPolyR + kPolyQ - 1; ++j) win[j] = w[j];
    const float* h = htap[p & 1];
#pragma unroll
    for (int q = 0; q < kPolyQ; ++q) {
      const float hq = h[q];
#pragma unroll
      for (int r = 0; r < kPolyR; ++r) {
        acc[r].x = fmaf(hq, win[r + kPolyQ - 1 - q].x, acc[r].x);
        acc[r].y = fmaf(hq, win[r + kPolyQ - 1 - q].y, acc[r].y);
      }
    }
    __syncthreads();  // tile[(p + 1) & 1] is filled, tile[p & 1] is free
  }
#pragma unroll
  for (int r = 0; r < kPolyR; ++r) {
    const int o = tid * kPolyR + r;
    if (o < count) {
      const long long oi = c.slot * a.out_stride + (mb + o - c.m0);
      if (a.out_i8) {  // complex_to_interleaved_char(vector, 127): rint, saturate
        const int re = max(-128, min(127, __float2int_rn(acc[r].x * 127.0f))), im = max(-128, min(127, __float2int_rn(acc[r].y * 127.0f)));
        reinterpret_cast<char2*>(a.out_i8)[oi] = make_char2(static_cast<signed char>(re), static_cast<signed char>(im));
      } else {
        a.out_f[oi] = acc[r];
      }
    }
  }
}

// ---- host side: GNU Radio's default resampler taps ----
namespace host {

inline double izero(double x) {  // gr::fft::window: modified Bessel function I0 by its power series (IzeroEPSILON 1e-21)
  double sum = 1.0, u = 1.0, n = 1.0;
  const double halfx = x / 2.0;
  do {
    double t = halfx / n;
    n += 1.0;
    t *= t;
    u *= t;
    sum += u;
  } while (u >= 1e-21 * sum);
  return sum;
}

// rational_resampler's design_resampler_filter(interpolation, decimation, fractional_bw = 0.4) -> firdes::low_pass(gain = I, fs = I,
// cutoff = mid_transition_band, transition width, WIN_KAISER, beta = 7), taps as float
inline std::vector<float> design_resampler_taps(unsigned interpolation, unsigned decimation, float fractional_bw = 0.4f) {
  const float beta = 7.0f, halfband = 0.5f;
  const float rate = static_cast<float>(interpolation) / static_cast<float>(decimation);
  float trans_width, mid;
  if (rate >= 1.0f) {
    trans_width = halfband - fractional_bw;
    mid = halfband - trans_width / 2.0f;
  } else {
    trans_width = rate * (halfband - fractional_bw);
    mid = rate * halfband - trans_width / 2.0f;
  }
  const double gain = interpolation, fs = interpolation, cutoff = mid, tw = trans_width;
  const double atten = beta / 0.1102 + 8.7;  // window::max_attenuation(WIN_KAISER, beta)
  int ntaps = static_cast<int>(atten * fs / (22.0 * tw));
  if ((ntaps & 1) == 0) ntaps++;
  std::vector<float> w(ntaps), taps(ntaps);
  {  // window::kaiser(ntaps, beta)
    const double ibeta = 1.0 / izero(beta), inm1 = 1.0 / static_cast<double>(ntaps - 1);
    for (int i = 0; i < ntaps; ++i) {
      const double t = 2 * i * inm1 - 1;
      w[i] = static_cast<float>(izero(beta * std::sqrt(1.0 - t * t)) * ibeta);
    }
  }
  const int M = (ntaps - 1) / 2;
  const double fwT0 = 2 * M_PI * cutoff / fs;
  for (int n = -M; n <= M; ++n) {
    if (n == 0) taps[n + M] = static_cast<float>(fwT0 / M_PI * w[n + M]);
    else taps[n + M] = static_cast<float>(std::sin(n * fwT0) / (n * M_PI) * w[n + M]);
  }
  double fmax = taps[0 + M];
  for (int n = 1; n <= M; ++n) fmax += 2 * taps[n + M];
  const double g = gain / fmax;
  for (int i = 0; i < ntaps; ++i) taps[i] = static_cast<float>(taps[i] * g);
  return taps;
}

// getPrimeFactors / split / getResamplersFactors — sources/utils/radio_utils.cpp:9-35,105-152
inline std::vector<int> prime_factors(int n) {
  if (n == 1) return {1};
  std::vector<int> f;
  while (n % 2 == 0) {
    f.push_back(2);
    n /= 2;
  }
  for (int i = 3; i <= std::sqrt(n); i += 2) {
    while (n % i == 0) {
      f.push_back(i);
      n /= i;
    }
  }
  if (n > 2) f.push_back(n);
  return f;
}
inline void split_factor(int value, std::vector<int>& out, int threshold) {
  if (threshold < value && prime_factors(value).size() != 1) {
    int f1 = 1, f2 = value;
    for (int i = static_cast<int>(std::sqrt(value)); i >= 1; --i) {
      if (value % i == 0) {
        f1 = i;
        f2 = value / i;
        break;
      }
    }
    if (threshold < f1) split_factor(f1, out, threshold); else out.push_back(f1);
    if (threshold < f2) split_factor(f2, out, threshold); else out.push_back(f2);
  } else {
    out.push_back(value);
  }
}
inline long long gcd_ll(long long a, long long b) {
  while (b) {
    const long long t = a % b;
    a = b;
    b = t;
  }
  return a;
}
inline std::vector<std::pair<int, int>> resamplers_factors(int32_t sample_rate, int32_t bandwidth, int threshold) {
  const int g = static_cast<int>(gcd_ll(sample_rate, bandwidth));
  std::vector<int> left, right;
  split_factor(bandwidth / g, left, threshold);
  split_factor(sample_rate / g, right, threshold);
  while (left.size() < right.size()) left.push_back(1);
  while (right.size() < left.size()) right.push_back(1);
  std::sort(left.begin(), left.end());
  std::sort(right.begin(), right.end());
  std::vector<std::pair<int, int>> r;
  for (size_t i = 0; i < left.size(); ++i) r.push_back({left[i], right[i]});
  return r;
}

}  // namespace host
}  // namespace b2s
