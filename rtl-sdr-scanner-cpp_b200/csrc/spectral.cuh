// K1 — the frame-parallel half of the hot path: int8-IQ unpack -> window -> N-point FFT -> fftshift -> |X|^2/fs -> dB,
// plus the per-frame first-maximum of the raw PSD row.
//
// Replaces, per frame, the reference's Decimator::work (sources/radio/blocks/decimator.h:11-22), the out-of-tree
// gr::fft::fft_v<gr_complex,true>(N, window::hamming(N), shift=true) (call site sources/radio/sdr_device.cpp:164),
// PSD::work (sources/radio/blocks/psd.cpp:11-22) and the argmax scan of NoiseLearner::work
// (sources/radio/blocks/noise_learner.cpp:53-59).
//
// Shape: one persistent CTA per SM slot; each CTA walks frames blockIdx.x, +gridDim.x, ...  The int8 frame (2N bytes)
// is staged into shared memory by ONE bulk async copy (TMA, cp.async.bulk + mbarrier) that is issued as soon as the
// previous frame's first pass has consumed the buffer, so the copy of frame f+1 overlaps passes 2.. of frame f.
// The FFT is a Stockham autosort (decimation in time, twiddle-then-butterfly) with radix-16/8/4/2 passes held in
// registers (32 complex values per thread); passes exchange through one padded complex buffer in shared memory.
// The last pass leaves thread b holding bins b + m*N/R, so dB rows leave the SM as fully coalesced 128-byte stores.
#pragma once
#include "b2s_device.cuh"

namespace b2s {

// ------------------------------------------------------------------------------------------------------------
// small DFTs in registers (forward transform, exp(-2 pi i k n / R)), natural-order in-place
// ------------------------------------------------------------------------------------------------------------
// C is the complex value type: float2 (scalar fp32 instructions) or cpk (packed two-wide instructions, b2s_device.cuh); the
// operations are the same IEEE operations either way.
template <int R>
struct Dft;

template <>
struct Dft<1> {
  template <typename C>
  __device__ __forceinline__ static void run(C*) {}
};
template <>
struct Dft<2> {
  template <typename C>
  __device__ __forceinline__ static void run(C* v) {
    const C a = v[0], b = v[1];
    v[0] = cadd(a, b);
    v[1] = csub(a, b);
  }
};
template <>
struct Dft<4> {
  template <typename C>
  __device__ __forceinline__ static void run(C* v) {
    const C t0 = cadd(v[0], v[2]), t1 = csub(v[0], v[2]);
    const C t2 = cadd(v[1], v[3]), t3 = mul_mi(csub(v[1], v[3]));
    v[0] = cadd(t0, t2);
    v[1] = cadd(t1, t3);
    v[2] = csub(t0, t2);
    v[3] = csub(t1, t3);
  }
};

// multiply by W_R^j = exp(-2 pi i j / R), j a compile-time constant after unrolling (R in {8, 16})
template <int R, typename C>
__device__ __forceinline__ C mul_w(C a, int j) {
  constexpr float C1 = 0.92387953251128674f, S1 = 0.38268343236508977f, H = 0.70710678118654752f;
  const int j16 = j * (16 / R);  // express as a 16th root
  switch (j16 & 15) {
    case 0: return a;
    case 4: return mul_mi(a);
    case 8: return cneg(a);
    case 12: return cneg(mul_mi(a));
    case 2: return cscale(cadd(a, mul_mi(a)), H);         // ((a.x + a.y) H, (a.y - a.x) H)
    case 6: return cscale(csub(mul_mi(a), a), H);         // ((a.y - a.x) H, -(a.x + a.y) H)
    case 10: return cscale(cneg(cadd(a, mul_mi(a))), H);  // (-(a.x + a.y) H, (a.x - a.y) H)
    case 14: return cscale(csub(a, mul_mi(a)), H);        // ((a.x - a.y) H, (a.x + a.y) H)
    case 1: return cmul(a, make_float2(C1, -S1));
    case 3: return cmul(a, make_float2(S1, -C1));
    case 5: return cmul(a, make_float2(-S1, -C1));
    case 7: return cmul(a, make_float2(-C1, -S1));
    case 9: return cmul(a, make_float2(-C1, S1));
    case 11: return cmul(a, make_float2(-S1, C1));
    case 13: return cmul(a, make_float2(S1, C1));
    default: return cmul(a, make_float2(C1, S1));  // 15
  }
}

// Cooley-Tukey R = 4 * (R/4): n = N2*n1 + n2, k = k1 + 4*k2
template <int R>
struct Dft {
  template <typename C>
  __device__ __forceinline__ static void run(C* v) {
    constexpr int N2 = R / 4;
    C y[N2][4];
#pragma unroll
    for (int n2 = 0; n2 < N2; ++n2) {
      C a[4];
#pragma unroll
      for (int n1 = 0; n1 < 4; ++n1) a[n1] = v[N2 * n1 + n2];
      Dft<4>::run(a);
#pragma unroll
      for (int k1 = 0; k1 < 4; ++k1) y[n2][k1] = mul_w<R>(a[k1], n2 * k1);
    }
#pragma unroll
    for (int k1 = 0; k1 < 4; ++k1) {
      C b[N2];
#pragma unroll
      for (int n2 = 0; n2 < N2; ++n2) b[n2] = y[n2][k1];
      Dft<N2>::run(b);
#pragma unroll
      for (int k2 = 0; k2 < N2; ++k2) v[k1 + 4 * k2] = b[k2];
    }
  }
};

// ------------------------------------------------------------------------------------------------------------
// pass plans
// ------------------------------------------------------------------------------------------------------------
template <int N>
struct FftPlanT;  // radices R0..R3 (1 = unused), elements per thread E
template <> struct FftPlanT<256>   { static constexpr int R0 = 8,  R1 = 8,  R2 = 4,  R3 = 1, E = 8;  };  // E = 8 keeps a full warp (32 threads)
template <> struct FftPlanT<512>   { static constexpr int R0 = 16, R1 = 8,  R2 = 4,  R3 = 1, E = 16; };
template <> struct FftPlanT<1024>  { static constexpr int R0 = 16, R1 = 16, R2 = 4,  R3 = 1, E = 16; };
template <> struct FftPlanT<2048>  { static constexpr int R0 = 16, R1 = 16, R2 = 8,  R3 = 1, E = 16; };
template <> struct FftPlanT<4096>  { static constexpr int R0 = 16, R1 = 16, R2 = 16, R3 = 1, E = 32; };
template <> struct FftPlanT<8192>  { static constexpr int R0 = 16, R1 = 16, R2 = 8,  R3 = 4, E = 32; };
template <> struct FftPlanT<16384> { static constexpr int R0 = 16, R1 = 16, R2 = 16, R3 = 4, E = 32; };

// padded index into the exchange buffer: one float2 of padding per 16 keeps both the strided stores of the first
// pass and the unit-stride loads of every pass on distinct bank pairs
__device__ __forceinline__ int pad16(int i) { return i + (i >> 4); }

template <int N>
__host__ __device__ constexpr int exchange_elems() { return N + (N >> 4); }

// Twiddles. Pass p (radix R, product of the previous radices P) multiplies input m of butterfly b by
// W_{P*R}^{k*m}, k = b mod P. Each pass has its own compact table laid out [m-1][k] so that consecutive lanes
// (consecutive k) read consecutive entries: conflict-free from shared memory, fully coalesced from global memory.
// Tables of up to kSmemTwiddleMax entries live in shared memory; the (large) table of the last pass stays in global
// memory / L2 (3 coalesced loads per radix-4 butterfly).
constexpr int kSmemTwiddleMax = 4096;
template <int R, int P>
__host__ __device__ constexpr int twiddle_entries() { return P > 1 ? (R - 1) * P : 0; }
template <int R, int P>
__host__ __device__ constexpr bool twiddle_in_smem() { return P > 1 && (R - 1) * P <= kSmemTwiddleMax; }

template <int N>
struct TwiddleLayout {
  using PL = FftPlanT<N>;
  static constexpr int P1 = PL::R0, P2 = PL::R0 * PL::R1, P3 = PL::R0 * PL::R1 * PL::R2;
  static constexpr int E1 = twiddle_entries<PL::R1, P1>();
  static constexpr int E2 = PL::R2 > 1 ? twiddle_entries<PL::R2, P2>() : 0;
  static constexpr int E3 = PL::R3 > 1 ? twiddle_entries<PL::R3, P3>() : 0;
  static constexpr int O1 = 0, O2 = E1, O3 = E1 + E2, TOTAL = E1 + E2 + E3;  // offsets into the global table
  static constexpr bool S1 = twiddle_in_smem<PL::R1, P1>();
  static constexpr bool S2 = PL::R2 > 1 && twiddle_in_smem<PL::R2, P2>();
  static constexpr bool S3 = PL::R3 > 1 && twiddle_in_smem<PL::R3, P3>();
  static constexpr int SO1 = 0, SO2 = S1 ? E1 : 0, SO3 = SO2 + (S2 ? E2 : 0);  // offsets into the shared copy
  static constexpr int SMEM = SO3 + (S3 ? E3 : 0);
};

// input modes
constexpr int kModeCs8Tma = 0;     // int8 IQ staged through shared memory by bulk async copy (16-byte aligned frames)
constexpr int kModeCs8Direct = 1;  // int8 IQ read straight from global memory (unaligned frames)
constexpr int kModeCf32 = 2;       // float IQ read straight from global memory

struct SpectralArgs {
  const void* iq;               // frame k starts at iq + k * frame_stride_bytes
  long long frame_stride_bytes;
  int n_frames;
  const float* wscale;          // [N] window[n] * iq_scale (CS8) or window[n] (CF32)
  const float2* twiddle;        // per-pass compact tables, TwiddleLayout<N>
  float inv_fs;                 // 1 / (float)sample_rate
  float* psd_db;                // [n_frames][N] raw PSD rows (fftshifted)
  float* power_lin;             // optional [n_frames][N] |X|^2 / fs (only read by the DEBUG instantiation)
  int* peak_index;              // [n_frames]
  float* peak_value;            // [n_frames]
  // per-frame counters of the NEXT kernel on the stream (K2's slot_count and cand_flag, its max_count scalar), zeroed here so that no
  // memset sits between K1 and K2 on the band's stream (three tiny stream operations per push otherwise); any may be null
  int* zero_per_frame[2];
  int* zero_scalar;
  // ---- k_spectrum3 only ----
  int* work_counter;            // [2] {next work item, CTAs finished}: dynamic work distribution; both zero between launches
  int reserve_sms;              // SMs the persistent grid leaves free (for the band's K4, which runs beside the next push's K1)
  // split mode, N = S * 16384 (S = 2..16): CTA-items (frame, c) each produce the bins k = S k' + c of one frame
  int split;                    // S (1 = off)
  const float2* split_tw;       // [S][16384]  W_N^(n' c)
  const float2* split_ws;       // [S]         W_S^j
  unsigned long long* peak_packed;  // [n_frames], zeroed before the launch: max over the S classes of (ordered(value) << 32 | ~index)
  // ---- sub-frames (the SUB instantiations only, B2S_FLAG_SUBFRAME_*) ----
  int sub_r;                    // sub-frames per frame, >= 2: sub-frame j of frame k starts at
                                //   iq + k * frame_stride_bytes + sub_off_bytes + j * sub_step_bytes
  int sub_max;                  // reduction over the sub-frames' |X|^2/fs: 0 = mean (sum in order, then / count), 1 = maximum
  long long sub_step_bytes;     // N samples back to back; N / 2 samples with B2S_FLAG_SUBFRAME_OVERLAP
  long long sub_off_bytes;      // 0; -N / 2 samples with the overlap (sub-frame 0 straddles the previous frame's end)
  // overlap: frame 0's sub-frame 0 is read from sub_lead (N contiguous samples: the lead-in, then the launch's first N / 2),
  // never from before iq; sub_first = 1 drops it (no lead-in) and frame 0 folds sub-frames 1 ... sub_r - 1
  const void* sub_lead;
  int sub_first;
};

// The first sub-frame a frame folds: 0, or a.sub_first for frame 0
__device__ __forceinline__ int sub_begin(const SpectralArgs& a, long long frame) { return frame == 0 ? a.sub_first : 0; }
// First sample of sub-frame `sub` of `frame`
__device__ __forceinline__ const char* sub_src(const SpectralArgs& a, const char* base, long long frame, int sub) {
  if (frame == 0 && sub == 0 && a.sub_lead) return static_cast<const char*>(a.sub_lead);
  return base + frame * a.frame_stride_bytes + a.sub_off_bytes + static_cast<long long>(sub) * a.sub_step_bytes;
}
// One sub-frame's |X|^2/fs folded into the frame's partial: MEAN adds in sub-frame order, MAX keeps the larger. On the last
// sub-frame the caller divides the mean by the number of sub-frames folded.
__device__ __forceinline__ float sub_fold(float part, float pw, bool first, int sub_max) {
  if (first) return pw;
  return sub_max ? fmaxf(part, pw) : __fadd_rn(part, pw);
}
__device__ __forceinline__ float sub_finish(float acc, const SpectralArgs& a, int count) {
  return a.sub_max ? acc : __fdiv_rn(acc, static_cast<float>(count));
}

// tw points at this pass's [m-1][k] table (shared or global)
template <int N, int R, int P, int E, int T>
__device__ __forceinline__ void pass_twiddle_butterfly(float2 (&v)[E], const float2* __restrict__ tw, int tid) {
  constexpr int BPT = E / R;
#pragma unroll
  for (int u = 0; u < BPT; ++u) {
    if (P > 1) {
      const int k = (tid + u * T) & (P - 1);
#pragma unroll
      for (int m = 1; m < R; ++m) v[u * R + m] = cmul(v[u * R + m], tw[(m - 1) * P + k]);
    }
    Dft<R>::run(&v[u * R]);
  }
}

template <int N, int R, int E, int T>
__device__ __forceinline__ void pass_load(const float2* X, float2 (&v)[E], int tid) {
  constexpr int NB = N / R, BPT = E / R;
  static_assert(NB % 16 == 0 && T % 16 == 0, "padding arithmetic below assumes multiples of 16");
  const int base = pad16(tid);
#pragma unroll
  for (int u = 0; u < BPT; ++u) {
#pragma unroll
    for (int m = 0; m < R; ++m) v[u * R + m] = X[base + (u * T + m * NB) + ((u * T + m * NB) >> 4)];  // == pad16(tid + u*T + m*NB)
  }
}

template <int N, int R, int P, int E, int T>
__device__ __forceinline__ void pass_store(float2* X, const float2 (&v)[E], int tid) {
  constexpr int BPT = E / R;
#pragma unroll
  for (int u = 0; u < BPT; ++u) {
    const int b = tid + u * T;
    if (P == 1) {
      // j = 16 b + m (R == 16 in every plan's first pass, else R*b): pad16(R*b + m)
      const int j = b * R;
#pragma unroll
      for (int m = 0; m < R; ++m) X[pad16(j + m)] = v[u * R + m];
    } else {
      const int k = b & (P - 1);
      const int j = ((b - k) * R) + k;
      const int pj = pad16(j);
      if (P % 16 == 0) {
#pragma unroll
        for (int m = 0; m < R; ++m) X[pj + m * P + ((m * P) >> 4)] = v[u * R + m];  // == pad16(j + m*P): m*P is a multiple of 16
      } else {
#pragma unroll
        for (int m = 0; m < R; ++m) X[pad16(j + m * P)] = v[u * R + m];
      }
    }
  }
}

__device__ __forceinline__ float fast_log2(float x) {
  float y;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// SUB (B2S_FLAG_SUBFRAME_*): a frame is a_.sub_r sub-frames of N samples, transformed one after the other by the CTA that takes
// the frame; the TMA buffer is filled with the next sub-frame (or the next frame's first) behind each pass 0. The thread that owns
// bin b in the epilogue folds every sub-frame's |X|^2/fs into acc[] (registers) and the last sub-frame converts the reduced row.
// Where the sub-frames lie (back to back, or overlapping by half with frame 0's first one from a.sub_lead) is sub_src's.
template <int N, int MODE, bool DEBUG_LIN, bool SUB>
__global__ void __launch_bounds__(N / FftPlanT<N>::E) k_spectrum(const SpectralArgs a) {
  using PL = FftPlanT<N>;
  using TL = TwiddleLayout<N>;
  constexpr int E = PL::E, T = N / E;
  constexpr int R0 = PL::R0, R1 = PL::R1, R2 = PL::R2, R3 = PL::R3;
  constexpr int NP = (R3 > 1) ? 4 : (R2 > 1 ? 3 : 2);
  constexpr int P1 = R0, P2 = R0 * R1, P3 = R0 * R1 * R2;
  constexpr int RL = (NP == 4) ? R3 : (NP == 3 ? R2 : R1);  // radix of the last pass
  static_assert(R0 * R1 * R2 * R3 == N, "plan");

  extern __shared__ __align__(128) unsigned char smem[];
  float2* X = reinterpret_cast<float2*>(smem);
  float2* tws = X + exchange_elems<N>();                                   // shared copy of the small twiddle tables
  unsigned char* raw = reinterpret_cast<unsigned char*>(tws + TL::SMEM);  // 2N bytes (TMA mode only), 16-byte aligned
  __shared__ __align__(8) uint64_t full_bar;
  __shared__ float red_v[32];
  __shared__ int red_i[32];

  const int tid = threadIdx.x;
  const int lane = tid & 31, warp = tid >> 5;
  const char* base = static_cast<const char*>(a.iq);
  // first sample of sub-frame `sub` of `frame` (sub = 0 without SUB)
  auto src = [&](long long frame, int sub) {
    if (SUB) return sub_src(a, base, frame, sub);
    return base + frame * a.frame_stride_bytes;
  };

  if (MODE == kModeCs8Tma) {
    if (tid == 0) {
      mbar_init(&full_bar, 1);
      fence_barrier_init();
    }
  }
  // stage the small twiddle tables once per CTA
  if (TL::S1) {
    for (int i = tid; i < TL::E1; i += T) tws[TL::SO1 + i] = a.twiddle[TL::O1 + i];
  }
  if (TL::S2) {
    for (int i = tid; i < TL::E2; i += T) tws[TL::SO2 + i] = a.twiddle[TL::O2 + i];
  }
  if (TL::S3) {
    for (int i = tid; i < TL::E3; i += T) tws[TL::SO3 + i] = a.twiddle[TL::O3 + i];
  }
  __syncthreads();
  const float2* tw1 = TL::S1 ? tws + TL::SO1 : a.twiddle + TL::O1;
  const float2* tw2 = TL::S2 ? tws + TL::SO2 : a.twiddle + TL::O2;
  const float2* tw3 = TL::S3 ? tws + TL::SO3 : a.twiddle + TL::O3;
  if (MODE == kModeCs8Tma) {
    if (tid == 0 && static_cast<int>(blockIdx.x) < a.n_frames) {
      mbar_arrive_expect_tx(&full_bar, 2 * N);
      bulk_g2s(raw, src(blockIdx.x, SUB ? sub_begin(a, blockIdx.x) : 0), 2 * N, &full_bar);
    }
  }

  uint32_t parity = 0;
  for (int frame = blockIdx.x; frame < a.n_frames; frame += gridDim.x) {
    float2 v[E];
    float acc[SUB ? E : 1];  // SUB: the frame's partial reduction of the bins this thread owns in the epilogue
    const int sub0 = SUB ? sub_begin(a, frame) : 0;
    for (int sub = sub0; sub < (SUB ? a.sub_r : 1); ++sub) {
    const char* sub_p = SUB ? src(frame, sub) : nullptr;  // SUB: the sub-frame's first sample, once per sub-frame
    // ---------------- pass 0: unpack + window, radix R0, no twiddles (P = 1) ----------------
    {
      constexpr int NB = N / R0, BPT = E / R0;
      if (MODE == kModeCs8Tma) mbar_wait(&full_bar, parity);
      parity ^= 1;
#pragma unroll
      for (int u = 0; u < BPT; ++u) {
        const int b = tid + u * T;
#pragma unroll
        for (int m = 0; m < R0; ++m) {
          const int n = b + m * NB;
          const float w = __ldg(&a.wscale[n]);
          if (MODE == kModeCs8Tma) {
            const char2 s = reinterpret_cast<const char2*>(raw)[n];
            v[u * R0 + m] = make_float2(static_cast<float>(s.x) * w, static_cast<float>(s.y) * w);
          } else if (MODE == kModeCs8Direct) {
            const signed char* fp = reinterpret_cast<const signed char*>(SUB ? sub_p : src(frame, sub));
            v[u * R0 + m] = make_float2(static_cast<float>(fp[2 * n]) * w, static_cast<float>(fp[2 * n + 1]) * w);
          } else {
            const float* fp = reinterpret_cast<const float*>(SUB ? sub_p : src(frame, sub));
            v[u * R0 + m] = make_float2(fp[2 * n] * w, fp[2 * n + 1] * w);
          }
        }
      }
      pass_twiddle_butterfly<N, R0, 1, E, T>(v, nullptr, tid);
      pass_store<N, R0, 1, E, T>(X, v, tid);
    }
    __syncthreads();
    // the staging buffer is consumed: start the copy of this CTA's next (sub-)frame (overlaps the remaining passes)
    if (MODE == kModeCs8Tma && tid == 0) {
      if (SUB && sub + 1 < a.sub_r) {
        mbar_arrive_expect_tx(&full_bar, 2 * N);
        bulk_g2s(raw, src(frame, sub + 1), 2 * N, &full_bar);
      } else {
        const int next = frame + gridDim.x;  // > 0: starts at its sub-frame 0
        if (next < a.n_frames) {
          mbar_arrive_expect_tx(&full_bar, 2 * N);
          bulk_g2s(raw, src(next, 0), 2 * N, &full_bar);
        }
      }
    }
    // ---------------- middle passes ----------------
    if (NP >= 3) {
      pass_load<N, R1, E, T>(X, v, tid);
      __syncthreads();
      pass_twiddle_butterfly<N, R1, P1, E, T>(v, tw1, tid);
      pass_store<N, R1, P1, E, T>(X, v, tid);
      __syncthreads();
    }
    if (NP >= 4) {
      pass_load<N, R2, E, T>(X, v, tid);
      __syncthreads();
      pass_twiddle_butterfly<N, R2, P2, E, T>(v, tw2, tid);
      pass_store<N, R2, P2, E, T>(X, v, tid);
      __syncthreads();
    }
    // ---------------- last pass + epilogue ----------------
    pass_load<N, RL, E, T>(X, v, tid);
    constexpr int PL_ = (NP == 4) ? P3 : (NP == 3 ? P2 : P1);
    pass_twiddle_butterfly<N, RL, PL_, E, T>(v, NP == 4 ? tw3 : (NP == 3 ? tw2 : tw1), tid);
    if (SUB) {
#pragma unroll
      for (int i = 0; i < E; ++i) acc[i] = sub_fold(acc[i], fmaf(v[i].x, v[i].x, v[i].y * v[i].y) * a.inv_fs, sub == sub0, a.sub_max);
      if (sub + 1 < a.sub_r) __syncthreads();  // every thread has read X before the next sub-frame's pass 0 overwrites it
    }
    }

    // thread holds bins k = b + m * (N / RL): |X|^2 / fs -> 10 log10 (psd.cpp:18), written at (k + N/2) mod N
    float* row = a.psd_db + static_cast<size_t>(frame) * N;
    float best_v = -INFINITY;
    {
      constexpr int NB = N / RL, BPT = E / RL;
      constexpr float kDbPerLog2 = 3.0102999566398120f;  // 10 * log10(2)
#pragma unroll
      for (int u = 0; u < BPT; ++u) {
        const int b = tid + u * T;
#pragma unroll
        for (int m = 0; m < RL; ++m) {
          const float2 z = v[u * RL + m];
          const int j = (b + m * NB + N / 2) & (N - 1);
          const float pw = SUB ? sub_finish(acc[u * RL + m], a, a.sub_r - sub0) : fmaf(z.x, z.x, z.y * z.y) * a.inv_fs;
          const float db = kDbPerLog2 * fast_log2(pw);
          row[j] = db;
          if (DEBUG_LIN) a.power_lin[static_cast<size_t>(frame) * N + j] = pw;
          v[u * RL + m].x = db;  // keep for the argmax resolution below
          best_v = fmaxf(best_v, db);
        }
      }
    }
    // first maximum of the row (noise_learner.cpp:53-59): reduce the VALUE, then the lowest index that attains it
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) best_v = fmaxf(best_v, __shfl_xor_sync(0xffffffffu, best_v, o));
    if (lane == 0) red_v[warp] = best_v;
    __syncthreads();  // also: all reads of X are done before the next frame's first pass overwrites it
    {
      constexpr int NW = (T + 31) / 32;
      float row_max = red_v[0];
#pragma unroll
      for (int w = 1; w < NW; ++w) row_max = fmaxf(row_max, red_v[w]);
      int best_i = 0x7fffffff;
      constexpr int NB = N / RL, BPT = E / RL;
#pragma unroll
      for (int u = 0; u < BPT; ++u) {
#pragma unroll
        for (int m = 0; m < RL; ++m) {
          if (v[u * RL + m].x == row_max) best_i = min(best_i, (tid + u * T + m * NB + N / 2) & (N - 1));
        }
      }
      if (tid == 0) red_i[0] = 0x7fffffff;
      __syncthreads();
      if (best_i != 0x7fffffff) atomicMin(&red_i[0], best_i);
      __syncthreads();
      if (tid == 0) {
        a.peak_index[frame] = red_i[0];
        if (a.zero_per_frame[0]) a.zero_per_frame[0][frame] = 0;
        if (a.zero_per_frame[1]) a.zero_per_frame[1][frame] = 0;
        if (frame == 0 && a.zero_scalar) *a.zero_scalar = 0;
        a.peak_value[frame] = row_max;
      }
    }
  }
}

}  // namespace b2s
