// K1, warp-local variant for N = RA * 1024 (RA = 4, 8, 16  ->  N = 4096, 8192, 16384).
//
// Same math as k_spectrum (spectral.cuh) — unpack, window, N-point forward FFT, fftshift, |X|^2/fs, dB, first maximum —
// but organised so that the shared-memory pipe and the FP32 pipe overlap instead of alternating:
//
//   pass A  (block-wide)  radix-RA decimation in frequency over n0 (stride 1024), fed straight from the TMA-staged int8
//                         frame, twiddled by W_N^(b*k0) (coalesced 8-byte loads from an L2-resident table) and written
//                         to block k0 of the exchange buffer.                                   -> ONE block barrier
//   pass B  (warp-local)  warp k0 owns block k0 (1024 points): radix-32 over n1 (stride 32), twiddle W_1024^(n2*k1) from
//                         a small shared table, written back TRANSPOSED with pitch 33 inside the warp's own block.
//   pass C  (warp-local)  radix-32 over n2 (now stride 33 -> conflict-free), no twiddles; lane k1 ends up holding bins
//                         k0 + RA*k1 + 32*RA*k2. dB values go back into the warp's block ([k2][k1], skewed per block).
//                                                                                              -> ONE block barrier
//   output  (block-wide)  every thread gathers 4 consecutive bins (conflict-free thanks to the skew) and issues 16-byte
//                         coalesced stores; row maximum / first index reduction.
//
// k_spectrum needs two barriers per pass (read-all / write-all of one shared buffer) which keeps all 16 warps in the same
// phase: the LSU pipe idles while everybody computes and the FP32 pipe idles while everybody loads. Here passes B and C
// only need __syncwarp, so warps drift apart and one warp's loads overlap another warp's butterflies.
#pragma once
#include "spectral.cuh"

namespace b2s {

// multiply by W32^j = exp(-2 pi i j / 32), j a compile-time constant after unrolling
template <typename C>
__device__ __forceinline__ C mul_w32(C a, int j) {
  constexpr float C1 = 0.98078528040323043f, S1 = 0.19509032201612825f;  // pi/16
  constexpr float C2 = 0.92387953251128674f, S2 = 0.38268343236508977f;  // 2pi/16
  constexpr float C3 = 0.83146961230254524f, S3 = 0.55557023301960218f;  // 3pi/16
  constexpr float H = 0.70710678118654752f;                               // 4pi/16
  switch (j & 31) {
    case 0: return a;
    case 8: return mul_mi(a);
    case 16: return cneg(a);
    case 24: return cneg(mul_mi(a));
    case 1: return cmul(a, make_float2(C1, -S1));
    case 2: return cmul(a, make_float2(C2, -S2));
    case 3: return cmul(a, make_float2(C3, -S3));
    case 4: return cmul(a, make_float2(H, -H));
    case 5: return cmul(a, make_float2(S3, -C3));
    case 6: return cmul(a, make_float2(S2, -C2));
    case 7: return cmul(a, make_float2(S1, -C1));
    case 9: return cmul(a, make_float2(-S1, -C1));
    case 10: return cmul(a, make_float2(-S2, -C2));
    case 11: return cmul(a, make_float2(-S3, -C3));
    case 12: return cmul(a, make_float2(-H, -H));
    case 13: return cmul(a, make_float2(-C3, -S3));
    case 14: return cmul(a, make_float2(-C2, -S2));
    case 15: return cmul(a, make_float2(-C1, -S1));
    case 17: return cmul(a, make_float2(-C1, S1));
    case 18: return cmul(a, make_float2(-C2, S2));
    case 19: return cmul(a, make_float2(-C3, S3));
    case 20: return cmul(a, make_float2(-H, H));
    case 21: return cmul(a, make_float2(-S3, C3));
    default: return cmul(a, make_float2(C1, S1));  // not reached: n2*k1 <= 21 in the 4x8 split
  }
}

// 32-point DFT in registers: Cooley-Tukey 4 x 8 (n = 8*n1 + n2, k = k1 + 4*k2)
template <typename C>
__device__ __forceinline__ void dft32(C* v) {
  C y[8][4];
#pragma unroll
  for (int n2 = 0; n2 < 8; ++n2) {
    C a[4];
#pragma unroll
    for (int n1 = 0; n1 < 4; ++n1) a[n1] = v[8 * n1 + n2];
    Dft<4>::run(a);
#pragma unroll
    for (int k1 = 0; k1 < 4; ++k1) y[n2][k1] = mul_w32(a[k1], n2 * k1);
  }
#pragma unroll
  for (int k1 = 0; k1 < 4; ++k1) {
    C b[8];
#pragma unroll
    for (int n2 = 0; n2 < 8; ++n2) b[n2] = y[n2][k1];
    Dft<8>::run(b);
#pragma unroll
    for (int k2 = 0; k2 < 8; ++k2) v[k1 + 4 * k2] = b[k2];
  }
}

// The complex values of k_spectrum3 are cpk: every half an explicitly rounded scalar operation, in the rounding order that
// defines this kernel's results (b2s_device.cuh).
//
// Two code paths are chosen by the transform size:
//   kPairA (RA < 16)  pass A handles two ADJACENT columns per thread step: 4-byte sample loads, 8-byte window loads, 16-byte
//                     twiddle loads and 16-byte exchange stores instead of twice as many half-width ones
//   kDefer (!SPLIT)   the dB row is gathered into registers, the block barrier follows at once, and the global stores (+ the
//                     first-maximum search) are issued behind it, beside the next frame's pass A
// Passes B and C load their 32 inputs in the order the first radix-4 butterflies consume them.

constexpr int kBlockPitch = 32 * 33;  // float2 elements per warp-owned block (32 rows of pitch 33 after pass B)

// twiddle tables for this kernel (host builds them in this order, all float2):
//   [0, (RA-1)*1024)            pass A: W_N^(b*k0), laid out [k0-1][b]
//   [(RA-1)*1024, +31*32)       pass B: W_1024^(n2*k1), laid out [k1-1][n2]
template <int RA>
struct TwiddleLayout3 {
  static constexpr int A = (RA - 1) * 1024, B = 31 * 32, TOTAL = A + B;
};

// order-preserving image of a float (atomicMax on the image == max on the floats)
__device__ __forceinline__ unsigned int ordered_bits(float f) {
  const unsigned int b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

constexpr int kSplitM = 16384;          // sub-transform length of the split mode (RA = 16)
constexpr int kSplitStageBytes = 32768; // one staging buffer: S row segments of 16384 / S int8 pairs each

// Work distribution: items are handed out through an atomic counter (a.work_counter[0]) instead of a fixed
// blockIdx-strided walk, so a CTA that starts late (another band's kernel still holds its SM, config 3 / 5) simply takes
// fewer items; the kernel leaves the counter pair zeroed for the next launch.
//
// SPLIT (N = S * 16384, S = 2 ... 64 -> N = 32768 ... 1048576): decimation in frequency over the S residue classes of
// the bin index. Item (frame, c) computes
//        y_c[n'] = W_N^(n' c) * sum_s x[n' + 16384 s] w[n' + 16384 s] W_S^(s c),     n' < 16384        (pre-pass)
// and X[S k' + c] = FFT_16384(y_c)[k'] with exactly the passes of the non-split kernel. The S items of one frame are
// adjacent in the work order: they read the same int8 frame (L2 hits after the first) and fill the same output sectors.
// The int8 frame reaches the pre-pass through a 2-stage ring of bulk copies (S row segments of 16384 / S samples per
// stage, so a stage stays kSplitStageBytes whatever S is); at S = 64 a stage has fewer points than the CTA has threads,
// and two threads share each point.
//
// SUB (B2S_FLAG_SUBFRAME_*): an item still is a frame, or a (frame, class) pair; its CTA transforms the frame's a.sub_r sub-frames
// one after the other, and the staging ring treats them as its sequence of frames (sub-frame j + 1, or its first chunks in split
// mode, is staged while j is transformed). The thread that owns a bin after pass C folds each sub-frame's |X|^2/fs into the
// partial it keeps at that bin's place in the item's own psd_db row: the same thread writes and rereads the same addresses, so
// no barrier or atomic is needed, and the row stays in L2. The last sub-frame reads the partial, finishes the reduction, and runs
// the dB conversion, the stores and the first-maximum search of a frame without sub-frames on the reduced row. Where the
// sub-frames lie is sub_src's; the items of frame 0 start at sub_begin (1 when an overlapping frame 0 has no lead-in).
template <int RA, int MODE, bool DEBUG_LIN, int SPLIT_S, bool SUB>
__global__ void __launch_bounds__(RA * 32) k_spectrum3(const SpectralArgs a) {
  constexpr bool SPLIT = SPLIT_S > 1;
  constexpr int M = RA * 1024, T = RA * 32, BPT = 32 / RA;  // sub-transform length, threads, pass-A butterflies per thread
  static_assert(!SPLIT || RA == 16, "the split mode runs 16384-point sub-transforms");
  static_assert(SPLIT_S == 1 || SPLIT_S == 2 || SPLIT_S == 4 || SPLIT_S == 8 || SPLIT_S == 16 || SPLIT_S == 32 || SPLIT_S == 64, "S");
  extern __shared__ __align__(128) unsigned char smem[];
  using C = cpk;
  C* X = reinterpret_cast<C*>(smem);                                           // [RA][kBlockPitch]
  float2* twB = reinterpret_cast<float2*>(X + RA * kBlockPitch);               // [31][32]
  unsigned char* raw = reinterpret_cast<unsigned char*>(twB + 31 * 32);        // TMA mode: 2M bytes, or 2 x kSplitStageBytes (split)
  float* Xf = reinterpret_cast<float*>(X);
  __shared__ __align__(8) uint64_t full_bar[2];
  __shared__ float red_v[32];
  __shared__ int red_i[2];
  __shared__ int s_item[2];
  __shared__ float2 s_ws[SPLIT_S > 16 ? SPLIT_S : 16];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const char* base = static_cast<const char*>(a.iq);
  const float2* twA = a.twiddle;
  constexpr int S = SPLIT_S;
  constexpr int N = S * M;
  const int n_items = a.n_frames * S;
  constexpr int pc = M / S;  // samples per row segment of a stage

  if (MODE == kModeCs8Tma && tid == 0) {
    mbar_init(&full_bar[0], 1);
    mbar_init(&full_bar[1], 1);
    fence_barrier_init();
  }
  if (tid == 0) s_item[0] = atomicAdd(a.work_counter, 1);
  for (int i = tid; i < 31 * 32; i += T) twB[i] = a.twiddle[TwiddleLayout3<RA>::A + i];
  __syncthreads();
  int item = s_item[0];

  // first sample of sub-frame `sub` of `frame` (sub = 0 without SUB)
  auto frame_src = [&](int frame, int sub) {
    if (SUB) return sub_src(a, base, frame, sub);
    return base + static_cast<long long>(frame) * a.frame_stride_bytes;
  };
  // the sub-frame an item starts at: 0, or a.sub_first for frame 0's items
  auto sub_begin_of = [&](int it_) { return SUB ? sub_begin(a, SPLIT ? it_ / S : it_) : 0; };
  // stage `q`-th chunk of sub-frame `sub` of `it_`: S segments [s][pc samples] of the frame (split) / the whole frame (non-split)
  auto issue = [&](int it_, int sub, int q, int stage) {
    if (SPLIT) {
      const int fr = it_ / S;
      const char* src = frame_src(fr, sub) + static_cast<long long>(q) * pc * 2;
      mbar_arrive_expect_tx(&full_bar[stage], kSplitStageBytes);
      for (int s = 0; s < S; ++s) bulk_g2s(raw + stage * kSplitStageBytes + s * pc * 2, src + static_cast<long long>(s) * M * 2, pc * 2, &full_bar[stage]);
    } else {
      mbar_arrive_expect_tx(&full_bar[0], 2 * M);
      bulk_g2s(raw, frame_src(it_, sub), 2 * M, &full_bar[0]);
    }
  };
  if (MODE == kModeCs8Tma && tid == 0 && item < n_items) {
    issue(item, sub_begin_of(item), 0, 0);
    if (SPLIT) issue(item, sub_begin_of(item), 1, 1);
  }

  constexpr bool kDefer = !SPLIT;
  constexpr bool kPairA = RA < 16;  // pairing helps where several CTAs share an SM (N <= 8192)
  int pend_frame = -1;   // kDefer: frame whose first maximum is still being collected in red_i[(round - 1) & 1]
  float pend_max = 0.0f;
  uint32_t parity = 0;   // non-split: phase of full_bar[0]
  uint32_t chunk_no = 0; // split: chunks consumed so far by this CTA (stage = chunk_no & 1, phase = (chunk_no >> 1) & 1)
  int round = 0;
  int sub = sub_begin_of(item);  // SUB: the sub-frame of `item` in hand
  while (item < n_items) {
    const int frame = SPLIT ? item / S : item;
    const int c = SPLIT ? item - frame * S : 0;
    const int sub0 = sub_begin_of(item);
    const bool first_sub = !SUB || sub == sub0;
    const char* sub_p = SUB ? frame_src(frame, sub) : nullptr;  // SUB: the sub-frame's first sample, once per sub-frame
    if (tid == 0 && first_sub) s_item[(round + 1) & 1] = atomicAdd(a.work_counter, 1);  // the item after this one (read after the next barrier)
    if (tid == 32 && c == 0 && first_sub) {  // K2's per-frame counters (SpectralArgs::zero_per_frame)
      if (a.zero_per_frame[0]) a.zero_per_frame[0][frame] = 0;
      if (a.zero_per_frame[1]) a.zero_per_frame[1][frame] = 0;
      if (frame == 0 && a.zero_scalar) *a.zero_scalar = 0;
    }
    if (SPLIT) {
      // ---------------- pre-pass: y_c into the exchange buffer, laid out like pass A's input [m][b] ----------------
      if (tid < S) s_ws[tid] = a.split_ws[(tid * c) & (S - 1)];
      __syncthreads();
      const float2* twc = a.split_tw + static_cast<size_t>(c) * M;
      for (int q = 0; q < S; ++q) {
        const unsigned char* st = raw + (chunk_no & 1u) * kSplitStageBytes;
        if (MODE == kModeCs8Tma) mbar_wait(&full_bar[chunk_no & 1u], (chunk_no >> 1) & 1u);
        // windowed sample n = np + 16384 s of the frame; i = np - q * pc is its column in the stage
        auto term = [&](int i, int np, int s) {
          const int n = np + s * M;
          const float w = __ldg(&a.wscale[n]);
          if (MODE == kModeCs8Tma) {
            const char2 smp = reinterpret_cast<const char2*>(st + s * pc * 2)[i];
            return cscale(cmake(C{}, static_cast<float>(smp.x), static_cast<float>(smp.y)), w);
          } else if (MODE == kModeCs8Direct) {
            const signed char* fp = reinterpret_cast<const signed char*>(SUB ? sub_p : frame_src(frame, sub));
            return cscale(cmake(C{}, static_cast<float>(fp[2 * n]), static_cast<float>(fp[2 * n + 1])), w);
          } else {
            const float* fp = reinterpret_cast<const float*>(SUB ? sub_p : frame_src(frame, sub));
            return cscale(cmake(C{}, fp[2 * n], fp[2 * n + 1]), w);
          }
        };
        if constexpr (S <= 16) {
#pragma unroll(S >= 8 ? 2 : 4)
        for (int u = 0; u < pc / T; ++u) {  // independent points: their loads overlap
          const int i = tid + u * T;
          const int np = q * pc + i;
          C acc = cmake(C{}, 0.0f, 0.0f);
#pragma unroll
          for (int s = 0; s < S; ++s) {
            const C xs = term(i, np, s);
            if (s == 0) {  // W_S^0 = 1
              acc = xs;
            } else if (S == 2) {  // W_2^c = +-1
              acc = c ? csub(acc, xs) : cadd(acc, xs);
            } else {
              acc = cmadd(xs, s_ws[s], acc);
            }
          }
          if (c != 0) acc = cmul(acc, __ldg(&twc[np]));
          X[(np >> 10) * kBlockPitch + (np & 1023)] = acc;
        }
        } else {
          // S = 32, 64: a stage has pc = 512 or 256 points for T = 512 threads, and every thread sums 32 terms. At S = 32 a thread
          // has one point. At S = 64 lanes l and l + 16 of a warp share a point: lane half h sums the terms s = 32 h ... 32 h + 31,
          // and one shuffle adds the two halves.
          constexpr int kLanes = T / pc, kPoints = 32 / kLanes, kTerms = S / kLanes;  // lanes per point, points per warp
          static_assert(kLanes * pc == T && kTerms == 32, "one or two threads per point");
          const int h = lane / kPoints, i = warp * kPoints + lane % kPoints;
          const int np = q * pc + i, s0 = h * kTerms;
          C acc = cmul(term(i, np, s0), s_ws[s0]);
#pragma unroll
          for (int s = 1; s < kTerms; ++s) acc = cmadd(term(i, np, s0 + s), s_ws[s0 + s], acc);
          if (kLanes == 2) acc = cadd(acc, cmake(C{}, __shfl_xor_sync(0xffffffffu, cre(acc), 16), __shfl_xor_sync(0xffffffffu, cim(acc), 16)));
          if (c != 0) acc = cmul(acc, __ldg(&twc[np]));
          if (h == 0) X[(np >> 10) * kBlockPitch + (np & 1023)] = acc;
        }
        __syncthreads();  // this stage is consumed (and, after the last chunk, y_c is complete)
        if (MODE == kModeCs8Tma && tid == 0) {  // refill it with the chunk two ahead (possibly of the next item)
          const int next = s_item[(round + 1) & 1];
          if (q + 2 < S) issue(item, sub, q + 2, chunk_no & 1u);
          else if (SUB && sub + 1 < a.sub_r) issue(item, sub + 1, q + 2 - S, chunk_no & 1u);
          else if (next < n_items) issue(next, sub_begin_of(next), q + 2 - S, chunk_no & 1u);
        }
        ++chunk_no;
      }
    }
    // ---------------- pass A: radix RA over n0 (stride 1024), input = windowed int8 samples (or y_c) ----------------
    if (!SPLIT && MODE == kModeCs8Tma) mbar_wait(&full_bar[0], parity);
    parity ^= 1;
    static_assert(BPT % 2 == 0, "pass A pairs adjacent columns");
    if constexpr (kPairA) {
#pragma unroll
    for (int u = 0; u < BPT / 2; ++u) {
      const int b = 2 * (tid + u * T);  // even: this step does columns b and b + 1
      C v0[RA], v1[RA];
#pragma unroll
      for (int m = 0; m < RA; ++m) {
        const int n = m * 1024 + b;
        if (SPLIT) {  // in place: this thread alone reads and writes columns b, b + 1 of every block
          const float4 x = *reinterpret_cast<const float4*>(&X[m * kBlockPitch + b]);
          v0[m] = cmake(C{}, x.x, x.y);
          v1[m] = cmake(C{}, x.z, x.w);
        } else {
          const float2 w = __ldg(reinterpret_cast<const float2*>(a.wscale + n));
          if (MODE == kModeCs8Tma) {
            const char4 s = reinterpret_cast<const char4*>(raw)[n >> 1];
            v0[m] = cscale(cmake(C{}, static_cast<float>(s.x), static_cast<float>(s.y)), w.x);
            v1[m] = cscale(cmake(C{}, static_cast<float>(s.z), static_cast<float>(s.w)), w.y);
          } else if (MODE == kModeCs8Direct) {
            const signed char* fp = reinterpret_cast<const signed char*>(SUB ? sub_p : frame_src(frame, sub)) + 2 * n;
            v0[m] = cscale(cmake(C{}, static_cast<float>(fp[0]), static_cast<float>(fp[1])), w.x);
            v1[m] = cscale(cmake(C{}, static_cast<float>(fp[2]), static_cast<float>(fp[3])), w.y);
          } else {
            const float2* fp = reinterpret_cast<const float2*>(SUB ? sub_p : frame_src(frame, sub)) + n;
            const float2 x0 = fp[0], x1 = fp[1];
            v0[m] = cscale(cmake(C{}, x0.x, x0.y), w.x);
            v1[m] = cscale(cmake(C{}, x1.x, x1.y), w.y);
          }
        }
      }
      Dft<RA>::run(v0);
      Dft<RA>::run(v1);
      *reinterpret_cast<float4*>(&X[b]) = make_float4(cre(v0[0]), cim(v0[0]), cre(v1[0]), cim(v1[0]));
#pragma unroll
      for (int k0 = 1; k0 < RA; ++k0) {
        const float4 t = __ldg(reinterpret_cast<const float4*>(twA + (k0 - 1) * 1024 + b));
        const C r0 = cmul(v0[k0], make_float2(t.x, t.y)), r1 = cmul(v1[k0], make_float2(t.z, t.w));
        *reinterpret_cast<float4*>(&X[k0 * kBlockPitch + b]) = make_float4(cre(r0), cim(r0), cre(r1), cim(r1));
      }
    }
    } else {
#pragma unroll
    for (int u = 0; u < BPT; ++u) {
      const int b = tid + u * T;  // 0..1023
      C v[RA];
#pragma unroll
      for (int m = 0; m < RA; ++m) {
        const int n = m * 1024 + b;
        if (SPLIT) {
          v[m] = X[m * kBlockPitch + b];  // in place: this thread alone reads and writes column b of every block
        } else {
          const float w = __ldg(&a.wscale[n]);
          if (MODE == kModeCs8Tma) {
            const char2 s = reinterpret_cast<const char2*>(raw)[n];
            v[m] = cscale(cmake(C{}, static_cast<float>(s.x), static_cast<float>(s.y)), w);
          } else if (MODE == kModeCs8Direct) {
            const signed char* fp = reinterpret_cast<const signed char*>(SUB ? sub_p : frame_src(frame, sub));
            v[m] = cscale(cmake(C{}, static_cast<float>(fp[2 * n]), static_cast<float>(fp[2 * n + 1])), w);
          } else {
            const float* fp = reinterpret_cast<const float*>(SUB ? sub_p : frame_src(frame, sub));
            v[m] = cscale(cmake(C{}, fp[2 * n], fp[2 * n + 1]), w);
          }
        }
      }
      Dft<RA>::run(v);
      X[b] = v[0];
#pragma unroll
      for (int k0 = 1; k0 < RA; ++k0) X[k0 * kBlockPitch + b] = cmul(v[k0], __ldg(&twA[(k0 - 1) * 1024 + b]));
    }
    }
    __syncthreads();
    if (kDefer && tid == 0 && pend_frame >= 0 && first_sub) {  // the previous frame's first maximum: every thread's atomicMin precedes this barrier
      a.peak_index[pend_frame] = red_i[(round + 1) & 1];
      a.peak_value[pend_frame] = pend_max;
    }
    const int next_item = s_item[(round + 1) & 1];
    if (!SPLIT && MODE == kModeCs8Tma && tid == 0) {  // staging buffer consumed: fetch the next (sub-)frame behind the remaining passes
      if (SUB && sub + 1 < a.sub_r) issue(item, sub + 1, 0, 0);
      else if (next_item < n_items) issue(next_item, sub_begin_of(next_item), 0, 0);
    }
    // ---------------- passes B and C: warp `warp` owns block k0 = warp ----------------
    C v[32];
    C* blk = X + warp * kBlockPitch;
#pragma unroll
    for (int q = 0; q < 32; ++q) {  // element (n1 = m, n2 = lane), in the order dft32's radix-4 butterflies take them: (n2 = 0: 0 8 16 24), (n2 = 1: 1 9 17 25), ...
      const int m = 8 * (q & 3) + (q >> 2);
      v[m] = blk[m * 32 + lane];
    }
    __syncwarp();                                             // every lane has its inputs before anyone overwrites the block
    dft32(v);
    blk[lane * 33] = v[0];
#pragma unroll
    for (int k1 = 1; k1 < 32; ++k1) blk[lane * 33 + k1] = cmul(v[k1], twB[(k1 - 1) * 32 + lane]);  // transposed: [n2][k1], pitch 33
    __syncwarp();
#pragma unroll
    for (int q = 0; q < 32; ++q) {  // element (k1 = lane, n2 = m), same order
      const int m = 8 * (q & 3) + (q >> 2);
      v[m] = blk[m * 33 + lane];
    }
    __syncwarp();
    dft32(v);
    // lane k1 holds X[k0 + RA*k1 + 32*RA*k2] in v[k2]
    // SUB: the partial of bin k0 + RA*k1 + 32*RA*k2 lives where the row stores that bin (fftshifted; split: class c's place)
    float* part = a.psd_db + static_cast<size_t>(frame) * N;
    auto part_at = [&](int k2) -> float& {
      const int bin = warp + RA * lane + 32 * RA * k2;
      return part[SPLIT ? S * ((bin + M / 2) & (M - 1)) + c : (bin + M / 2) & (M - 1)];
    };
    if (SUB && sub + 1 < a.sub_r) {
#pragma unroll
      for (int k2 = 0; k2 < 32; ++k2) {
        const float re = cre(v[k2]), im = cim(v[k2]);
        float& p = part_at(k2);
        p = sub_fold(p, fmaf(re, re, im * im) * a.inv_fs, first_sub, a.sub_max);
      }
      __syncthreads();  // every warp has read its block before the next sub-frame's pass A overwrites the exchange buffer
      ++sub;
      continue;
    }
    // |X|^2/fs -> dB (psd.cpp:18), parked in the warp's block as [k2][k1]; SUB: of the reduced row
    float best_v = -INFINITY;
    float* res = Xf + warp * (2 * kBlockPitch) + 2 * warp;  // skew of 2 floats per block keeps the gather below conflict-free
    constexpr float kDbPerLog2 = 3.0102999566398120f;
#pragma unroll
    for (int k2 = 0; k2 < 32; ++k2) {
      const float re = cre(v[k2]), im = cim(v[k2]);
      float pw = fmaf(re, re, im * im) * a.inv_fs;
      if (SUB) pw = sub_finish(sub_fold(part_at(k2), pw, first_sub, a.sub_max), a, a.sub_r - sub0);
      const float db = kDbPerLog2 * fast_log2(pw);
      res[k2 * 32 + lane] = DEBUG_LIN ? pw : db;
      best_v = fmaxf(best_v, db);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) best_v = fmaxf(best_v, __shfl_xor_sync(0xffffffffu, best_v, o));
    if (lane == 0) red_v[warp] = best_v;
    const int ri = kDefer ? (round & 1) : 0;
    if (tid == 0) red_i[ri] = 0x7fffffff;
    __syncthreads();
    // ---------------- output: 4 consecutive (local) bins per thread, stored at (bin + N/2) mod N ----------------
    float row_max = red_v[0];
#pragma unroll
    for (int w = 1; w < RA; ++w) row_max = fmaxf(row_max, red_v[w]);
    float* row = a.psd_db + static_cast<size_t>(frame) * N;
    int best_i = 0x7fffffff;
    if (SPLIT) {
      // the S classes of a frame interleave (global bin = S * local + c): consecutive lanes take consecutive local bins, so one warp
      // store covers 32 * S consecutive floats of the row (every S-th one); the other classes' CTAs fill the rest of the sectors
      float* lin = DEBUG_LIN ? a.power_lin + static_cast<size_t>(frame) * N : nullptr;
#pragma unroll 8
      for (int i = 0; i < M / T; ++i) {
        const int bin = tid + i * T;
        const int q = bin / RA, k1 = q & 31, k2 = q >> 5, k0 = bin & (RA - 1);
        float o = Xf[k0 * (2 * kBlockPitch + 2) + k2 * 32 + k1];  // lanes: 16 blocks x 2 adjacent words -> distinct banks
        const int j = S * ((bin + M / 2) & (M - 1)) + c;
        if (DEBUG_LIN) {
          lin[j] = o;
          o = kDbPerLog2 * fast_log2(o);
        }
        row[j] = o;
        if (o == row_max) best_i = min(best_i, j);
      }
    } else {
      float4 og[M / (4 * T)];
      if (kDefer) {  // gather the row into registers, release the exchange buffer, then store: the stores drain beside the next pass A
#pragma unroll
        for (int i = 0; i < M / (4 * T); ++i) {
          const int bin = 4 * (tid + i * T);
          const int q = bin / RA, k1 = q & 31, k2 = q >> 5;
          const int k0 = bin & (RA - 1);
          const float* src = Xf + k2 * 32 + k1;
          og[i].x = src[(k0 + 0) * (2 * kBlockPitch + 2)];
          og[i].y = src[(k0 + 1) * (2 * kBlockPitch + 2)];
          og[i].z = src[(k0 + 2) * (2 * kBlockPitch + 2)];
          og[i].w = src[(k0 + 3) * (2 * kBlockPitch + 2)];
        }
        __syncthreads();  // the exchange buffer is free again
      }
#pragma unroll
      for (int i = 0; i < M / (4 * T); ++i) {
        const int bin = 4 * (tid + i * T);
        const int q = bin / RA, k1 = q & 31, k2 = q >> 5;
        const int k0 = bin & (RA - 1);
        float4 o;
        if (kDefer) {
          o = og[i];
        } else {
          const float* src = Xf + k2 * 32 + k1;
          o.x = src[(k0 + 0) * (2 * kBlockPitch + 2)];
          o.y = src[(k0 + 1) * (2 * kBlockPitch + 2)];
          o.z = src[(k0 + 2) * (2 * kBlockPitch + 2)];
          o.w = src[(k0 + 3) * (2 * kBlockPitch + 2)];
        }
        const int j = (bin + M / 2) & (M - 1);
        if (DEBUG_LIN) {  // debug instantiation: the block holds |X|^2/fs; dB is recomputed here
          *reinterpret_cast<float4*>(a.power_lin + static_cast<size_t>(frame) * N + j) = o;
          o.x = kDbPerLog2 * fast_log2(o.x);
          o.y = kDbPerLog2 * fast_log2(o.y);
          o.z = kDbPerLog2 * fast_log2(o.z);
          o.w = kDbPerLog2 * fast_log2(o.w);
        }
        *reinterpret_cast<float4*>(row + j) = o;
        if (o.x == row_max) best_i = min(best_i, j);
        if (o.y == row_max) best_i = min(best_i, j + 1);
        if (o.z == row_max) best_i = min(best_i, j + 2);
        if (o.w == row_max) best_i = min(best_i, j + 3);
      }
    }
    if (best_i != 0x7fffffff) atomicMin(&red_i[ri], best_i);
    if (kDefer) {  // red_i[ri] is final after the next block barrier (pass A of the next item, or the one behind the loop)
      pend_frame = frame;
      pend_max = row_max;
    } else {
      __syncthreads();  // the exchange buffer is free again; red_i is final
    }
    if (!kDefer && tid == 0) {
      if (SPLIT) {  // first maximum over the S classes: larger value wins, equal values -> lower index
        atomicMax(a.peak_packed + frame, (static_cast<unsigned long long>(ordered_bits(row_max)) << 32) | (0xffffffffu - static_cast<unsigned int>(red_i[0])));
      } else {
        a.peak_index[frame] = red_i[0];
        a.peak_value[frame] = row_max;
      }
    }
    item = next_item;
    ++round;
    sub = sub_begin_of(item);
  }
  if (kDefer) {
    __syncthreads();
    if (tid == 0 && pend_frame >= 0) {
      a.peak_index[pend_frame] = red_i[(round + 1) & 1];
      a.peak_value[pend_frame] = pend_max;
    }
  }
  // leave the counters zeroed for the next launch: the last CTA to get here resets them (every CTA has drawn its last item)
  if (tid == 0) {
    __threadfence();
    if (atomicAdd(a.work_counter + 1, 1) == static_cast<int>(gridDim.x) - 1) {
      a.work_counter[0] = 0;
      a.work_counter[1] = 0;
    }
  }
}

// split mode: (value, index) out of the packed per-frame maxima
__global__ void k_peak_unpack(const unsigned long long* packed, int n_frames, int* peak_index, float* peak_value) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= n_frames) return;
  const unsigned long long p = packed[f];
  const unsigned int u = static_cast<unsigned int>(p >> 32);
  peak_value[f] = __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
  peak_index[f] = static_cast<int>(0xffffffffu - static_cast<unsigned int>(p & 0xffffffffu));
}

}  // namespace b2s
