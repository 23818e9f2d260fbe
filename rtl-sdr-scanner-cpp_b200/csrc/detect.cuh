// K2/K3 — the time-ordered half of the hot path, one thread per FFT bin marching through the frames of a push:
//   NoiseLearner (learn max / subtract)        reference sources/radio/blocks/noise_learner.cpp:11-28,36-67
//   Averager (ring + running sum, bit-exact)   reference sources/radio/averager.cpp:14-25,40-60
//   average(avg, GROUPING_X) frequency boxcar  reference sources/utils/utils.cpp:31-53
//   threshold predicate -> detection entries   reference sources/radio/blocks/transmission.cpp:88-96,113-130
//   Spectrogram decimate + accumulate + send   reference sources/radio/blocks/spectrogram.cpp:45-75
// The signal-map bookkeeping (transmission.cpp:70-176) consumes the compact detection entries on the host (tracker.h).
//
// Arithmetic contract: every float operation that feeds Averager state is the reference's operation in the reference's
// order (separate sub / add / IEEE division, no FMA contraction) so m_sum, the ring and m_average are bit-identical.
// The frequency boxcar is evaluated per aligned segment of kBoxSegment (16) bins: the first bin's window is summed left to
// right, the next 15 slide it exactly like the reference does (sum -= leaving; sum += entering), see boxcar_segment().
// The reference carries ONE running sum across the whole row (a 16384-long serial float chain); restarting it every
// 16 bins changes rounding only (<= 1e-3 dB vs the reference's own drift, asserted in tests) and keeps the work
// parallel. b2s_average(..., exact=1) provides the serial form for operator-level bit parity.
#pragma once
#include <cstring>

#include "b2s_device.cuh"

namespace b2s {

constexpr int kDetectBinsPerCta = 128;  // most bins one CTA can own (also the largest spectrogram decimation supported); DetectArgs::bins_per_cta
                                        // is what a launch uses (b2s_band::init picks it from the SM count)
constexpr int kDetectTileFrames = 32;   // frames per shared-memory tile
constexpr int kDetectBuffers = 6;       // at most this many PSD tiles in the shared ring (DetectArgs::n_buffers: what fits)
constexpr int kMaxSpecEmits = 16;       // spectrogram rows that one push (chunk) may complete
constexpr int kMaxWatch = 16;           // live signal keys whose window maxima K2 reports directly
constexpr int kCheckpointEvery = 64;    // frames between Averager-sum checkpoints (replay points for K3)

struct __align__(8) DetectEntry {  // one bin whose boxcar power reached min(start, stop) in one frame (8-byte aligned: ONE 8-byte store per entry)
  int bin;
  float value;  // boxcar-averaged power (dB above learned noise)
};
// Slot lists in memory: entry `pos` of frame t lives at ((t / 32) * capacity + pos) * 32 + t % 32 — the 32 frames of a K2 tile are the
// minor index. A box warp's lanes are the 32 frames of a tile, and lanes with equal list positions then write adjacent 8-byte
// cells: a warp-wide store touches 2 cache lines instead of 32. (With frame-major lists [t][capacity] every store of the CTA that
// carries an emitter's core touches 32 lines, its SUM warps' shared-memory traffic queues behind them, and the kernel ends with
// its slowest CTA.)
__host__ __device__ __forceinline__ size_t slot_index(int t, int pos, int capacity) {
  return (static_cast<size_t>(t >> 5) * capacity + pos) * 32 + (t & 31);
}

struct DetectArgs {
  // geometry
  int n;         // N
  int n_frames;  // T
  int group_y;   // Averager depth Y
  int group_x;   // boxcar width X
  int n_buffers; // PSD tiles in the shared-memory ring (2..kDetectBuffers)
  int bins_per_cta;  // bins owned by one CTA: a multiple of kBoxSegment, <= kDetectBinsPerCta (the tensor map's box is this + 2 * halo wide)
  // inputs
  const float* psd;  // [T][N] raw PSD rows from K1
  // noise state (per centre frequency)
  // State that a CTA's HALO columns read while the owning CTA updates it is double-buffered (in: before the push, out: after): a
  // CTA of a later wave (N >= 32768 has more CTAs than SMs; other bands' kernels delay CTAs) must not see its neighbour's results.
  const float* threshold;  // [N] before the push
  float* threshold_out;    // [N] after the push (differs only while learning)
  int noise_samples;  // samples learned before this push
  int learn_frames;   // frames 0.. with noise_samples + t < learn_frames are learning frames
  // averager state
  const float* avg_sum;   // [N] m_sum before the push
  float* avg_sum_out;     // [N] m_sum after the push
  const float* ring_in;   // [Y][N] ring before the push, oldest -> newest
  float* ring_out;        // [Y][N] ring after the push (a different buffer)
  int avg_frames;         // m_frames before the push
  float* avg_last;        // [N] m_average after the last frame
  float* checkpoints;     // [ceil(T/64)][N] m_sum before frame 64*c
  // detection: per-frame slot lists
  float detect_level;     // min(start, stop)
  // the same two levels as thresholds on the UNDIVIDED boxcar sum of an interior bin, whose window holds XD = 2 * (X / 2) + 1 bins
  // (X + 1 for an even X): x >= detect_sum  <=>  x / XD >= detect_level
  // (IEEE division is monotonic, so the set {x : fl(x / X) >= level} is an upper interval; the host finds its least element)
  float detect_sum, start_sum;
  DetectEntry* slots;     // [ceil(T/32)][slot_capacity][32], see slot_index()
  int* slot_count;        // [T] (zeroed before launch); may exceed slot_capacity -> overflow, reported by the host
  int slot_capacity;
  // spectrogram
  int spec_out;           // M (0 = off)
  float* spec_sum;        // [M]
  // watch list: the signal-map keys known when the push was enqueued. For each, K2 reports the maximum of the boxcar row
  // over [key - g/2, key + g/2] per frame (getMaxIndex(avgPower, N, key, groupSize) of Transmission::updateSignals,
  // transmission.cpp:114-117) and, per frame, whether any bin at or above the start level lies outside every key's
  // containsWithMargin interval (collection_utils.h:17-27) — i.e. whether addSignals could create a signal at all.
  int n_watch;
  int watch_key[kMaxWatch];
  int group_size;            // m_groupSize in bins
  float start_level;
  unsigned int* watch_max;   // [T][kMaxWatch] order-preserving encoding of the float maximum (0 = nothing written)
  int* cand_flag;            // [T] set to 1 when an uncovered candidate exists
  // rows to emit during this push, planned by the host from the frame clock (Spectrogram::send, spectrogram.cpp:62-75).
  // Carried in the kernel arguments so that no small host->device copy sits on the critical path behind the bulk IQ copy.
  int n_emit;                      // <= kMaxSpecEmits
  int emit_frame[kMaxSpecEmits];   // frame after which row i is emitted (ascending)
  int emit_div[kMaxSpecEmits];     // Container::m_counter at that moment
  signed char* spec_rows;          // [n_emit][M]
  unsigned long long* cta_ns;      // optional [2 * grid]: %globaltimer at CTA start / end (profiling: load balance)
  float* box_last;  // optional [N]: the boxcar row of the push's last frame (K4 reads the signals' m_power from it)
  // optional dense rows [T][N]
  float* dense_q;
  float* dense_avg;
  float* dense_box;
};

// noise-subtracted power of in-push frame t for bin j (NoiseLearner output), recomputable anywhere from the PSD rows
__device__ __forceinline__ float noise_sub(float p, float thr, bool learning) { return learning ? kNoData : __fsub_rn(p, thr); }

// One Averager::push for one bin: subtract the leaving value, add the new one (two separate roundings, in this order),
// then m_average = m_sum / groupSize (IEEE division) once groupSize frames were seen — averager.cpp:14-25,40-60.
__device__ __forceinline__ float averager_step(float& sum, float leaving, float entering, int frames_after, int group) {
  sum = __fsub_rn(sum, leaving);
  sum = __fadd_rn(sum, entering);
  return (frames_after >= group) ? __fdiv_rn(sum, static_cast<float>(group)) : kNoData;
}

// x / D for a small integer constant D, bit-identical to IEEE division: Markstein's sequence q = x*r, e = fma(-q, D, x),
// q' = fma(e, r, q) with r = RN(1/D). Verified exhaustively against x / D for every float with |x| in [2^-60, 2^60] and
// for +0 (D = 1..21; see DESIGN.md); anything outside that range takes the IEEE path. Three FMA-pipe instructions
// instead of the ~10 instruction + subroutine-call sequence the compiler emits for a correctly rounded division.
template <int D>
__device__ __forceinline__ float div_const(float x) {
  constexpr float d = static_cast<float>(D);
  constexpr float r = 1.0f / d;
  const uint32_t bits = __float_as_uint(x);
  const uint32_t ex = (bits >> 23) & 0xffu;
  if ((ex - 67u) <= 120u || bits == 0u) {
    const float q = __fmul_rn(x, r);
    const float e = __fmaf_rn(-q, d, x);
    return __fmaf_rn(e, r, q);
  }
  return __fdiv_rn(x, d);
}

// Same, without the range guard: for callers whose operands are sums of finite dB values (|x| < 2^60 by construction).
template <int D>
__device__ __forceinline__ float div_const_fast(float x) {
  constexpr float d = static_cast<float>(D);
  constexpr float r = 1.0f / d;
  const float q = __fmul_rn(x, r);
  const float e = __fmaf_rn(-q, d, x);
  return __fmaf_rn(e, r, q);
}

// order-preserving map float -> unsigned (so atomicMax on the image is max on the floats); never yields 0 for a real number
__host__ __device__ __forceinline__ unsigned int float_to_ordered(float f) {
#ifdef __CUDA_ARCH__
  const unsigned int b = __float_as_uint(f);
#else
  unsigned int b;
  memcpy(&b, &f, 4);
#endif
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
inline float ordered_to_float(unsigned int u) {
  const unsigned int b = (u & 0x80000000u) ? (u & 0x7fffffffu) : ~u;
  float f;
  memcpy(&f, &b, 4);
  return f;
}

constexpr int kBoxSegment = 16;  // bins per boxcar segment (segments are aligned to multiples of 16 bins)

// Boxcar running sums of one aligned segment of kBoxSegment bins over the ZERO-EXTENDED row: w[i] holds the averaged value of bin
// (b0 - H + i), i in [0, 8 + 2H), with 0.0f wherever that bin lies outside [0, N) (adding or subtracting 0.0f is exact,
// so clipped windows come out as the left-to-right sum of their valid bins). sums[0] = w[0] + w[1] + ... + w[2H];
// sums[k] continues the running sum exactly like utils.cpp:41-48: drop the leaving element, then add the entering one.
template <int H>
__device__ __forceinline__ void boxcar_segment(const float (&w)[kBoxSegment + 2 * H], float (&sums)[kBoxSegment]) {
  float s = w[0];
#pragma unroll
  for (int i = 1; i <= 2 * H; ++i) s = __fadd_rn(s, w[i]);
  sums[0] = s;
#pragma unroll
  for (int k = 1; k < kBoxSegment; ++k) {
    s = __fsub_rn(s, w[k - 1]);
    s = __fadd_rn(s, w[k + 2 * H]);
    sums[k] = s;
  }
}
// number of valid bins in the window of bin j (the reference's `count`, utils.cpp:34-49)
__device__ __forceinline__ int boxcar_count(int j, int n, int half) { return min(n - 1, j + half) - max(0, j - half) + 1; }
// a segment is interior when none of its 8 windows is clipped by the row ends (then every count is 2*half + 1)
__device__ __forceinline__ bool segment_interior(int b0, int n, int half) { return b0 - half >= 0 && b0 + kBoxSegment - 1 + half < n; }

// Boxcar value of ONE bin under the same definition, for any half; `at(bin)` returns the averaged value of a valid bin.
template <typename At>
__device__ __forceinline__ float boxcar_value(At at, int j, int n, int half) {
  if (half == 0 && j == n - 1) return 0.0f;  // reference quirk: groupSize 1 never writes the last element (utils.cpp:38)
  const int b0 = j & ~(kBoxSegment - 1);
  auto z = [&](int bin) { return (bin >= 0 && bin < n) ? at(bin) : 0.0f; };
  float s = z(b0 - half);
  for (int i = 1; i <= 2 * half; ++i) s = __fadd_rn(s, z(b0 - half + i));
  for (int k = 1; k <= j - b0; ++k) {
    s = __fsub_rn(s, z(b0 - half + k - 1));
    s = __fadd_rn(s, z(b0 + half + k));
  }
  return __fdiv_rn(s, static_cast<float>(boxcar_count(j, n, half)));
}

__device__ __forceinline__ unsigned long long global_timer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
// named barriers (id 0 is __syncthreads)
__device__ __forceinline__ void bar_sync(int id, int count) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory"); }
__device__ __forceinline__ void bar_arrive(int id, int count) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(count) : "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory"); }

// Warp roles of k_detect. One CTA owns kDetectBinsPerCta bins plus a halo of X/2 bins (rounded up to 4) on each side,
// computed redundantly; every role walks the push in tiles of kDetectTileFrames frames and the roles meet only through
// mbarriers, so each runs as far ahead as its buffers allow.
constexpr int kBoxGroups = 2;  // box-warp groups; group g takes the tiles with (tile % kBoxGroups) == g
constexpr int kSumWarps = 5, kBoxWarps = kDetectBinsPerCta / kBoxSegment;
constexpr int kSumThreads = 32 * kSumWarps;    // one thread per column (<= 160 columns: the CTA's bins plus both halos)
constexpr int kBoxThreads = 32 * kBoxWarps;    // threads of ONE box group: one warp per boxcar segment, lane = frame of the tile
constexpr int kSpecWarps = 2;                  // decimating spectrograms (N / out = d > 1): thread = spectrogram column, kDetectBinsPerCta / 2 at most
constexpr int kSpecThreads = 32 * kSpecWarps;
constexpr int kDetectThreads = kSumThreads + 32 /*producer*/ + kBoxGroups * kBoxThreads + kSpecThreads;
// Role of every warp. A CTA's warps are dealt round robin to the four SM sub-partitions (warp id % 4), each with its own issue
// port. The SUM warps carry the kernel's only serial chain and never wait (profile: the box warps spend half their samples at the
// FULL barrier), so their issue rate is the tile rate. The roles take contiguous warp ranges — box, producer, SPEC, SUM — which
// spreads the five SUM warps over all four sub-partitions.
enum : int { kRoleSum = 0, kRoleProducer = 1, kRoleSpec = 2, kRoleBox = 3 };
struct WarpRole {
  int role, index;  // index: SUM warp 0..4 (columns 32 * index ...), SPEC warp 0..1, box: group * kBoxWarps + segment
};
__device__ __forceinline__ WarpRole warp_role(int wid) {
  if (wid < kBoxGroups * kBoxWarps) return {kRoleBox, wid};
  if (wid == kBoxGroups * kBoxWarps) return {kRoleProducer, 0};
  if (wid < kBoxGroups * kBoxWarps + 1 + kSpecWarps) return {kRoleSpec, wid - kBoxGroups * kBoxWarps - 1};
  return {kRoleSum, wid - kBoxGroups * kBoxWarps - 1 - kSpecWarps};
}
// registers per thread: 24 warps, 6 per sub-partition (16384 registers each): 6 x 32 x 80 = 15360
constexpr int kDetectRegs = 80;
// the register file is split over the 4 SM sub-partitions (16384 registers each) and a CTA's warps are dealt round robin
static_assert(((kDetectThreads / 32 + 3) / 4) * ((kDetectRegs * 32 + 511) / 512 * 512) <= 16384, "k_detect must fit the register file");
static_assert(kDetectBinsPerCta / 2 <= kSpecThreads, "one SPEC thread per spectrogram column of a CTA");
constexpr int kAvgBuffers = 2;  // average tiles between the SUM and the box warps (a multiple of kBoxGroups)
static_assert(kAvgBuffers % kBoxGroups == 0 && kAvgBuffers <= 4, "each box group owns whole buffers; barrier ids 2..9");
constexpr int kBarFull = 2, kBarEmpty = 2 + kAvgBuffers;  // hardware barriers (one pair per average buffer): waiting warps sleep instead of polling

// SPEC warps, one full tile without an emission: out += mean of D adjacent raw bins, frame after frame (spectrogram.cpp:50-58). D is a
// compile-time constant so that the loads of 8 frames are in flight together; the sum over the D bins runs left to right from 0.0f
// like the reference's `sum` (0 + x0 is exact), the division by the power of two D is exact as a multiplication.
template <int D>
__device__ __forceinline__ float spec_tile(const float* __restrict__ raw, int width, float spec) {
  constexpr float inv_d = 1.0f / static_cast<float>(D);
#pragma unroll
  for (int h = 0; h < kDetectTileFrames; h += 8) {
    float v[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) v[u] = raw[(h + u) * width];
#pragma unroll
    for (int i = 1; i < D; ++i) {
#pragma unroll
      for (int u = 0; u < 8; ++u) v[u] = __fadd_rn(v[u], raw[(h + u) * width + i]);
    }
#pragma unroll
    for (int u = 0; u < 8; ++u) spec = __fadd_rn(spec, __fmul_rn(v[u], inv_d));
  }
  return spec;
}

// Y_T / HALF_T: Averager depth and X/2 as compile-time constants (21 / 10 = the reference's GROUPING_Y / GROUPING_X),
// or 0 / -1 for the generic runtime-parameter instantiation.
//
//   PRODUCER warp  streams PSD tiles [32 frames][width] into a shared ring with ONE 2-D TMA load per tile (the rows are short,
//                  so the copy engine's per-request cost dominates a row-by-row copy); completion counted on an mbarrier (p_full), slots recycled
//                  through p_empty.
//   SUM warps      (thread = column) the only truly serial chain of the path: NoiseLearner subtraction and
//                  m_sum -= leaving; m_sum += entering (averager.cpp:40-50), two dependent FADDs per frame. The last Y
//                  noise-subtracted values stay in registers from tile to tile (never stored, never re-read);
//                  m_average = m_sum / Y (off the chain) goes to a transposed shared tile (hardware barriers FULL / EMPTY
//                  per buffer). The spectrogram accumulation (the second serial chain, spectrogram.cpp:46-49) rides along.
//   SPEC warps     (thread = spectrogram column, only for decimating spectrograms d = N / out > 1) mean of d adjacent raw bins, then
//                  the accumulation chain of spectrogram.cpp:46-58; with d == 1 the chain rides in the SUM warps instead.
//   BOX warps      (warp = 16-bin segment, lane = frame) m_average = m_sum / Y for the steady tiles (the SUM warps hand over the raw
//                  sums: three instructions per value that the serial chain's warps do not have to issue), boxcar over the
//                  averaged tile, threshold (on the undivided boxcar sum, see DetectArgs::detect_sum), watched-window maxima;
//                  a lane with bins at or above the level reserves room in the frame's slot list with one global atomic
//                  and writes its entries once the atomic has returned (after the watch block). Two groups of box
//                  warps take alternate tiles, one per average buffer.
// Steady-state tiles (no learning frame, ring look-back inside the push, full tile, no dense debug rows) take a
// register-resident fully unrolled march; all others a generic one with the same float operations in the same order
// (bit-identical, tested).
// WIDTH_T: the CTA's column count (bins_per_cta + both halos) as a compile-time constant (152 = 128 bins + 2 x 12, the N = 16384 launch on
// 132 SMs; 136 = 112 bins + 2 x 12),
// or 0 for the runtime value: with a constant the SUM warps' 32 tile loads per column take immediate offsets instead of 32 address
// instructions on the kernel's critical warps.
template <int Y_T, int HALF_T, int WIDTH_T = 0>
__global__ void __maxnreg__(kDetectRegs) k_detect(const DetectArgs a, const __grid_constant__ CUtensorMap psd_map) {
  extern __shared__ __align__(128) float sm[];
  constexpr int TF = kDetectTileFrames;
  static_assert(Y_T <= TF, "the register-resident ring look-back needs Y <= tile frames");
  const int half = HALF_T >= 0 ? HALF_T : a.group_x / 2;
  const int hp = (half + 3) & ~3;                   // halo padded to a 16-byte multiple
  const int bins = WIDTH_T > 0 ? WIDTH_T - 2 * hp : a.bins_per_cta;  // bins owned by this CTA
  const int width = WIDTH_T > 0 ? WIDTH_T : bins + 2 * hp;          // columns held by this CTA (<= kSumThreads)
  const int tile_elems = TF * width;
  float* psd_tiles = sm;                            // [kDetectBuffers][TF][width] raw PSD rows (bulk-copy target)
  // averaged values (m_average) handed to the box warps, TRANSPOSED: [kAvgBuffers][width][kSumPitch] (column-major, pitch 33). The
  // SUM thread of column c writes avg[c*33 + f] (lane stride 33: conflict-free); a box warp reads one column for 32
  // frames at once (lane = frame: consecutive words, conflict-free).
  constexpr int kSumPitch = TF + 1;
  const int sum_elems = width * kSumPitch;
  float* sum_tiles = psd_tiles + a.n_buffers * tile_elems;
  float* box_park = sum_tiles + kAvgBuffers * sum_elems;  // [kBoxGroups][kBoxWarps][kBoxSegment][TF] per-lane scratch of the box warps
  __shared__ int rel_n, rel_key[kMaxWatch], rel_slot[kMaxWatch];          // watched keys that touch this CTA's bins
  __shared__ __align__(8) uint64_t p_full[kDetectBuffers], p_empty[kDetectBuffers];
  __shared__ int tile_raw[kAvgBuffers];  // the average buffer holds undivided m_sum values (steady tile) instead of m_average

  const int n = a.n, T = a.n_frames, Y = Y_T > 0 ? Y_T : a.group_y;
  const int j0 = blockIdx.x * bins;
  const int col0 = j0 - hp;  // bin of column 0
  const int tid = threadIdx.x;
  const int n_tiles = (T + TF - 1) / TF;
  const bool dense = a.dense_q || a.dense_avg || a.dense_box;
  const float* __restrict__ psd = a.psd;
  const float* __restrict__ ring_in = a.ring_in;

  // ---- one-time setup (all threads) ----
  if (tid == 0) {
    int cnt = 0;
    const int reach = a.group_size / 2 + 1;
    for (int w = 0; w < a.n_watch; ++w) {
      if (a.watch_key[w] + reach >= j0 && a.watch_key[w] - reach < j0 + bins) {
        rel_key[cnt] = a.watch_key[w];
        rel_slot[cnt] = w;
        ++cnt;
      }
    }
    rel_n = cnt;
    for (int i = 0; i < a.n_buffers; ++i) {
      mbar_init(&p_full[i], 1);  // the producer's arrival + the bytes of its TMA load
      mbar_init(&p_empty[i], kSumWarps + ((a.spec_out > 0 && n / a.spec_out > 1) ? kSpecWarps : 0));  // the SPEC warps only run for decimating spectrograms
    }
    fence_barrier_init();
  }
  if (tid < width && (col0 + tid < 0 || col0 + tid >= n)) {  // columns outside the row: the boxcar sees the zero-extended row
    for (int f = 0; f < kSumPitch; ++f) {
#pragma unroll
      for (int b = 0; b < kAvgBuffers; ++b) sum_tiles[b * sum_elems + tid * kSumPitch + f] = 0.0f;
    }
  }
  __syncthreads();

  const int lane = tid & 31;
  if (a.cta_ns && tid == 0) a.cta_ns[2 * blockIdx.x] = global_timer_ns();
  const WarpRole me = warp_role(tid >> 5);
  const int ct = me.index * 32 + lane;  // SUM warps: my column of the CTA's tile
  if (me.role == kRoleSum) {
    // ============================================ SUM warps ============================================
    const int j = col0 + ct;  // my column's bin
    const bool active = ct < width && j >= 0 && j < n;
    const bool owner = active && ct >= hp && ct < hp + bins;
    float thr = active ? a.threshold[j] : 0.0f;
    float sum = active ? a.avg_sum[j] : 0.0f;
    constexpr int YC = Y_T > 0 ? Y_T : 1;
    float lead[YC];  // noise-subtracted values of the last Y frames of the previous tile (the rows about to leave the ring)
#pragma unroll
    for (int f = 0; f < YC; ++f) lead[f] = 0.0f;
    // steady tiles: ring look-back inside the push (t0 >= Y), no learning frame left, no dense debug rows
    int first_steady = 0x7fffffff;
    if (Y_T > 0 && !dense) first_steady = max((Y + TF - 1) / TF, (max(a.learn_frames - a.noise_samples, 0) + TF - 1) / TF);
    // Spectrogram::process on the RAW rows (spectrogram.cpp:46-58): a second serial chain, carried by the owner threads
    const int d = a.spec_out > 0 ? n / a.spec_out : 0;
    const bool spec_owner = owner && d == 1;  // decimating spectrograms (d > 1) are carried by the SPEC warps
    float spec = spec_owner ? a.spec_sum[j] : 0.0f;
    int next_emit = 0;  // index of the first planned spectrogram row not yet emitted (rows are in frame order)
    // tile in which that row completes: ONE register compare per tile on the kernel's critical warps (the emission table lives in the
    // kernel arguments; an indexed constant load + a scan per tile would stall the SUM warps)
    int emit_tile = a.n_emit > 0 ? a.emit_frame[0] / TF : 0x7fffffff;

    int ps = 0;            // PSD ring slot of the current tile and the parity of its mbarrier phase
    uint32_t ps_phase = 0;
    for (int tile = 0; tile < n_tiles; ++tile) {
      const int t0 = tile * TF;
      const int tf = min(TF, T - t0);
      const int sb = tile % kAvgBuffers;
      const float* __restrict__ cur = psd_tiles + ps * tile_elems + ct;
      float* __restrict__ sum_col = sum_tiles + sb * sum_elems + ct * kSumPitch;  // my column of the transposed tile
      const bool steady = tile >= first_steady && tf == TF;  // the previous tile was full, so `lead` is valid
      mbar_wait_sleepy(&p_full[ps], ps_phase);                              // the PSD tile has landed
      if (tile >= kAvgBuffers) bar_sync(kBarEmpty + sb, kSumThreads + kBoxThreads);  // the box warps are done with this average buffer
      float q[TF];
      float checkpoint = 0.0f;
      // a spectrogram row completes inside this tile: one bit per tile, set by the host (a scan of the emission table with its
      // indexed constant loads sat on the serial chain's warps every tile)
      const bool emits = tile == emit_tile;
      const bool spec_inline = steady && d == 1 && !emits;
      if (steady) {
        if (active) {
          checkpoint = sum;  // m_sum before frame t0
          // two halves: the second half of the tile is loaded only when most of `lead` is dead, which keeps the live set at
          // ~40 frame values instead of 53 (no spills on the serial chain)
          constexpr int kSplit = TF / 2, kLate = kSplit - 4;
          const bool spec_here = spec_inline && spec_owner;
          // the spectrogram chain is accumulated by every thread and kept by the owners of an inline tile: with no branch around
          // it, ptxas can fill the Averager chain's latency gaps with it
          float sp = spec;
          auto load_half = [&](int f0) {
#pragma unroll
            for (int f = f0; f < f0 + kSplit; ++f) q[f] = cur[f * width];
#pragma unroll
            for (int f = f0; f < f0 + kSplit; ++f) sp = __fadd_rn(sp, q[f]);
#pragma unroll
            for (int f = f0; f < f0 + kSplit; ++f) q[f] = __fsub_rn(q[f], thr);  // NoiseLearner::work, noise_learner.cpp:54
          };
          auto march = [&](int f0, int f1) {
#pragma unroll
            for (int f = f0; f < f1; ++f) {
              const float old = (f >= YC) ? q[f - YC] : lead[f];
              sum = __fsub_rn(sum, old);   // Averager::subtract, averager.cpp:46-50
              sum = __fadd_rn(sum, q[f]);  // Averager::add, averager.cpp:40-44
              sum_col[f] = sum;            // m_sum; the box warps divide (t0 >= Y: the ring is full, m_average = m_sum / Y, averager.cpp:20-24)
            }
          };
          load_half(0);
          march(0, kLate);
          asm volatile("" ::: "memory");  // keep the compiler from hoisting the second half's loads to the top
          load_half(kSplit);
          march(kLate, TF);
          spec = spec_here ? sp : spec;
        }
      } else if (active) {
        // ---- generic march (learning frames, first tile of a push, partial tiles, dense debug rows, runtime Y) ----
        // frames leaving the ring that this tile does not hold: fetched together (one latency)
        float oldraw[TF];
#pragma unroll
        for (int f = 0; f < TF; ++f) {
          const int t = t0 + f;
          oldraw[f] = 0.0f;
          if (f < tf && (f < Y || t < Y)) oldraw[f] = (t < Y) ? ring_in[static_cast<size_t>(t) * n + j] : psd[static_cast<size_t>(t - Y) * n + j];
        }
#pragma unroll
        for (int f = 0; f < TF; ++f) {
          q[f] = 0.0f;
          if (f < tf) {
            const int t = t0 + f;
            const float p = cur[f * width];
            const bool learning = a.noise_samples + t < a.learn_frames;
            if (learning) thr = fmaxf(thr, p);  // Noise::add, noise_learner.cpp:19-21
            q[f] = noise_sub(p, thr, learning);
            // value leaving the ring (frame t - Y): thr is final for every frame that was not a learning frame
            float old;
            if (t < Y) {
              old = oldraw[f];  // the t-th oldest row of the pre-push ring
            } else {
              const float po = (f >= Y) ? cur[(f - Y) * width] : oldraw[f];
              old = noise_sub(po, thr, a.noise_samples + (t - Y) < a.learn_frames);
            }
            if (owner && (t % kCheckpointEvery) == 0) a.checkpoints[static_cast<size_t>(t / kCheckpointEvery) * n + j] = sum;  // m_sum before frame t
            const float avg = averager_step(sum, old, q[f], min(a.avg_frames + t + 1, Y), Y);
            sum_col[f] = avg;
            if (owner) {
              if (a.dense_q) a.dense_q[static_cast<size_t>(t) * n + j] = q[f];
              if (a.dense_avg) a.dense_avg[static_cast<size_t>(t) * n + j] = avg;
            }
          }
        }
      }
      if (ct == 0) tile_raw[sb] = steady ? 1 : 0;
      // (no fence: the barrier instruction orders this warp's shared-memory stores before the waiting warps' loads — the
      // producer / consumer pattern of the PTX manual; MEMBAR.SC.CTA here also waited for the warp's global stores)
      bar_arrive(kBarFull + sb, kSumThreads + kBoxThreads);  // hand the tile of averages to the box warps
      if (spec_owner && !spec_inline) {  // tiles with an emission, non-steady tiles
        const float* __restrict__ raw = cur;
        for (int f = 0; f < tf; ++f) {
          const float v = raw[f * width];
          spec = __fadd_rn(spec, v);
          int slot = -1;  // planned row emitted after frame t0 + f
          for (int i = next_emit; emits && i < a.n_emit && a.emit_frame[i] <= t0 + f; ++i) slot = (a.emit_frame[i] == t0 + f) ? i : slot;
          if (slot >= 0) {  // Spectrogram::send, spectrogram.cpp:66-72: float -> int8 truncation, then clear
            a.spec_rows[static_cast<size_t>(slot) * a.spec_out + j] = static_cast<signed char>(static_cast<int>(__fdiv_rn(spec, static_cast<float>(a.emit_div[slot]))));
            spec = 0.0f;
          }
        }
      }
      if (emits) {  // past this tile's rows
        while (next_emit < a.n_emit && a.emit_frame[next_emit] < t0 + TF) ++next_emit;
        emit_tile = next_emit < a.n_emit ? a.emit_frame[next_emit] / TF : 0x7fffffff;
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&p_empty[ps]);               // the PSD slot may be refilled
      if (++ps == a.n_buffers) {
        ps = 0;
        ps_phase ^= 1;
      }
      // global stores only after the hand-over: the fence above must not wait for a DRAM round trip
      if (steady && owner && (t0 % kCheckpointEvery) == 0) a.checkpoints[static_cast<size_t>(t0 / kCheckpointEvery) * n + j] = checkpoint;
      if (Y_T > 0) {
#pragma unroll
        for (int f = 0; f < YC; ++f) lead[f] = q[TF - YC + f];
      }
    }
    if (spec_owner) a.spec_sum[j] = spec;
    if (owner) {
      a.threshold_out[j] = thr;
      a.avg_sum_out[j] = sum;
      a.avg_last[j] = (T > 0 && a.avg_frames + T >= Y) ? __fdiv_rn(sum, static_cast<float>(Y)) : kNoData;
      // ring after the push, oldest -> newest: row i is in-push frame T - Y + i, or a surviving row of ring_in
      for (int i0 = 0; i0 < Y; i0 += 8) {
        float v[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const int i = i0 + u, t = T - Y + i;
          v[u] = 0.0f;
          if (i < Y) v[u] = (t >= 0) ? psd[static_cast<size_t>(t) * n + j] : ring_in[static_cast<size_t>(T + i) * n + j];
        }
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const int i = i0 + u, t = T - Y + i;
          if (i < Y) a.ring_out[static_cast<size_t>(i) * n + j] = (t >= 0) ? noise_sub(v[u], thr, a.noise_samples + t < a.learn_frames) : v[u];
        }
      }
    }
  } else if (me.role == kRoleProducer) {
    // ============================================ PRODUCER warp ============================================
    // Streams the tile [32 frames][width columns] of the PSD rows at (col0, t0) into the ring. Columns left of bin 0 / right of bin
    // N-1 and rows past the push arrive as zeros (nobody reads them).
    // One 2-D TMA load per tile: the rows are only (bins + halo) floats long in a row-major [T][N] matrix, so the copy engine's
    // per-request cost dominates whichever way a tile is fetched; one request per tile keeps that cost lowest.
    int ps = 0;
    uint32_t ps_phase = 1;  // waiting for the "previous" phase passes at once during the first round
    for (int tile = 0; tile < n_tiles; ++tile) {
      mbar_wait_sleepy(&p_empty[ps], ps_phase);  // the SUM (and SPEC) warps released the slot
      if (lane == 0) {
        mbar_arrive_expect_tx(&p_full[ps], static_cast<uint32_t>(tile_elems * sizeof(float)));
        tma_load_2d(psd_tiles + ps * tile_elems, &psd_map, col0, tile * TF, &p_full[ps]);
      }
      if (++ps == a.n_buffers) {
        ps = 0;
        ps_phase ^= 1;
      }
    }
  } else if (me.role == kRoleSpec) {
    // ============================================ SPEC warps ============================================
    // Spectrogram::process with decimation (spectrogram.cpp:45-58): out[i] += mean(p[i d .. i d + d - 1]) per frame, and
    // Spectrogram::send (spectrogram.cpp:62-72) on the frames the host planned. d is a power of two, so the mean's division is exact.
    const int d = a.spec_out > 0 ? n / a.spec_out : 0;
    if (d <= 1) return;                                   // nothing to do (and p_empty does not count these warps)
    const int sc = me.index * 32 + lane;                  // my spectrogram column inside the CTA
    const bool on = d > 1 && sc * d < bins && j0 + sc * d < n;
    const int col = on ? (j0 + sc * d) / d : 0;           // global spectrogram column
    float spec = on ? a.spec_sum[col] : 0.0f;
    const float inv_d = d > 0 ? 1.0f / static_cast<float>(d) : 0.0f;
    int next_emit = 0;
    int emit_tile = a.n_emit > 0 ? a.emit_frame[0] / TF : 0x7fffffff;
    int ps = 0;
    uint32_t ps_phase = 0;
    for (int tile = 0; tile < n_tiles; ++tile) {
      const int t0 = tile * TF;
      const int tf = min(TF, T - t0);
      mbar_wait_sleepy(&p_full[ps], ps_phase);
      const bool emits = tile == emit_tile;
      if (on) {
        const float* __restrict__ raw = psd_tiles + ps * tile_elems + hp + sc * d;
        if (!emits && tf == TF && d <= 16) {
          switch (d) {
            case 2: spec = spec_tile<2>(raw, width, spec); break;
            case 4: spec = spec_tile<4>(raw, width, spec); break;
            case 8: spec = spec_tile<8>(raw, width, spec); break;
            default: spec = spec_tile<16>(raw, width, spec); break;
          }
        } else {
          for (int f = 0; f < tf; ++f) {
            float v = raw[f * width];
            for (int i = 1; i < d; ++i) v = __fadd_rn(v, raw[f * width + i]);
            spec = __fadd_rn(spec, __fmul_rn(v, inv_d));
            int slot = -1;  // planned row emitted after frame t0 + f
            for (int i = next_emit; i < a.n_emit && a.emit_frame[i] <= t0 + f; ++i) slot = (a.emit_frame[i] == t0 + f) ? i : slot;
            if (slot >= 0) {  // float -> int8 truncation, then clear (spectrogram.cpp:66-72)
              a.spec_rows[static_cast<size_t>(slot) * a.spec_out + col] = static_cast<signed char>(static_cast<int>(__fdiv_rn(spec, static_cast<float>(a.emit_div[slot]))));
              spec = 0.0f;
            }
          }
        }
      }
      if (emits) {
        while (next_emit < a.n_emit && a.emit_frame[next_emit] < t0 + TF) ++next_emit;
        emit_tile = next_emit < a.n_emit ? a.emit_frame[next_emit] / TF : 0x7fffffff;
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&p_empty[ps]);
      if (++ps == a.n_buffers) {
        ps = 0;
        ps_phase ^= 1;
      }
    }
    if (on) a.spec_sum[col] = spec;
  } else {
    // ============================================ BOX warps ============================================
    // warp w owns segment w (kBoxSegment bins) of the CTA's 128 bins; lane = frame of the tile
    const int group = me.index / kBoxWarps;
    const int btid = (me.index - group * kBoxWarps) * 32 + lane;
    const int seg = btid >> 5;
    constexpr int SEG = kBoxSegment;
    static_assert(kBoxThreads / 32 == kDetectBinsPerCta / kBoxSegment && kDetectTileFrames == 32, "one box warp per segment, one lane per frame");
    const int b0 = seg * SEG, bin0 = j0 + b0;
    float* my_box = box_park + (group * kBoxWarps + seg) * SEG * TF + lane;  // [k * TF]: written and read by this lane only
    for (int tile = group; tile < n_tiles; tile += kBoxGroups) {
      const int t0 = tile * TF;
      const int tf = min(TF, T - t0);
      const int sb = tile % kAvgBuffers;
      bar_sync(kBarFull + sb, kSumThreads + kBoxThreads);  // the SUM warps have written this tile
      const float* avg_tile = sum_tiles + sb * sum_elems;
      const bool raw = tile_raw[sb] != 0;  // the SUM warps handed over m_sum: m_average = m_sum / Y is computed here
      const int f = lane, t = t0 + f;
      float box[SEG];
      bool have = false;
      bool released = false;  // this lane has already handed the average buffer back
      // `scaled`: box[] holds the UNDIVIDED boxcar sums of an interior segment and is compared with the sum thresholds; the
      // quotient is only formed for values that leave the kernel (entries, watch maxima, box_last, dense rows)
      bool scaled = false;
      if (f < tf && bin0 < n && b0 < bins) {  // (a launch with bins_per_cta < 128 leaves its last box warps idle: they only keep the barriers)
        have = true;
        if (HALF_T > 0) {
          constexpr int H = HALF_T > 0 ? HALF_T : 1;
          constexpr int YD = Y_T > 0 ? Y_T : 1;
          float w[SEG + 2 * H];
#pragma unroll
          for (int i = 0; i < SEG + 2 * H; ++i) w[i] = avg_tile[(hp + b0 - H + i) * kSumPitch + f];  // columns outside [0, N) hold 0.0f
          if (raw) {
#pragma unroll
            for (int i = 0; i < SEG + 2 * H; ++i) w[i] = div_const_fast<YD>(w[i]);  // averager.cpp:52-60 (0 / Y = 0 for the zero extension)
            // every value of the tile this lane needs has been read AND used: hand the buffer back before the serial boxcar chain, so
            // the SUM warps are not held up by it (with two average buffers they would otherwise wait for this warp's whole tile)
            if (tile + kAvgBuffers < n_tiles) bar_arrive(kBarEmpty + sb, kSumThreads + kBoxThreads);
            released = true;
          }
          boxcar_segment<H>(w, box);
          if (segment_interior(bin0, n, half)) {
            scaled = !a.dense_box;
            if (!scaled) {
#pragma unroll
              for (int k = 0; k < SEG; ++k) box[k] = div_const_fast<2 * H + 1>(box[k]);
            }
          } else {  // a row end cuts some windows: the boxcar sees the zero-extended row and divides by the clipped count
#pragma unroll
            for (int k = 0; k < SEG; ++k) box[k] = __fdiv_rn(box[k], static_cast<float>(boxcar_count(bin0 + k, n, half)));
          }
        } else {
#pragma unroll
          for (int k = 0; k < SEG; ++k) {
            const int bin = bin0 + k;
            box[k] = (bin >= n) ? -INFINITY
                                : boxcar_value([&](int bb) { return avg_tile[(hp + (bb - j0)) * kSumPitch + f]; }, bin, n, half);
          }
        }
      }
      if (!released && tile + kAvgBuffers < n_tiles) bar_arrive(kBarEmpty + sb, kSumThreads + kBoxThreads);  // this average buffer may be overwritten
      constexpr int XD = HALF_T > 0 ? 2 * HALF_T + 1 : 1;
      auto value_of = [&](float b) { return scaled ? div_const_fast<XD>(b) : b; };  // average(avg, X)[bin], utils.cpp:49
      const float lvl_detect = scaled ? a.detect_sum : a.detect_level, lvl_start = scaled ? a.start_sum : a.start_level;
      // bins at or above the detection level: reserve room in the frame's slot list now (one atomic per lane with hits);
      // the entries are written after the watch block below, when the atomic's round trip has been paid by other work
      unsigned int hits = 0;  // bit k: bin0 + k is at or above the detection level in my frame
      float top = -INFINITY;
      bool parked = false;
      int pos = 0;
      if (have) {
        top = box[0];
#pragma unroll
        for (int k = 1; k < SEG; ++k) top = fmaxf(top, box[k]);
        if (a.dense_box) {
#pragma unroll
          for (int k = 0; k < SEG; ++k)
            if (bin0 + k < n) a.dense_box[static_cast<size_t>(t) * n + bin0 + k] = box[k];
        }
        if (a.box_last && t == T - 1) {
#pragma unroll
          for (int k = 0; k < SEG; ++k)
            if (bin0 + k < n) a.box_last[bin0 + k] = value_of(box[k]);
        }
        if (top >= lvl_detect) {
          // A segment inside an emitter's skirt has all 16 bins at or above the level (the benchmark scene: ~260 bins per carrier):
          // that case is decided with 8 three-input minima and written out from registers below, without the mask, the parking
          // and the bit loop (the box warps of a CTA that carries an emitter take issue slots from its SUM warps).
          float bot = box[0];
#pragma unroll
          for (int k = 1; k < SEG; ++k) bot = fminf(bot, box[k]);
          if (bot >= lvl_detect && bin0 + SEG <= n) {
            hits = (1u << SEG) - 1u;
          } else {
#pragma unroll
            for (int k = 0; k < SEG; ++k) hits |= (bin0 + k < n && box[k] >= lvl_detect) ? (1u << k) : 0u;
#pragma unroll
            for (int k = 0; k < SEG; ++k) my_box[k * TF] = box[k];  // parked: the write-out below indexes them dynamically
            parked = true;
          }
          pos = atomicAdd(a.slot_count + t, __popc(hits));
        }
      }
      // watched keys: window maxima over ALL bins (also below the detection level), and the uncovered-candidate flag
      if (have && (rel_n > 0 || top >= lvl_start)) {
        const int gh = a.group_size / 2, margin = (a.group_size % 2 == 0) ? gh : gh + 1;
        const int last = min(bin0 + SEG, n) - 1 - bin0;  // last valid bin of the segment (local)
        unsigned int covered = 0;  // bit k: bin0 + k lies inside some key's containsWithMargin interval
        for (int r = 0; r < rel_n; ++r) {
          const int key = rel_key[r] - bin0, w = rel_slot[r];  // key position relative to the segment
          const int lo = max(key - gh, 0), hi = min(key + gh, last);
          if (lo <= hi) {  // the key's window touches this segment (same for every lane of the warp)
            if (!parked) {  // park my values in shared memory once: the windows below index them dynamically
#pragma unroll
              for (int k = 0; k < SEG; ++k) my_box[k * TF] = box[k];
              parked = true;
            }
            float m = my_box[lo * TF];
            for (int k = lo + 1; k <= hi; ++k) m = fmaxf(m, my_box[k * TF]);
            atomicMax(a.watch_max + static_cast<size_t>(t) * kMaxWatch + w, float_to_ordered(value_of(m)));  // max, then the (monotonic) division
          }
          const int clo = max(key - margin, 0), chi = min(key + margin, SEG - 1);
          if (clo <= chi) covered |= ((2u << (chi - clo)) - 1u) << clo;
        }
        if (top >= lvl_start) {
          unsigned int over = 0;
#pragma unroll
          for (int k = 0; k < SEG; ++k) over |= (k <= last && box[k] >= lvl_start) ? (1u << k) : 0u;
          if (over & ~covered) a.cand_flag[t] = 1;
        }
      }
      if (hits == (1u << SEG) - 1u && pos + SEG <= a.slot_capacity) {  // the whole segment, straight from the registers
        DetectEntry* dst = a.slots + slot_index(t, pos, a.slot_capacity);
#pragma unroll
        for (int k = 0; k < SEG; ++k) dst[k * 32] = DetectEntry{bin0 + k, value_of(box[k])};
      } else if (hits) {  // detection entries of my (frame, segment), bins ascending; the per-frame list is ordered later (k_entries_sort)
        if (!parked) {
#pragma unroll
          for (int k = 0; k < SEG; ++k) my_box[k * TF] = box[k];
        }
        DetectEntry* dst = a.slots + slot_index(t, 0, a.slot_capacity);
        for (unsigned int mm = hits; mm; mm &= mm - 1) {
          const int k = __ffs(mm) - 1;
          if (pos < a.slot_capacity) dst[static_cast<size_t>(pos) * 32] = DetectEntry{bin0 + k, value_of(my_box[k * TF])};
          ++pos;
        }
      }
    }
    if (a.cta_ns && btid == 0 && group == (n_tiles - 1) % kBoxGroups) a.cta_ns[2 * blockIdx.x + 1] = global_timer_ns();
  }
}

// Exclusive prefix of min(slot_count[t], capacity) over the T frames (one CTA), then per-frame ordering of the slot
// lists by bin into one dense array (one warp per frame, rank sort: bins are distinct inside a frame).
__global__ void __launch_bounds__(1024) k_entries_prefix(const int* slot_count, int capacity, int n_frames, int* offsets /*[T+1]*/, int* max_count) {
  __shared__ int part[1024];
  const int tid = threadIdx.x;
  const int per = (n_frames + 1023) / 1024;
  const int begin = tid * per, end = min(n_frames, begin + per);
  int local = 0, biggest = 0;
  for (int t = begin; t < end; ++t) {
    local += min(slot_count[t], capacity);
    biggest = max(biggest, slot_count[t]);
  }
  part[tid] = local;
  __syncthreads();
  for (int o = 1; o < 1024; o <<= 1) {
    const int v = tid >= o ? part[tid - o] : 0;
    __syncthreads();
    part[tid] += v;
    __syncthreads();
  }
  int run = part[tid] - local;
  for (int t = begin; t < end; ++t) {
    offsets[t] = run;
    run += min(slot_count[t], capacity);
  }
  if (tid == 1023) offsets[n_frames] = part[1023];
  atomicMax(max_count, biggest);
}

// Runs of consecutive bins of a frame's ordered entries, per level: [0] bins at or above the stop level, [1] start-level candidates
// (in range, not ignored: isIndexInRange / isIndexIgnored as bin intervals). K4 works on these instead of the raw entries, so
// its per-frame work does not grow with the width of a signal. Folded here because this kernel has a warp per frame and the whole
// GPU; K4 is a single CTA.
constexpr int kRunCap = 8;  // runs kept per frame and level; K4 replays a frame with more from its raw entries
struct RunFold {
  float stop_level, start_level;
  int bin_lo, bin_hi;                                                       // candidate bins: inside the scanned range ...
  int n_ignored, ignored_lo[16], ignored_hi[16];                            // ... and outside every ignored interval (bins, inclusive)
  int* lo;     // [2][kRunCap][n_frames] first bin of run r of level L of frame t at ((L * kRunCap + r) * n_frames + t)
  int* hi;     // same layout: last bin
  int* count;  // [2][n_frames]; may exceed kRunCap
};
__device__ __forceinline__ bool run_member(const RunFold& f, int level, const DetectEntry& d) {
  if (d.bin < 0) return false;
  if (level == 0) return f.stop_level <= d.value;
  if (!(f.start_level <= d.value) || d.bin < f.bin_lo || d.bin > f.bin_hi) return false;
  for (int r = 0; r < f.n_ignored; ++r) {
    if (f.ignored_lo[r] <= d.bin && d.bin <= f.ignored_hi[r]) return false;
  }
  return true;
}

__global__ void __launch_bounds__(256) k_entries_sort(const DetectEntry* slots, const int* slot_count, int capacity, int n_frames, const int* offsets, DetectEntry* out, const RunFold fold) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= n_frames) return;
  const int count = min(slot_count[warp], capacity);
  const DetectEntry* src = slots + slot_index(warp, 0, capacity);  // entry i of this frame: src[32 * i]
  DetectEntry* dst = out + offsets[warp];
  for (int i = lane; i < count; i += 32) {
    const DetectEntry e = src[static_cast<size_t>(i) * 32];
    int rank = 0;
    for (int k = 0; k < count; ++k) rank += (src[static_cast<size_t>(k) * 32].bin < e.bin) ? 1 : 0;
    dst[rank] = e;
  }
  if (!fold.count) return;
  __syncwarp();  // the ordered list is visible to the whole warp
  int n_runs[2] = {0, 0};
  for (int base = 0; base < count; base += 32) {
    const int e = base + lane;
    const bool valid = e < count;
    const DetectEntry none{-10, 0.0f};
    const DetectEntry cur = valid ? dst[e] : none;
    const DetectEntry prev = (valid && e > 0) ? dst[e - 1] : none;
    const DetectEntry next = (valid && e + 1 < count) ? dst[e + 1] : none;
#pragma unroll
    for (int L = 0; L < 2; ++L) {
      const bool me = valid && run_member(fold, L, cur);
      const bool starts = me && !(prev.bin == cur.bin - 1 && run_member(fold, L, prev));
      const bool ends = me && !(next.bin == cur.bin + 1 && run_member(fold, L, next));
      const unsigned sm = __ballot_sync(0xffffffffu, starts);
      const unsigned below = (1u << lane) - 1u;
      if (starts) {
        const int r = n_runs[L] + __popc(sm & below);
        if (r < kRunCap) fold.lo[static_cast<size_t>(L * kRunCap + r) * n_frames + warp] = cur.bin;
      }
      if (ends) {  // the run that ends here started at or before this lane: (#starts up to and including me) - 1
        const int r = n_runs[L] + __popc(sm & (below | (1u << lane))) - 1;
        if (r < kRunCap) fold.hi[static_cast<size_t>(L * kRunCap + r) * n_frames + warp] = cur.bin;
      }
      n_runs[L] += __popc(sm);
    }
  }
  if (lane == 0) {
    fold.count[warp] = n_runs[0];
    fold.count[n_frames + warp] = n_runs[1];
  }
}

// ------------------------------------------------------------------------------------------------------------
// K3 — window query: max / first-argmax of the boxcar row over [bin_lo, bin_hi] for a range of frames of the last push.
// This is getMaxIndex(avgPower, N, key, groupSize) of Transmission::updateSignals (transmission.cpp:114-117) for the
// (rare) frames where no bin of the window reached the detection level, so no detection entry carries the value.
// Each work item replays the Averager for the window's bins from the nearest m_sum checkpoint (same device functions
// as k_detect => bit-identical values).
// ------------------------------------------------------------------------------------------------------------
struct WindowWork {
  int bin_lo, bin_hi;      // inclusive window, already clipped to [0, N)
  int frame_lo, frame_hi;  // [frame_lo, frame_hi) inside one checkpoint interval
  int out_offset;          // results for frame f go to out[out_offset + (f - frame_lo)]
};

struct WindowArgs {
  int n, group_y, group_x;
  const float* psd;
  const float* threshold;  // final threshold of the push
  int noise_samples, learn_frames;
  const float* ring_in;
  int avg_frames;
  const float* checkpoints;
  const WindowWork* work;
  float* out_value;
  int* out_index;
};

__global__ void __launch_bounds__(256) k_window_query(const WindowArgs a) {
  extern __shared__ float sm[];
  const WindowWork w = a.work[blockIdx.x];
  const int n = a.n, Y = a.group_y, half = a.group_x / 2;
  // columns needed: the windows of every 8-bin segment that intersects [bin_lo, bin_hi]
  const int lo = max(0, (w.bin_lo & ~(kBoxSegment - 1)) - half), hi = min(n - 1, (w.bin_hi | (kBoxSegment - 1)) + half);
  const int width = hi - lo + 1;
  float* sum_s = sm;          // [width]
  float* avg_s = sm + width;  // [width]
  __shared__ float red_v[8];
  __shared__ int red_i[8];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int c = w.frame_lo / kCheckpointEvery;
  for (int i = tid; i < width; i += blockDim.x) sum_s[i] = a.checkpoints[static_cast<size_t>(c) * n + lo + i];
  __syncthreads();
  for (int t = c * kCheckpointEvery; t < w.frame_hi; ++t) {
    for (int i = tid; i < width; i += blockDim.x) {
      const int j = lo + i;
      const float thr = a.threshold[j];
      const float q = noise_sub(a.psd[static_cast<size_t>(t) * n + j], thr, a.noise_samples + t < a.learn_frames);
      float old;
      if (t >= Y) {
        old = noise_sub(a.psd[static_cast<size_t>(t - Y) * n + j], thr, a.noise_samples + (t - Y) < a.learn_frames);
      } else {
        old = a.ring_in[static_cast<size_t>(t) * n + j];
      }
      float s = sum_s[i];
      avg_s[i] = averager_step(s, old, q, min(a.avg_frames + t + 1, Y), Y);
      sum_s[i] = s;
    }
    __syncthreads();
    if (t >= w.frame_lo) {
      float bv = -INFINITY;
      int bi = 0x7fffffff;
      for (int j = w.bin_lo + tid; j <= w.bin_hi; j += blockDim.x) {
        const float box = boxcar_value([&](int bb) { return avg_s[bb - lo]; }, j, n, half);
        argmax_combine(bv, bi, box, j);
      }
      warp_argmax(bv, bi);
      if (lane == 0) {
        red_v[warp] = bv;
        red_i[warp] = bi;
      }
      __syncthreads();
      if (warp == 0) {
        const int nw = blockDim.x >> 5;
        bv = lane < nw ? red_v[lane] : -INFINITY;
        bi = lane < nw ? red_i[lane] : 0x7fffffff;
        warp_argmax(bv, bi);
        if (lane == 0) {
          a.out_value[w.out_offset + (t - w.frame_lo)] = bv;
          a.out_index[w.out_offset + (t - w.frame_lo)] = bi;
        }
      }
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------------------------
// stand-alone operators (operator-level parity with tests/test_averager.cpp and tests/test_utils.cpp)
// ------------------------------------------------------------------------------------------------------------
// Averager::push for `count` rows: same per-bin step as k_detect. ring_in/ring_out are [group][size], oldest first.
__global__ void k_averager_push(const float* rows, int count, int size, int group, float* sum, const float* ring_in, float* ring_out, int frames_before,
                                float* avg_out) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= size) return;
  float s = sum[j];
  float avg = kNoData;
  for (int t = 0; t < count; ++t) {
    const float old = (t >= group) ? rows[static_cast<size_t>(t - group) * size + j] : ring_in[static_cast<size_t>(t) * size + j];
    avg = averager_step(s, old, rows[static_cast<size_t>(t) * size + j], min(frames_before + t + 1, group), group);
  }
  sum[j] = s;
  avg_out[j] = avg;
  for (int i = 0; i < group; ++i) {
    const int t = count - group + i;
    ring_out[static_cast<size_t>(i) * size + j] = (t >= 0) ? rows[static_cast<size_t>(t) * size + j] : ring_in[static_cast<size_t>(count + i) * size + j];
  }
}

// average(in, out, size, groupSize), engine form: zero-extended 8-bin segments (same definition as k_detect)
__global__ void k_boxcar(const float* in, float* out, int size, int group, int rows) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  const int r = blockIdx.y;
  if (j >= size || r >= rows) return;
  const int half = group / 2;
  const float* row = in + static_cast<size_t>(r) * size;
  out[static_cast<size_t>(r) * size + j] = boxcar_value([&](int bb) { return row[bb]; }, j, size, half);
}

// average(in, out, size, groupSize), reference form (utils.cpp:31-53): one serial running sum per row, bit-exact.
__global__ void k_boxcar_serial(const float* in, float* out, int size, int group, int rows) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  const float* x = in + static_cast<size_t>(r) * size;
  float* y = out + static_cast<size_t>(r) * size;
  const int half = group / 2;
  float running = 0.0f;
  int terms = 0;
  if (half == 0 && size > 0) y[size - 1] = 0.0f;
  for (int pos = -half; pos < size + half - 1; ++pos) {
    const int leaving = pos - half - 1, entering = pos + half;
    if (0 <= leaving && leaving < size) {
      running = __fsub_rn(running, x[leaving]);
      terms--;
    }
    if (0 <= entering && entering < size) {
      running = __fadd_rn(running, x[entering]);
      terms++;
    }
    if (0 <= pos && pos < size) y[pos] = __fdiv_rn(running, static_cast<float>(terms));
  }
}

__global__ void k_fill(float* p, float value, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = value;
}

// ------------------------------------------------------------------------------------------------------------
// self-test: div_const<D> / div_const_fast<D> against IEEE division for every float of the guarded range
// ------------------------------------------------------------------------------------------------------------
// All floats with a biased exponent in [67, 187] (|x| in [2^-60, 2^61)), both signs, plus +-0: 2 * 121 * 2^23 + 2 values.
template <int D>
__global__ void k_check_div_const(unsigned long long* mismatches) {
  const unsigned long long total = 2ull * 121ull * 8388608ull;
  unsigned long long bad = 0;
  for (unsigned long long i = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x; i < total + 2; i += static_cast<unsigned long long>(gridDim.x) * blockDim.x) {
    uint32_t bits;
    if (i >= total) {
      bits = (i - total) ? 0x80000000u : 0u;
    } else {
      const uint32_t mant = static_cast<uint32_t>(i & 0x7fffffu), e = static_cast<uint32_t>((i >> 23) % 121ull), sign = static_cast<uint32_t>((i >> 23) / 121ull);
      bits = (sign << 31) | ((e + 67u) << 23) | mant;
    }
    const float x = __uint_as_float(bits);
    const uint32_t want = __float_as_uint(__fdiv_rn(x, static_cast<float>(D)));
    if (__float_as_uint(div_const<D>(x)) != want) ++bad;
    if (__float_as_uint(div_const_fast<D>(x)) != want && bits != 0x80000000u) ++bad;  // (-0 / D: the unguarded form returns +0; sums of dB values are never -0 after an add)
  }
  if (bad) atomicAdd(mismatches, bad);
}

}  // namespace b2s
