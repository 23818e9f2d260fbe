// Spectrum occupancy (b2s_band_set_occupancy): per-bin duty cycles and a max-hold trace, accumulated per centre frequency over
// the pushes of a band. Two kernels, enqueued on the band's stream behind the list ordering (k_entries_sort) of a push:
//   k_occupancy_count  the push's ordered detection entries: a bin is counted above a level in a frame iff its entry's value is at or
//                      above the level (the predicate of k_entries_sort's run fold). Every entry belongs to a frame past noise
//                      learning, and a frame's entries are distinct bins, so the counts are per-bin frame counts.
//   k_occupancy_max    the column maximum of the push's raw PSD rows (K1's psd_db, after sub-frame folding), folded into max_db.
// Neither writes anything the band's own results read.
#pragma once
#include "detect.cuh"

namespace b2s {

// One thread per entry, grid-stride over the push's whole ordered list (offsets[n_frames] entries): the work follows the entries,
// not T x N. Entries of one frame are distinct bins, so the reductions only meet across frames; the adds are fire-and-forget (RED).
__global__ void __launch_bounds__(256) k_occupancy_count(const DetectEntry* sorted, const int* offsets, int n_frames, float start_level,
                                                         float stop_level, unsigned int* above_start, unsigned int* above_stop) {
  const int total = offsets[n_frames];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const DetectEntry e = sorted[i];
    if (stop_level <= e.value) atomicAdd(above_stop + e.bin, 1u);
    if (start_level <= e.value) atomicAdd(above_start + e.bin, 1u);
  }
}

// A CTA owns kOccupancyBins consecutive bins (one 128-byte line of a row) and walks the T rows with `row_groups` groups of 8 threads,
// each thread loading one float4 of every row_groups-th row. The groups' maxima meet in shared memory, and 8 threads then fold the
// CTA's bins into max_db with one plain read-modify-write: no other CTA touches them, so no atomics. The grid is N / 32 CTAs; the
// host raises row_groups (32..128) where that grid is small, so that a small N still keeps every SM streaming.
constexpr int kOccupancyBins = 32;
constexpr int kOccupancyCols = kOccupancyBins / 4;  // float4 columns per CTA

__device__ __forceinline__ float4 fmax4(float4 a, float4 b) { return make_float4(fmaxf(a.x, b.x), fmaxf(a.y, b.y), fmaxf(a.z, b.z), fmaxf(a.w, b.w)); }

__global__ void __launch_bounds__(1024, 1) k_occupancy_max(const float* __restrict__ psd, int n, int n_frames, float* max_db) {
  extern __shared__ float4 occ_part[];  // [row_groups][kOccupancyCols]
  const int tid = threadIdx.x, col = tid % kOccupancyCols, rg = tid / kOccupancyCols, groups = blockDim.x / kOccupancyCols;
  const size_t col0 = static_cast<size_t>(blockIdx.x) * kOccupancyBins + 4 * col;
  const float4* rows = reinterpret_cast<const float4*>(psd + col0);
  const size_t pitch = static_cast<size_t>(n) / 4;  // float4 per row
  float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
  int t = rg;
  for (; t + 3 * groups < n_frames; t += 4 * groups) {  // four rows in flight per thread
    const float4 a = __ldg(rows + static_cast<size_t>(t) * pitch);
    const float4 b = __ldg(rows + static_cast<size_t>(t + groups) * pitch);
    const float4 c = __ldg(rows + static_cast<size_t>(t + 2 * groups) * pitch);
    const float4 d = __ldg(rows + static_cast<size_t>(t + 3 * groups) * pitch);
    m = fmax4(fmax4(m, a), fmax4(fmax4(b, c), d));
  }
  for (; t < n_frames; t += groups) m = fmax4(m, __ldg(rows + static_cast<size_t>(t) * pitch));
  occ_part[tid] = m;
  __syncthreads();
  for (int half = groups / 2; half > 0; half /= 2) {  // groups is a power of two
    if (rg < half) occ_part[tid] = fmax4(occ_part[tid], occ_part[tid + half * kOccupancyCols]);
    __syncthreads();
  }
  if (tid < kOccupancyCols) {
    float4* out = reinterpret_cast<float4*>(max_db + col0);
    *out = fmax4(*out, occ_part[tid]);
  }
}

}  // namespace b2s
