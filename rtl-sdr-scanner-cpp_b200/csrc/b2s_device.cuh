// Device-side helpers shared by the b2s kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace b2s {

constexpr float kNoData = -100.0f;  // setNoData, reference sources/utils/radio_utils.cpp:72-76

// ---------------------------------------------------------------------------------------------------------
// mbarrier + 1-D bulk async copy (TMA, SASS: UBLKCP). Used to stage each int8 IQ frame into shared memory.
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}
// Same, for waits that are expected to be long: the warp is suspended by the hardware (up to the hint, in ns) instead of
// polling, so it does not take issue slots from the warps doing the work.
__device__ __forceinline__ void mbar_wait_sleepy(uint64_t* bar, uint32_t parity) {
  uint32_t ok = 0;
  while (!ok) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity), "r"(1000000u)
        : "memory");
  }
}
// global -> shared bulk copy; dst/src 16-byte aligned, bytes a multiple of 16; completion is signalled on `bar`.
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// 2-D tiled TMA load: the box described by the tensor map at coordinates (c0 = innermost, c1) -> shared memory; elements
// outside the tensor are zero-filled and still counted in the mbarrier's transaction bytes.
__device__ __forceinline__ void tma_load_2d(void* dst_smem, const void* tensor_map, int c0, int c1, uint64_t* bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(smem_u32(dst_smem)),
               "l"(tensor_map), "r"(c0), "r"(c1), "r"(smem_u32(bar))
               : "memory");
}

// ---------------------------------------------------------------------------------------------------------
// complex helpers
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float2 cadd(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ float2 csub(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }
__device__ __forceinline__ float2 cmul(float2 a, float2 w) { return make_float2(fmaf(a.x, w.x, -a.y * w.y), fmaf(a.x, w.y, a.y * w.x)); }
__device__ __forceinline__ float2 mul_mi(float2 a) { return make_float2(a.y, -a.x); }  // a * (-i)
__device__ __forceinline__ float2 cneg(float2 a) { return make_float2(-a.x, -a.y); }
__device__ __forceinline__ float2 cscale(float2 a, float s) { return make_float2(a.x * s, a.y * s); }

// ---------------------------------------------------------------------------------------------------------
// cpk: complex value whose arithmetic is fixed half by half — every half is one IEEE round-to-nearest add, sub, mul or fma
// (the __f*_rn intrinsics, so the compiler never contracts or reorders them). A complex product rounds its partial
// products in the order of cmul below, which differs from the float2 helpers above; the FFT of k_spectrum3 is defined
// by this order (it is the one of the packed two-wide fp32 instructions of later GPUs, so both give identical bits).
// Hopper has no two-wide fp32 instructions: a complex add is two FADDs, a product two FMULs + two FFMAs. A negation or
// a multiplication by -i still folds into the consumer's operand modifiers.
// ---------------------------------------------------------------------------------------------------------
struct __align__(8) cpk {
  float x, y;
};
__device__ __forceinline__ cpk cpk_make(float re, float im) {
  cpk r;
  r.x = re;
  r.y = im;
  return r;
}
__device__ __forceinline__ float cre(cpk a) { return a.x; }
__device__ __forceinline__ float cim(cpk a) { return a.y; }
__device__ __forceinline__ cpk cmake(cpk, float re, float im) { return cpk_make(re, im); }
__device__ __forceinline__ cpk cadd(cpk a, cpk b) { return cpk_make(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ cpk csub(cpk a, cpk b) { return cpk_make(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y)); }
__device__ __forceinline__ cpk cpk_mul2(cpk a, cpk b) { return cpk_make(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }  // per half
__device__ __forceinline__ cpk cpk_fma2(cpk a, cpk b, cpk c) { return cpk_make(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }  // per half
__device__ __forceinline__ cpk mul_mi(cpk a) { return cpk_make(cim(a), -cre(a)); }  // a * (-i)
__device__ __forceinline__ cpk cneg(cpk a) { return cpk_make(-cre(a), -cim(a)); }
__device__ __forceinline__ cpk cscale(cpk a, float s) { return cpk_mul2(a, cpk_make(s, s)); }
__device__ __forceinline__ cpk cmul(cpk a, float2 w) {  // (a.x w.x - a.y w.y, a.y w.x + a.x w.y)
  const cpk t = cpk_mul2(a, cpk_make(w.x, w.x));
  return cpk_fma2(cpk_make(-cim(a), cre(a)), cpk_make(w.y, w.y), t);
}
__device__ __forceinline__ cpk cmadd(cpk a, float2 w, cpk acc) {  // acc + a * w
  const cpk t = cpk_fma2(cpk_make(-cim(a), cre(a)), cpk_make(w.y, w.y), acc);
  return cpk_fma2(a, cpk_make(w.x, w.x), t);
}

// first-maximum argmax reduction (ties -> lower index), matching the strict '<' scan of noise_learner.cpp:53-59
__device__ __forceinline__ void argmax_combine(float& v, int& i, float ov, int oi) {
  if (ov > v || (ov == v && oi < i)) {
    v = ov;
    i = oi;
  }
}
__device__ __forceinline__ void warp_argmax(float& v, int& i) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, v, o);
    const int oi = __shfl_xor_sync(0xffffffffu, i, o);
    argmax_combine(v, i, ov, oi);
  }
}

}  // namespace b2s
