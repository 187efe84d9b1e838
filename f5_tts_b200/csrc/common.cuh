// Shared device helpers for the sm_90a kernels: mbarrier, TMA load, programmatic-dependent-launch and
// wgmma-descriptor wrappers (inline PTX), small math.  No torch, no CUTLASS — plain CUDA 12.9.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#ifndef F5_SPIN_TIMEOUT_CYCLES
#define F5_SPIN_TIMEOUT_CYCLES (4000000000LL)  // ~2 s at 2 GHz: trap instead of hanging the device
#endif

namespace f5 {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred P;\n\t.reg .b32 R;\n\telect.sync R|P, 0xffffffff;\n\tselp.b32 %0, 1, 0, P;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}

// ----------------------------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P;\n\tmbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\tselp.b32 %0, 1, 0, P;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    // no printf here: a function call inside a wgmma pipeline makes ptxas serialise the MMAs
    if (clock64() - t0 > F5_SPIN_TIMEOUT_CYCLES) __trap();
  }
}

// ----------------------------------------------------------------------------------------------
// TMA (cp.async.bulk.tensor), tile mode, mbarrier completion
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                            int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::
          "r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::
          "r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// Programmatic dependent launch: a kernel launched with the PDL attribute may start while its predecessor is still
// draining; everything before pdl_wait() (smem carve-up, barrier init, descriptor prefetch) overlaps the predecessor's
// tail.  pdl_wait() returns once the predecessor grid has completed and its writes are visible.
// Both are no-ops for a normal launch.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// ----------------------------------------------------------------------------------------------
// wgmma shared-memory matrix descriptor (sm_90), 128-byte swizzle, tiles 1024-byte aligned.
// K-major operand: rows of 64 fp16 (128 B), 8-row groups 1024 B apart (SBO); advance along K inside the swizzle atom
// by adding bytes >> 4 to the low word (+2 per 16 fp16).  MN-major operand (attention V, rows = k index, 128 B = 64 MN
// elements): 8 k-rows per 1024-byte atom, SBO = 1024 B as well; a 16-row k step is +2048 B.
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t make_wgmma_desc_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= uint64_t((smem_addr & 0x3FFFF) >> 4);
  d |= uint64_t(1) << 16;          // leading byte offset (unused for 128B swizzle): 16 B
  d |= uint64_t(1024 >> 4) << 32;  // stride byte offset: 8 rows * 128 B
  d |= uint64_t(1) << 62;          // layout type 1 = SWIZZLE_128B
  return d;
}

// ----------------------------------------------------------------------------------------------
// math
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ float gelu_tanh(float x) {  // F.gelu(approximate="tanh") = x * sigmoid(2u), u = k0 (x + k1 x^3)
  // exp(-2u) = 2^(x * (c0 + c1 x^2)) with the constants folded: 3 FMA-pipe ops + MUFU.EX2 + FADD + MUFU.RCP + FMUL
  const float c0 = -2.3022081981f;   // -2 * sqrt(2/pi) * log2(e)
  const float c1 = -0.1029432396f;   // c0 * 0.044715
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * fmaf(x * x, c1, c0)));
  return __fdividef(x, 1.0f + e);
}
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.7071067811865476f)); }
__device__ __forceinline__ float silu(float x) { return x / (1.0f + __expf(-x)); }
__device__ __forceinline__ float mish(float x) {  // x * tanh(softplus(x)), softplus threshold 20 as torch
  float sp = x > 20.0f ? x : log1pf(__expf(x));
  return x * tanhf(sp);
}
__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

}  // namespace f5
