// Thin inline-PTX wrappers for the sm_90a features the attention kernels use: 16-byte cp.async copies (zero-filling
// padding), ldmatrix fragment loads, the fp16 m16n8k16 tensor-core MMA with fp32 accumulation, MUFU ex2 and the
// acquire load of the in-kernel grid barrier.
//
// Fragment layouts (PTX ISA, "mma.m16n8k16" with .f16 inputs), g = lane / 4, q = lane % 4:
//   A (16 x 16, row-major)  a0 = A[g][2q..2q+1]  a1 = A[g+8][2q..]  a2 = A[g][8+2q..]  a3 = A[g+8][8+2q..]
//   B (16 x 8,  "col")      b0 = B[2q..2q+1][g]  b1 = B[8+2q..][g]
//   C (16 x 8,  fp32)       c0,c1 = C[g][2q..2q+1]  c2,c3 = C[g+8][2q..2q+1]
// so the C fragments of two neighbouring n-tiles, packed to fp16, are exactly the A fragment of one k-step: P = softmax(S)
// goes from the Q K^T accumulators to the P V MMA without leaving registers.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace pww {
namespace ptx {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---------------------------------------------------------------- cp.async (global -> shared, 16 bytes)
// src_bytes = 0 writes 16 zero bytes and reads nothing (padding rows / columns).
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// ---------------------------------------------------------------- ldmatrix
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x2_t(uint32_t addr, uint32_t& r0, uint32_t& r1) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0, %1}, [%2];" : "=r"(r0), "=r"(r1) : "r"(addr));
}

// ---------------------------------------------------------------- tensor-core MMA: C (+)= A B, fp16 in, fp32 accumulate
__device__ __forceinline__ void mma16816(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
      "{%0, %1, %2, %3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// ---------------------------------------------------------------- misc
__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ uint32_t pack_h2(float lo, float hi) {
  const __half2 h = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<const uint32_t*>(&h);
}
__device__ __forceinline__ float2 unpack_h2(uint32_t v) { return __half22float2(*reinterpret_cast<const __half2*>(&v)); }
__device__ __forceinline__ unsigned long long ld_acquire_gpu_u64(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}

}  // namespace ptx
}  // namespace pww
