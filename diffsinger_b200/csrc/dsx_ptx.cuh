// sm_90a PTX wrappers used by the tensor-core kernels (dsx_hopper.cu): warpgroup MMA (wgmma) with shared-memory
// descriptors, cp.async copies into the 128-byte-swizzled operand layout, and the gate math of the epilogues.
#pragma once
#include <cuda_fp16.h>
#include <stdint.h>

namespace dsx {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---- operand layout --------------------------------------------------------------------------
// K-major operand tile, 128-byte swizzle: rows of 64 fp16 (128 B), 8-row swizzle atoms 1024 B apart.  The 16-byte chunk c
// of row r lives at r * 128 + ((c ^ (r & 7)) << 4); tiles start on 1024-byte boundaries.
__device__ __forceinline__ uint32_t sw128(int r, int c) { return static_cast<uint32_t>(r * 128 + ((c ^ (r & 7)) << 4)); }

// wgmma shared-memory matrix descriptor (sm_90): start >> 4 in bits [0,14), leading byte offset >> 4 in [16,30) (unused by
// swizzled K-major layouts, 1 by convention), stride byte offset >> 4 in [32,46) = 1024 B between 8-row atoms, swizzle mode
// in [62,64) with 1 = 128-byte swizzle.  Advancing K by 16 fp16 inside the 128-byte row is +32 bytes = +2 on the descriptor.
__device__ __forceinline__ uint64_t wg_desc(uint32_t smem_addr) {
  return static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4) | (static_cast<uint64_t>(1) << 16) |
         (static_cast<uint64_t>(1024 >> 4) << 32) | (static_cast<uint64_t>(1) << 62);
}

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// generic-proxy writes to shared memory (st.shared, cp.async) -> visible to the async proxy that wgmma reads through
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// D[64 x 128] (+)= A[64 x 16] . B[128 x 16]^T, fp16 operands from shared memory (both K-major), fp32 accumulators in
// registers.  Thread t of the warpgroup holds d[4 i + j] = D[16 (t / 32) + (t % 32) / 4 + 8 (j / 2)][8 i + 2 (t % 4) + j % 2].
__device__ __forceinline__ void wgmma_n128(float (&d)[64], uint64_t da, uint64_t db, int accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
      "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, "
      "%47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),
        "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
        "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
        "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),
        "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(accumulate)
      : "memory");
}

// ---- cp.async -----------------------------------------------------------------------------------
// 16 bytes global -> shared; valid == false writes zeros (src is not read)
__device__ __forceinline__ void cp16(uint32_t dst, const void* src, bool valid) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(valid ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// ---- math ---------------------------------------------------------------------------------------
__device__ __forceinline__ float tanh_approx(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float rcp_approx(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// sigmoid(g) * tanh(f) with tanh.approx (relative error ~2^-11, below the fp16 rounding of the gate output that follows)
__device__ __forceinline__ float gate_fast(float g, float f) {
  return fmaf(0.5f, tanh_approx(0.5f * g), 0.5f) * tanh_approx(f);
}
// sigmoid(g) * tanh(f) = (1 - E2) / ((1 + E1)(1 + E2)), E1 = e^-g, E2 = e^-2f: absolute error ~2e-7.  f is clamped at -15
// (tanh = -1 to 2e-13) so E2 stays finite.
__device__ __forceinline__ float gate_acc(float g, float f) {
  const float e1 = ex2_approx(-1.4426950408889634f * g);
  const float e2 = ex2_approx(-2.8853900817779268f * fmaxf(f, -15.f));
  return (1.f - e2) * rcp_approx((1.f + e1) * (1.f + e2));
}
__device__ __forceinline__ uint32_t h2_bits(__half2 v) { return *reinterpret_cast<uint32_t*>(&v); }

}  // namespace dsx
