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
// The same layout in fp16 elements: where (row r, k) of a tile goes when it is packed in global memory already swizzled,
// so that one bulk copy of the tile into a 1024-aligned shared-memory slot lands it as sw128 places it.
__host__ __device__ __forceinline__ int sw128_elem(int r, int k) { return r * 64 + ((((k >> 3) ^ r) & 7) << 3) + (k & 7); }

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
// all but the most recent wgmma group of this warpgroup complete
__device__ __forceinline__ void wg_wait1() { asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory"); }
// barrier over the 128 threads of this thread's warpgroup, of at most two (ids 1 and 2; 0 is __syncthreads)
__device__ __forceinline__ void wg_bar_sync() {
  if (threadIdx.x < 128) asm volatile("bar.sync 1, 128;" ::: "memory");
  else asm volatile("bar.sync 2, 128;" ::: "memory");
}
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

// The same product for N = 16, 32, 64 or 128 output columns (the vocoder's convolutions are as narrow as 16 channels):
// d holds N / 2 accumulators in the layout of wgmma_n128, i < N / 8.
template <int N>
__device__ __forceinline__ void wgmma_f16(float (&d)[N / 2], uint64_t da, uint64_t db, int accumulate);
template <>
__device__ __forceinline__ void wgmma_f16<128>(float (&d)[64], uint64_t da, uint64_t db, int accumulate) {
  wgmma_n128(d, da, db, accumulate);
}
template <>
__device__ __forceinline__ void wgmma_f16<16>(float (&d)[8], uint64_t da, uint64_t db, int accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(da), "l"(db), "r"(accumulate)
      : "memory");
}
template <>
__device__ __forceinline__ void wgmma_f16<32>(float (&d)[16], uint64_t da, uint64_t db, int accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(da), "l"(db), "r"(accumulate)
      : "memory");
}
template <>
__device__ __forceinline__ void wgmma_f16<64>(float (&d)[32], uint64_t da, uint64_t db, int accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(accumulate)
      : "memory");
}

// MN-major operands (both A and B stored with M / N contiguous: frames-major activations read with the frame axis as K),
// 128-byte swizzle: K row k of a 64-wide MN atom is 128 bytes at k * 128 with the 16-byte chunks swizzled as sw128(k, c);
// 8-row K groups are 1024 B apart (stride byte offset) and MN atoms `atom_bytes` apart (leading byte offset).  Advancing
// K by 16 is +2048 bytes = +128 on the descriptor.
__device__ __forceinline__ uint64_t wg_desc_mn(uint32_t smem_addr, uint32_t atom_bytes) {
  return static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4) | (static_cast<uint64_t>((atom_bytes >> 4) & 0x3FFF) << 16) |
         (static_cast<uint64_t>(1024 >> 4) << 32) | (static_cast<uint64_t>(1) << 62);
}

// D[64 x 128] (+)= A[64 x 16] . B[128 x 16]^T with both operands MN-major (the transpose immediates set); the
// accumulator layout is wgmma_n128's.
__device__ __forceinline__ void wgmma_n128_mn(float (&d)[64], uint64_t da, uint64_t db, int accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
      "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, "
      "%47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 1, 1;\n\t}"
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

// D[64 x N] (+)= A[64 x 16] . B[N x 16]^T with A K-major and B MN-major (its N axis contiguous in 64-wide atoms, the
// layout of wg_desc_mn): the attention backward's products with a [keys or queries][D] tile as B.  N = 64 or 128.
template <int N>
__device__ __forceinline__ void wgmma_f16_bmn(float (&d)[N / 2], uint64_t da, uint64_t db, int accumulate);
template <>
__device__ __forceinline__ void wgmma_f16_bmn<64>(float (&d)[32], uint64_t da, uint64_t db, int accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(accumulate)
      : "memory");
}
template <>
__device__ __forceinline__ void wgmma_f16_bmn<128>(float (&d)[64], uint64_t da, uint64_t db, int accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(accumulate)
      : "memory");
}

// accumulator element e of thread wtid of the warpgroup: its row and column inside the 64 x N block
__device__ __forceinline__ int acc_row(int wtid, int e) { return ((wtid >> 5) << 4) + ((wtid & 31) >> 2) + ((e & 2) ? 8 : 0); }
__device__ __forceinline__ int acc_col(int wtid, int e) { return ((e >> 2) << 3) + ((wtid & 3) << 1) + (e & 1); }

// ---- cp.async -----------------------------------------------------------------------------------
// 16 bytes global -> shared; valid == false writes zeros (src is not read)
__device__ __forceinline__ void cp16(uint32_t dst, const void* src, bool valid) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(valid ? 16 : 0) : "memory");
}
// cp16 with a policy for the source lines
__device__ __forceinline__ void cp16_hint(uint32_t dst, const void* src, bool valid, uint64_t pol) {
  asm volatile("cp.async.cg.shared.global.L2::cache_hint [%0], [%1], 16, %2, %3;" ::"r"(dst), "l"(src),
               "r"(valid ? 16 : 0), "l"(pol)
               : "memory");
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// ---- mbarriers and bulk copies ------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
// makes mbarrier.init visible to the other threads and to the async proxy (bulk copies); a __syncthreads must follow
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// spins until the phase of parity `parity` of the barrier has completed (returns at once for the phase before the current)
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n"
      "WAIT:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@!p bra WAIT;\n\t}" ::"r"(bar),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// one arrival, and `bytes` more transaction bytes that bulk copies must complete before the phase can
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// one arrival (counted in the barrier's init count) once every cp.async this thread issued so far has landed
__device__ __forceinline__ void cp_arrive_noinc(uint32_t bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(bar) : "memory");
}
// bytes (a multiple of 16) global -> shared, completing as transaction bytes on the barrier bar
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}

// ---- progress flags between CTAs ----------------------------------------------------------------
// release: the writes this thread has made or observed (through a __syncthreads before it) become visible at gpu scope
// to any thread whose acquire load reads the value
__device__ __forceinline__ void st_release_gpu(unsigned* p, unsigned v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned ld_acquire_gpu(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// spins until *p >= n
__device__ __forceinline__ void wait_geq(const unsigned* p, unsigned n) {
  while (ld_acquire_gpu(p) < n) {
  }
}

// ---- global memory hints ------------------------------------------------------------------------
// load of data that is read once and never written by the kernel: no L1 allocation, first out of L2.  Not volatile, so
// the compiler may move it across the stores around it.
__device__ __forceinline__ float2 ld_stream_f2(const float* src) {
  float2 v;
  asm("{\n\t.reg .b64 pol;\n\tcreatepolicy.fractional.L2::evict_first.b64 pol, 1.0;\n\t"
      "ld.global.nc.L1::no_allocate.L2::cache_hint.v2.f32 {%0, %1}, [%2], pol;\n\t}"
      : "=f"(v.x), "=f"(v.y)
      : "l"(src));
  return v;
}
// L2 cache policies, the 64-bit operand of the .L2::cache_hint forms below.  Each is one createpolicy with immediate
// operands, so the kernels create it where they use it.
// evict_last: lines a later phase of the same tile reads, which the traffic in between must not push out of L2
__device__ __forceinline__ uint64_t l2_evict_last() {
  uint64_t pol;
  asm("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
// evict_first: lines that are dead once read
__device__ __forceinline__ uint64_t l2_evict_first() {
  uint64_t pol;
  asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
// bytes (a multiple of 16) at a 16-byte aligned global address -> L2 with policy pol, asynchronously; nothing waits for it
__device__ __forceinline__ void prefetch_l2_hint(const void* src, uint32_t bytes, uint64_t pol) {
  asm volatile("cp.async.bulk.prefetch.L2.global.L2::cache_hint [%0], %1, %2;" ::"l"(src), "r"(bytes), "l"(pol) : "memory");
}

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
