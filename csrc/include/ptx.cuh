// Thin inline-PTX wrappers for the sm_90a features the kernels use: mbarrier, TMA
// (cp.async.bulk.tensor), wgmma operand descriptors, ldmatrix, proxy fences, and the .sys-scope
// loads / stores / multimem ops used by the cross-GPU kernels.  Nothing here is portable on
// purpose: every .cu in this tree is compiled for compute_90a only.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>

#include "wgmma.cuh"

namespace b200 {

#ifndef B200_SPIN_LIMIT
// Spin bound for every device-side wait (~ seconds at 1.98 GHz).  A wait that exceeds it records
// where it was in mbar_timeout_info and traps, so a protocol bug kills the context instead of
// hanging the GPU.  No printf: a function call inside the wait loops of the wgmma kernels would make
// ptxas serialise every wgmma (warning C7510).  The record is visible in a GPU core dump
// (CUDA_ENABLE_COREDUMP_ON_EXCEPTION=1).
#define B200_SPIN_LIMIT (1ull << 31)
#endif

// {tag, block x, thread, parity} of the first wait that timed out in this module.
static __device__ uint32_t mbar_timeout_info[4];

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t lane_id() {
  uint32_t l;
  asm volatile("mov.u32 %0, %%laneid;" : "=r"(l));
  return l;
}
__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

// ------------------------------------------------------------------------------------ mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
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
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity, int tag = 0) {
  unsigned long long spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (B200_SPIN_LIMIT >> 6)) {   // try_wait itself blocks for a HW-defined slice
      if (atomicCAS(&mbar_timeout_info[0], 0u, static_cast<uint32_t>(tag) | 0x80000000u) == 0u) {
        mbar_timeout_info[1] = blockIdx.x;
        mbar_timeout_info[2] = threadIdx.x;
        mbar_timeout_info[3] = parity;
        __threadfence();
      }
      __trap();
    }
  }
}

// The same wait for warps that issue no wgmma and run under a raised setmaxnreg budget (the epilogue
// warpgroup).  A trap inlined into such a region makes ptxas keep the region within the launch
// allocation, so the timeout report and trap are out of line, after the loop.
static __device__ __noinline__ void mbar_timeout(int tag, uint32_t parity) {
  if (atomicCAS(&mbar_timeout_info[0], 0u, static_cast<uint32_t>(tag) | 0x80000000u) == 0u) {
    mbar_timeout_info[1] = blockIdx.x;
    mbar_timeout_info[2] = threadIdx.x;
    mbar_timeout_info[3] = parity;
    __threadfence();
  }
  __trap();
}
__device__ __forceinline__ void mbar_wait_outlined_timeout(uint64_t* bar, uint32_t parity, int tag) {
  unsigned long long spins = 0;
  bool ok;
  while (!(ok = mbar_try_wait(bar, parity)) && ++spins <= (B200_SPIN_LIMIT >> 6)) {
  }
  if (!ok) mbar_timeout(tag, parity);
}

// ----------------------------------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, uint64_t* bar,
                                            int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* map, uint64_t* bar,
                                            int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, const void* src, int c0,
                                             int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(map)),
               "r"(smem_u32(src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* map, const void* src, int c0,
                                             int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
          reinterpret_cast<uint64_t>(map)),
      "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;"); }
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// ------------------------------------------------------------------------------ wgmma operands
// Shared-memory matrix descriptor for wgmma, 128-byte swizzle (cute::GMMA::GmmaDescriptor):
//   [0,14) start>>4 | [16,30) LBO>>4 | [32,46) SBO>>4 | [49,52) base offset | [62,64) layout (1 = SWIZZLE_128B).
// K-major operand  (rows = M/N index, 128 B of K per row): SBO = 1024 (8 rows), LBO ignored.
// MN-major operand (rows = K index, 128 B = 64 MN elements per row): SBO = 1024 (8 K rows),
//   LBO = byte distance between consecutive 64-element MN slabs.
// Every descriptor built here starts on a 1024-byte boundary plus a K offset inside the swizzle
// row, so the base offset stays 0.  Tiles that are read at other row offsets (the halo kernels'
// tap views) are loaded into registers with ldmatrix instead.
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= 1ull << 62;                                            // SWIZZLE_128B
  return d;
}
// Byte offset of 16-byte chunk `chunk` of row `row` in a SWIZZLE_128B tile whose base is 1024-byte
// aligned (what a TMA load with CU_TENSOR_MAP_SWIZZLE_128B writes).
__device__ __forceinline__ uint32_t sw128_offset(uint32_t row, uint32_t chunk) {
  return row * 128 + ((chunk ^ (row & 7)) << 4);
}
__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}
// Barrier over a subset of the CTA's warps (ids 1..15; 0 is __syncthreads).
__device__ __forceinline__ void named_bar_sync(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}
// Per-warpgroup register budget (executed by all 128 threads of a warpgroup; N a multiple of 8 in
// [24, 256]).  The budgets of all warpgroups together must fit the allocation the kernel launched with.
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() {
  static_assert(N % 8 == 0 && N >= 24 && N <= 256, "setmaxnreg: multiple of 8 in [24, 256]");
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N));
}
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() {
  static_assert(N % 8 == 0 && N >= 24 && N <= 256, "setmaxnreg: multiple of 8 in [24, 256]");
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N));
}

// --------------------------------------------------------------------- cross-GPU memory ops
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t ld_relaxed_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void fence_acq_rel_sys() {
  asm volatile("fence.acq_rel.sys;" ::: "memory");
}
__device__ __forceinline__ uint4 ld_nc_v4(const void* p) {   // streaming 16-byte load
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p));
  return v;
}
__device__ __forceinline__ uint4 ld_relaxed_sys_v4(const void* p) {   // peer data written this step
  uint4 v;
  asm volatile("ld.relaxed.sys.global.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p)
               : "memory");
  return v;
}
__device__ __forceinline__ void st_v4(void* p, uint4 v) {
  asm volatile("st.global.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z),
               "r"(v.w)
               : "memory");
}
// NVLS: the switch reduces 8 bf16 (as 4 x bf16x2, fp32 accumulation) across all devices bound
// to the multicast address, and broadcasts a 16-byte store to all of them.
__device__ __forceinline__ uint4 multimem_ld_reduce_bf16x8(const void* mc_ptr) {
  uint4 v;
  asm volatile(
      "multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0, %1, %2, %3}, [%4];"
      : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
      : "l"(mc_ptr)
      : "memory");
  return v;
}
__device__ __forceinline__ float4 multimem_ld_reduce_f32x4(const void* mc_ptr) {
  float4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(mc_ptr)
               : "memory");
  return v;
}
__device__ __forceinline__ void multimem_st_v4(void* mc_ptr, uint4 v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(mc_ptr),
               "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w)
               : "memory");
}
__device__ __forceinline__ void multimem_red_add_u32(uint32_t* mc_ptr, uint32_t v) {
  asm volatile("multimem.red.release.sys.global.add.u32 [%0], %1;" ::"l"(mc_ptr), "r"(v)
               : "memory");
}

// ------------------------------------------------------------------------------- bf16 helpers
// 32-byte global accesses as two 16-byte vector instructions.  An epilogue thread owns 64
// contiguous bytes of one pixel while its neighbours own other pixels; writing a full 32-byte
// sector per pair keeps every sector it touches complete.  The address must be 32-byte aligned.
__device__ __forceinline__ void st_global_v8(void* p, const uint32_t (&v)[8]) {
  asm volatile("st.global.v4.b32 [%0], {%1,%2,%3,%4};\n\t"
               "st.global.v4.b32 [%0+16], {%5,%6,%7,%8};" ::"l"(p), "r"(v[0]), "r"(v[1]), "r"(v[2]),
               "r"(v[3]), "r"(v[4]), "r"(v[5]), "r"(v[6]), "r"(v[7])
               : "memory");
}
__device__ __forceinline__ void ld_global_nc_v8(const void* p, uint32_t* v) {
  asm volatile("ld.global.nc.v4.b32 {%0,%1,%2,%3}, [%8];\n\t"
               "ld.global.nc.v4.b32 {%4,%5,%6,%7}, [%8+16];"
               : "=r"(v[0]), "=r"(v[1]), "=r"(v[2]), "=r"(v[3]), "=r"(v[4]), "=r"(v[5]), "=r"(v[6]), "=r"(v[7])
               : "l"(p));
}

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 t = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&t);
}
__device__ __forceinline__ uint32_t max_bf16x2(uint32_t a, uint32_t b) {
  uint32_t d;
  asm("max.bf16x2 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b));
  return d;
}
__device__ __forceinline__ float2 unpack_bf16x2(uint32_t v) {
  __nv_bfloat162 t = *reinterpret_cast<__nv_bfloat162*>(&v);
  return __bfloat1622float2(t);
}

}  // namespace b200
