// First convolution (3 -> 64 channels, K = 27) without an im2col matrix in HBM.
//
// The first version expanded the 3-channel image into im2col rows [pixels][64] in global memory
// (411 MB written by the input kernel, read by the fprop GEMM, read again by the wgrad GEMM).  Here
// eight producer warps build the 128B-swizzled operand tile DIRECTLY IN SHARED MEMORY from the
// 8-byte NHWC4 pixels (row = pixel, 64 bf16 = 27 taps*channels + zero tail; 16-byte chunk j of row r
// lives at r*128 + ((j ^ (r & 7)) << 4), exactly what a SWIZZLE_128B TMA load would have written),
// make it visible to the async proxy (fence.proxy.async) and hand it to wgmma through the same
// full/empty mbarrier ring a TMA producer would use:
//   fprop : the tile is the K-major A operand (rows = M = pixels; 64 per consumer warpgroup),
//           B = the 64x64 weight (resident), epilogue bias + ReLU -> bf16 NHWC;
//   wgrad : the same bytes are the MN-major B operand (rows = K = pixels); A = dZ via TMA (MN-major,
//           M = 64 output channels).  The two consumer warpgroups take alternate k-blocks, keep
//           their accumulators in registers over the CTA's pixel range and add them into dW
//           (PARTIAL: each stores its own slice ws[2 * CTA + consumer][64][64], zeros when it had
//           no k-block, for splitk_reduce to add up in slice order).
#pragma once
#include "umma_core.cuh"

namespace b200 {

constexpr int C0_STAGES = 4;
constexpr int C0_PROD_WARPS = 8;                                  // 256 producer threads, in row-groups
constexpr int C0_MMA_THREADS = 128 * (1 + UMMA_CONSUMERS);       // TMA warpgroup + 2 consumer warpgroups
constexpr int C0_THREADS = C0_MMA_THREADS + 32 * C0_PROD_WARPS;   // ... + 2 builder warpgroups
constexpr int C0_TILE_BYTES = 128 * 128;                          // 128 rows x 64 bf16

struct Conv0Params {
  CUtensorMap mapW;            // fprop: weight [64][64] bf16, box {64, 64}
  CUtensorMap mapZ;            // wgrad: dZ [pixels][64] bf16 as {64, pixels}, box {64, 64}
  const __nv_bfloat16* x4;     // [N][H][W][4] bf16 (3 channels + pad)
  __nv_bfloat16* out;          // fprop: [pixels][64] bf16
  const float* bias;
  float* dW;                   // wgrad: [64][64] fp32; PARTIAL: [2 * grid][64][64]
  int N, H, W;
  long long pixels;            // N*H*W
  int num_tiles;               // fprop: ceil(pixels/128); wgrad: k-blocks of 64 pixels
  int blocks_per_cta;          // wgrad: k-blocks per CTA
};

// One im2col row (pixel `pix`) into a swizzled 128-byte smem row.  32-bit index arithmetic: the
// pixel count of a batch (3.2 M at 64 x 224 x 224) is far below 2^31.
__device__ __forceinline__ void c0_build_row(const Conv0Params& p, int pix, uint8_t* tile, int r) {
  uint32_t h[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) h[i] = 0u;
  if (pix < static_cast<int>(p.pixels)) {
    const int w = pix % p.W;
    const int t = pix / p.W;
    const int hh = t % p.H;
    const uint2* base = reinterpret_cast<const uint2*>(p.x4);       // one uint2 = one NHWC4 pixel
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) {
      const int dy = tap / 3 - 1, dx = tap % 3 - 1;
      const int yy = hh + dy, xx = w + dx;
      uint2 px = make_uint2(0u, 0u);
      if (yy >= 0 && yy < p.H && xx >= 0 && xx < p.W) px = __ldg(base + (pix + dy * p.W + dx));
      h[tap * 3 + 0] = px.x & 0xffffu;
      h[tap * 3 + 1] = px.x >> 16;
      h[tap * 3 + 2] = px.y & 0xffffu;
    }
  }
  uint8_t* row = tile + r * 128;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (j < 4) v = make_uint4(h[8 * j] | (h[8 * j + 1] << 16), h[8 * j + 2] | (h[8 * j + 3] << 16),
                              h[8 * j + 4] | (h[8 * j + 5] << 16), h[8 * j + 6] | (h[8 * j + 7] << 16));
    *reinterpret_cast<uint4*>(row + ((j ^ (r & 7)) << 4)) = v;
  }
}

template <bool WGRAD, bool PARTIAL = false>
__global__ void __launch_bounds__(C0_THREADS, 1) conv0_kernel(const __grid_constant__ Conv0Params prm) {
  constexpr int ROWS = WGRAD ? 64 : 128;                       // pixels per stage
  constexpr int A_BYTES = WGRAD ? UMMA_SLAB_BYTES : 0;         // wgrad: the dZ slab
  constexpr int STAGE = C0_TILE_BYTES + A_BYTES;
  // fprop: both consumer warpgroups read every stage; wgrad: one warpgroup per stage
  constexpr int CONSUMERS_PER_STAGE = WGRAD ? 1 : UMMA_CONSUMERS;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* sW = smem + C0_STAGES * STAGE;                      // fprop: resident weight (8 KB)
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(sW + 8192);
  uint64_t* empty_bar = full_bar + C0_STAGES;
  uint64_t* w_bar = empty_bar + C0_STAGES;

  const int wg = threadIdx.x >> 7;
  const int warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) {
    for (int s = 0; s < C0_STAGES; ++s) {
      // builders arrive once per thread that writes rows; wgrad adds the TMA transaction arrival
      mbar_init(&full_bar[s], ROWS + (WGRAD ? 1 : 0));
      mbar_init(&empty_bar[s], CONSUMERS_PER_STAGE);
    }
    mbar_init(w_bar, 1);
    fence_mbar_init();
  }
  __syncthreads();

  // wgrad: this CTA's contiguous range of 64-pixel k-blocks
  const int kb0 = WGRAD ? blockIdx.x * prm.blocks_per_cta : 0;
  const int kb1 = WGRAD ? min(prm.num_tiles, kb0 + prm.blocks_per_cta) : 0;

  if (wg == 0) {
    if (warp == 0) {
      if constexpr (!WGRAD) {
        if (elect_one()) {
          tma_prefetch_desc(&prm.mapW);
          mbar_arrive_expect_tx(w_bar, 8192);
          tma_load_2d(sW, &prm.mapW, w_bar, 0, 0);
        }
      } else {
        tma_prefetch_desc(&prm.mapZ);
        uint32_t it = 0;
        for (int kb = kb0; kb < kb1; ++kb, ++it) {
          const uint32_t s = it % C0_STAGES;
          mbar_wait(&empty_bar[s], ((it / C0_STAGES) & 1) ^ 1, 41);
          if (elect_one()) {
            mbar_arrive_expect_tx(&full_bar[s], UMMA_SLAB_BYTES);
            tma_load_2d(smem + s * STAGE + C0_TILE_BYTES, &prm.mapZ, &full_bar[s], 0, kb * 64);
          }
          __syncwarp();
        }
      }
    }
  } else if (wg <= UMMA_CONSUMERS) {
    const int cw = wg - 1;
    const int t = threadIdx.x & 127;
    const int lane = t & 31;
    const int r0 = 16 * (t >> 5) + (lane >> 2);               // fragment rows r0, r0 + 8
    const int cq = 2 * (lane & 3);                            // fragment columns 8 j + cq, + 1
    float d[32];
    if constexpr (!WGRAD) {
      mbar_wait(w_bar, 0, 42);
      const uint64_t bd0 = wgmma_desc_sw128(smem_u32(sW), 16, 1024);
      uint32_t it = 0;
      for (int tile = blockIdx.x; tile < prm.num_tiles; tile += gridDim.x, ++it) {
        const uint32_t s = it % C0_STAGES;
        mbar_wait(&full_bar[s], (it / C0_STAGES) & 1, 44);
        const uint64_t ad0 = wgmma_desc_sw128(smem_u32(smem + s * STAGE) + cw * 8192, 16, 1024);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_ss<0, 0>(d, ad0 + k * 2, bd0 + k * 2, k != 0 ? 1 : 0);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_acc(d);
        if (t == 0) mbar_arrive(&empty_bar[s]);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int pix = tile * 128 + cw * 64 + r0 + 8 * h;
          if (pix < prm.pixels) {
            __nv_bfloat16* o = prm.out + static_cast<long long>(pix) * 64 + cq;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const float lo = fmaxf(d[4 * j + 2 * h] + __ldg(prm.bias + 8 * j + cq), 0.f);
              const float hi = fmaxf(d[4 * j + 2 * h + 1] + __ldg(prm.bias + 8 * j + cq + 1), 0.f);
              *reinterpret_cast<uint32_t*>(o + 8 * j) = pack_bf16x2(lo, hi);
            }
          }
        }
      }
    } else {
      uint32_t it = 0, mine = 0;
      for (int kb = kb0; kb < kb1; ++kb, ++it) {
        if (static_cast<int>(it & 1) != cw) continue;          // alternate k-blocks between the consumers
        const uint32_t s = it % C0_STAGES;
        mbar_wait(&full_bar[s], (it / C0_STAGES) & 1, 45);
        const uint32_t st = smem_u32(smem + s * STAGE);
        const uint64_t bd0 = wgmma_desc_sw128(st, UMMA_SLAB_BYTES, 1024);                    // col tile, MN-major
        const uint64_t ad0 = wgmma_desc_sw128(st + C0_TILE_BYTES, UMMA_SLAB_BYTES, 1024);    // dZ slab
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_ss<1, 1>(d, ad0 + k * 128, bd0 + k * 128, (mine | k) != 0 ? 1 : 0);
        wgmma_commit();
        wgmma_wait<0>();
        if (t == 0) mbar_arrive(&empty_bar[s]);
        ++mine;
      }
      wgmma_fence_acc(d);
      if constexpr (PARTIAL) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float* o = prm.dW + (2 * blockIdx.x + cw) * (64 * 64) + (r0 + 8 * h) * 64 + cq;
#pragma unroll
          for (int j = 0; j < 8; ++j)
            *reinterpret_cast<float2*>(o + 8 * j) =
                mine > 0 ? make_float2(d[4 * j + 2 * h], d[4 * j + 2 * h + 1]) : make_float2(0.f, 0.f);
        }
      } else if (mine > 0) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float* o = prm.dW + (r0 + 8 * h) * 64 + cq;
#pragma unroll
          for (int j = 0; j < 8; ++j)
            asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(o + 8 * j), "f"(d[4 * j + 2 * h]),
                         "f"(d[4 * j + 2 * h + 1])
                         : "memory");
        }
      }
    }
  } else {
    // ---- operand builders: swizzled im2col rows in shared memory -------------------------------
    // 256 threads in groups of ROWS (one thread per row); group g builds the stages of iterations
    // it = g, g + NGROUPS, ... so several tiles are under construction at once.
    constexpr int NGROUPS = (32 * C0_PROD_WARPS) / ROWS;
    const int pt = threadIdx.x - C0_MMA_THREADS;        // 0..255
    const int grp = pt / ROWS, r = pt % ROWS;
    if constexpr (!WGRAD) {
      uint32_t it = 0;
      for (int tile = blockIdx.x; tile < prm.num_tiles; tile += gridDim.x, ++it) {
        if (static_cast<int>(it % NGROUPS) != grp) continue;
        const uint32_t s = it % C0_STAGES;
        mbar_wait(&empty_bar[s], ((it / C0_STAGES) & 1) ^ 1, 48);
        c0_build_row(prm, tile * 128 + r, smem + s * STAGE, r);
        fence_proxy_async_smem();                        // generic-proxy stores -> visible to wgmma
        mbar_arrive(&full_bar[s]);
      }
    } else {
      uint32_t it = 0;
      for (int kb = kb0; kb < kb1; ++kb, ++it) {
        if (static_cast<int>(it % NGROUPS) != grp) continue;
        const uint32_t s = it % C0_STAGES;
        mbar_wait(&empty_bar[s], ((it / C0_STAGES) & 1) ^ 1, 49);
        c0_build_row(prm, kb * 64 + r, smem + s * STAGE, r);
        fence_proxy_async_smem();
        mbar_arrive(&full_bar[s]);
      }
    }
  }
}

}  // namespace b200
