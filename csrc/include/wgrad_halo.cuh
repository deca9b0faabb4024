// Weight gradient of a 3x3 convolution with 64 input channels (VGG features.2 / features.5),
// as nine views of ONE activation halo per pixel tile.
//
//   dW[co][tap][ci] = sum over pixels p of dZ[p][co] * X[p + tap][ci]
//
// The generic WgradPolicy gives each filter tap its own CTA and TMA-loads the shifted X tile nine
// times; with Cin = Cout = 64 that is 24 KB of operand traffic per 128 cycles of tensor work and
// the kernel sits at 22 % tensor-pipe utilisation, L2/DRAM bound.
// Here, per 8x8-pixel tile (one k-block, K = 64 pixels):
//   * X comes in once as a (8+2)x(8+2) halo box (100 rows x 128 B: one row = the 64 channels of a
//     pixel), dZ as the dense 8x8 box of one 64-channel slab;
//   * A = the tap view of X (M = 64 ci, K = pixels): tap (kh,kw) of pixel (y, x) is halo row
//     (y+kh)*10 + x+kw.  Such views do not start on a swizzle-pattern boundary, so each warp loads
//     its 16 channels of the view with ldmatrix.trans and issues wgmma with A from registers;
//     B = dZ (N = 64 co, MN-major) from shared memory;
//   * three consumer warpgroups own three taps each (kh = warpgroup); the nine 64 x 64 fp32
//     accumulators stay in registers for the CTA's whole pixel range (split-K over pixel tiles,
//     one work item per CTA);
//   * epilogue: fp32 red.add straight into dW[co][tap][ci]; PARTIAL: plain stores into the work
//     item's own slice ws[split][co][tap][ci], added up in split order by splitk_reduce.
// Operand traffic per k-block drops from 9 x 24 KB to 21 KB.
#pragma once
#include "umma_core.cuh"

namespace b200 {

constexpr int WH_T = 8;                                   // 8 x 8 pixel tile = 64 K rows
constexpr int WH_PITCH = WH_T + 2;
constexpr int WH_X_BYTES = WH_PITCH * WH_PITCH * 128;     // 12800 (TMA transaction)
constexpr int WH_X_SLOT = 13 * 1024;                      // 1 KB aligned slot
constexpr int WH_Z_BYTES = WH_T * WH_T * 128;             // 8192
constexpr int WH_STAGE = WH_X_SLOT + WH_Z_BYTES;
constexpr int WH_STAGES = 8;
constexpr int WH_CONSUMERS = 3;                           // one per filter row kh
constexpr int WH_THREADS = 128 * (1 + WH_CONSUMERS);
constexpr int WH_SMEM = WH_STAGES * WH_STAGE + 1024 + 512;
// Registers per thread (setmaxnreg; launch allocation 4 x 128): the producer warpgroup gives up what
// the consumers need for three 64 x 64 fp32 accumulators (96) and two sets of A fragments (32).
constexpr int WH_PRODUCER_REGS = 24;
constexpr int WH_CONSUMER_REGS = 160;
static_assert(WH_PRODUCER_REGS + WH_CONSUMERS * WH_CONSUMER_REGS <= 4 * (65536 / WH_THREADS), "register budgets");

struct WgradHaloParams {
  CUtensorMap mapX;        // X  {64, W, H, N}, box {64, 10, 10, 1}
  CUtensorMap mapZ;        // dZ {Cout, W, H, N}, box {64, 8, 8, 1}
  int num_items;           // tiles_n * ksplit
  int tiles_n;             // Cout / 64
  int tiles_w, tiles_h;    // W / 8, H / 8
  int total_tiles;         // N * tiles_h * tiles_w
  int tiles_per_split;
  int Cout;
  float* dW;               // [Cout][9][64] fp32; PARTIAL: [splits][Cout][9][64]
  float scale;
};

template <bool PARTIAL = false>
__global__ void __launch_bounds__(WH_THREADS, 1)
wgrad_halo64_kernel(const __grid_constant__ WgradHaloParams prm) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + WH_STAGES * WH_STAGE);
  uint64_t* empty_bar = full_bar + WH_STAGES;

  const int wg = threadIdx.x >> 7;
  const int warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&prm.mapX);
    tma_prefetch_desc(&prm.mapZ);
    for (int s = 0; s < WH_STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], WH_CONSUMERS); }
    fence_mbar_init();
  }
  __syncthreads();

  auto item_range = [&](int item, int& n_tile, int& t0, int& nk) {
    n_tile = item % prm.tiles_n;
    const int split = item / prm.tiles_n;
    t0 = split * prm.tiles_per_split;
    const int rem = prm.total_tiles - t0;
    nk = rem < 0 ? 0 : (rem < prm.tiles_per_split ? rem : prm.tiles_per_split);
  };

  if (wg == 0) {
    setmaxnreg_dec<WH_PRODUCER_REGS>();
    if (warp == 0) {
      uint32_t it = 0;
      for (int item = blockIdx.x; item < prm.num_items; item += gridDim.x) {
        int n_tile, t0, nk;
        item_range(item, n_tile, t0, nk);
        for (int i = 0; i < nk; ++i, ++it) {
          const uint32_t s = it % WH_STAGES;
          mbar_wait(&empty_bar[s], ((it / WH_STAGES) & 1) ^ 1, 31);
          const int tile = t0 + i;
          const int tw = tile % prm.tiles_w;
          const int r = tile / prm.tiles_w;
          const int th = r % prm.tiles_h;
          const int n = r / prm.tiles_h;
          if (elect_one()) {
            uint8_t* st = smem + s * WH_STAGE;
            mbar_arrive_expect_tx(&full_bar[s], WH_X_BYTES + WH_Z_BYTES);
            tma_load_4d(st, &prm.mapX, &full_bar[s], 0, tw * WH_T - 1, th * WH_T - 1, n);
            tma_load_4d(st + WH_X_SLOT, &prm.mapZ, &full_bar[s], n_tile * 64, tw * WH_T, th * WH_T, n);
          }
          __syncwarp();
        }
      }
    }
  } else {
    setmaxnreg_inc<WH_CONSUMER_REGS>();
    const int kh = wg - 1;                    // this warpgroup's taps: (kh, 0), (kh, 1), (kh, 2)
    const int t = threadIdx.x & 127;
    const int lane = t & 31, w = t >> 5;
    // ldmatrix.trans source rows: matrix j = lane / 8 covers channels 16 w + 8 (j & 1) and pixels
    // 8 (j >> 1) .. +7 of the k16 step; lane supplies pixel row (lane & 7) of it.
    const int mchunk = 2 * w + ((lane >> 3) & 1);
    const int prow = (lane >> 4) & 1;         // which of the two 8-pixel rows of a k16 step
    const int px = lane & 7;
    uint32_t it = 0;
    for (int item = blockIdx.x; item < prm.num_items; item += gridDim.x) {
      int n_tile, t0, nk;
      item_range(item, n_tile, t0, nk);
      float d[3][32];
      for (int i = 0; i < nk; ++i, ++it) {
        const uint32_t s = it % WH_STAGES;
        mbar_wait_outlined_timeout(&full_bar[s], (it / WH_STAGES) & 1, 33);   // no wgmma in flight here
        const uint32_t x0 = smem_u32(smem + s * WH_STAGE);
        const uint64_t zd0 = wgmma_desc_sw128(x0 + WH_X_SLOT, UMMA_SLAB_BYTES, 1024);
        // Two sets of A fragments: kw = 2 reloads the first set once kw = 0's wgmmas have retired.
        uint32_t af[2][4][4];
#pragma unroll
        for (int kw = 0; kw < 3; ++kw) {
          uint32_t (&f)[4][4] = af[kw & 1];
          if (kw == 2) wgmma_wait<1>();
#pragma unroll
          for (int ks = 0; ks < 4; ++ks) {   // k16 step = pixel rows 2 ks, 2 ks + 1 of the 8 x 8 tile
            const int hr = (2 * ks + prow + kh) * WH_PITCH + px + kw;
            ldmatrix_x4_trans(f[ks], x0 + sw128_offset(hr, mchunk));
          }
          wgmma_fence();
#pragma unroll
          for (int ks = 0; ks < 4; ++ks)
            wgmma_rs<1>(d[kw], f[ks], zd0 + ks * ((16 * 128) >> 4), (i | ks) != 0 ? 1 : 0);
          wgmma_commit();
        }
        wgmma_wait<0>();
        if (t == 0) mbar_arrive(&empty_bar[s]);
      }
#pragma unroll
      for (int kw = 0; kw < 3; ++kw) wgmma_fence_acc(d[kw]);
      if (nk > 0) {
        // fragment rows = ci (16 w + lane / 4, + 8), columns = co (8 j + 2 (lane & 3), + 1)
        const int ci0 = 16 * w + (lane >> 2);
        const int co0 = n_tile * 64 + 2 * (lane & 3);
        float* dW = prm.dW;
        if constexpr (PARTIAL) dW += static_cast<long long>(item / prm.tiles_n) * prm.Cout * (9 * 64);
#pragma unroll
        for (int kw = 0; kw < 3; ++kw) {
          const int tap = kh * 3 + kw;
#pragma unroll
          for (int j = 0; j < 8; ++j) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const int ci = ci0 + 8 * (e >> 1);
              const int co = co0 + 8 * j + (e & 1);
              if (co < prm.Cout) {
                float* o = dW + (static_cast<long long>(co) * 9 + tap) * 64 + ci;
                if constexpr (PARTIAL) *o = d[kw][4 * j + e] * prm.scale;
                else atomicAdd(o, d[kw][4 * j + e] * prm.scale);
              }
            }
          }
        }
      }
    }
  }
}

}  // namespace b200
