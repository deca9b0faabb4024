// Halo-tile 3x3 convolution (fprop / dgrad) for the large-spatial layers.
//
// The generic ConvPolicy issues nine TMA loads of the same activation pixels (one per filter tap)
// per 64-channel chunk, which makes the early VGG layers (64/128 channels, 224^2 / 112^2 pixels)
// L2-bandwidth bound: 16 KB of A per 128x64x64 MMA block.  Here one TMA box brings the (8+2) x
// (16+2) pixel halo of an 8 x 16 output tile into shared memory ONCE per channel chunk (23 KB),
// and the nine taps are nine *views* of it: tap (kh, kw) of output pixel (h, w) is halo row
// (h + kh) * 10 + w + kw.  Such views start at arbitrary 128-byte rows, which a wgmma descriptor
// cannot express, so each consumer warp loads its 16 rows of the view with ldmatrix (swizzle
// applied by hand, sw128_offset) and issues wgmma with A from registers; B comes from shared
// memory as usual.  A traffic drops 6.25x.
//
// Two rings instead of one: A halos (NA slots) and B weight tiles (NB slots, one per (tap, chunk)).
// When all 9 * chunks weight tiles fit in the B ring and there is a single channel tile, they are
// loaded once per CTA and stay resident for every tile the persistent CTA processes.
//
// Warp roles (producer, two consumers, epilogue warpgroup), the staging hand-off and the epilogue
// (bias / ReLU / ReLU-mask / fused column sum, shared with ConvPolicy) are those of umma_core.cuh.
#pragma once
#include "umma_policies.cuh"

namespace b200 {

constexpr int HALO_WT = 8;                    // output tile: 8 (w) x 16 (h) pixels = 128 rows
constexpr int HALO_HT = 16;
constexpr int HALO_PITCH = HALO_WT + 2;       // halo rows per image row
constexpr int HALO_ROWS = HALO_PITCH * (HALO_HT + 2);       // 180
constexpr int HALO_BYTES = HALO_ROWS * 128;                 // 23040 (TMA transaction size)
constexpr int HALO_SLOT = 23 * 1024;                        // 1 KB aligned slot

template <int BN>
struct HaloCfg {
  static constexpr int NA = BN >= 128 ? 2 : 3;
  static constexpr int B_SLOT = BN * 128;
  static constexpr int BAR_BYTES = 512;       // a_full/a_empty[NA], b_full/b_empty[NB], stage_full, stage_empty
  static constexpr int EPI_MAX = 2048;        // ConvPolicy::EPI_SMEM
  static constexpr int ROOM = UMMA_MAX_SMEM - NA * HALO_SLOT - UMMA_CONSUMERS * stage_bytes<BN>() - 1024 - BAR_BYTES - EPI_MAX;
  static constexpr int NB = ROOM / B_SLOT > 18 ? 18 : ROOM / B_SLOT;
  static constexpr int SMEM = NA * HALO_SLOT + NB * B_SLOT + UMMA_CONSUMERS * stage_bytes<BN>() + 1024 + BAR_BYTES;
  static_assert((2 * NA + 2 * NB + 2) * 8 <= BAR_BYTES, "mbarriers");
};

template <int BN, bool DGRAD, bool POOL = false>
__global__ void __launch_bounds__(UMMA_THREADS, 1)
conv_halo_kernel(const __grid_constant__ ConvParams prm) {
  using Cfg = HaloCfg<BN>;
  using Epi = ConvPolicy<BN, 1, DGRAD, POOL>;
  constexpr int NA = Cfg::NA, NB = Cfg::NB, B_SLOT = Cfg::B_SLOT;
  using Regs = RoleRegs<BN>;
  static_assert(Epi::EPI_SMEM <= Cfg::EPI_MAX, "epilogue scratch");
  // A fragments of the next tap are loaded while the previous tap's wgmmas run (two buffers) where
  // the accumulator leaves registers for it.
  constexpr bool AFRAG_DB = BN <= 128;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* sA = smem;
  uint8_t* sB = smem + NA * HALO_SLOT;
  float* stage_base = reinterpret_cast<float*>(sB + NB * B_SLOT);
  uint64_t* a_full = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(stage_base) + UMMA_CONSUMERS * stage_bytes<BN>());
  uint64_t* a_empty = a_full + NA;
  uint64_t* b_full = a_empty + NA;
  uint64_t* b_empty = b_full + NB;
  uint64_t* stage_full = b_empty + NB;
  uint64_t* stage_empty = stage_full + 1;
  float* epi_smem = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(a_full) + Cfg::BAR_BYTES);

  const int wg = threadIdx.x >> 7;
  const int warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&prm.mapA);
    tma_prefetch_desc(&prm.mapB);
    for (int s = 0; s < NA; ++s) { mbar_init(&a_full[s], 1); mbar_init(&a_empty[s], UMMA_CONSUMERS); }
    for (int s = 0; s < NB; ++s) { mbar_init(&b_full[s], 1); mbar_init(&b_empty[s], UMMA_CONSUMERS); }
    mbar_init(stage_full, STAGE_FULL_ARRIVALS);
    mbar_init(stage_empty, STAGE_EMPTY_ARRIVALS);
    fence_mbar_init();
  }
  __syncthreads();
  const int num_tiles = prm.num_tiles;
  const int cchunks = prm.Ca / UMMA_BK;
  const bool resident = prm.resident != 0;

  if (wg == 0) {
    set_role_regs<Regs::PRODUCER>();
    if (warp == 0) {                             // converged producer warp, elect.sync-predicated issue
      uint32_t a = 0, aph = 0, bs = 0, bph = 0;  // ring positions / phases as counters
      bool first = true;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const typename Epi::Ctx ctx = Epi::make_ctx(prm, tile);
        for (int c = 0; c < cchunks; ++c) {
          mbar_wait(&a_empty[a], aph ^ 1, 21);
          if (elect_one()) {
            mbar_arrive_expect_tx(&a_full[a], HALO_BYTES);
            tma_load_4d(sA + a * HALO_SLOT, &prm.mapA, &a_full[a], c * UMMA_BK, ctx.w0 - 1, ctx.h0 - 1, ctx.n0);
          }
          __syncwarp();
          if (++a == NA) { a = 0; aph ^= 1; }
          if (resident && !first) continue;
          for (int tap = 0; tap < 9; ++tap) {
            uint32_t b;
            if (resident) {
              b = c * 9 + tap;
            } else {
              b = bs;
              mbar_wait(&b_empty[b], bph ^ 1, 22);
              if (++bs == NB) { bs = 0; bph ^= 1; }
            }
            if (elect_one()) {
              mbar_arrive_expect_tx(&b_full[b], B_SLOT);
              uint8_t* dst = sB + b * B_SLOT;
              if constexpr (!DGRAD) {
                tma_load_2d(dst, &prm.mapB, &b_full[b], tap * prm.wcols_per_tap + c * UMMA_BK, ctx.c0);
              } else {
                const int wt = 8 - tap;
#pragma unroll
                for (int j = 0; j < BN / 64; ++j)
                  tma_load_2d(dst + j * UMMA_SLAB_BYTES, &prm.mapB, &b_full[b],
                              wt * prm.wcols_per_tap + ctx.c0 + 64 * j, c * UMMA_BK);
              }
            }
            __syncwarp();
          }
        }
        first = false;
      }
    }
  } else if (wg <= UMMA_CONSUMERS) {
    set_role_regs<Regs::CONSUMER>();
    const int cw = wg - 1;
    const int t = threadIdx.x & 127;
    const int lane = t & 31;
    constexpr uint32_t B_KSTEP = DGRAD ? 16 * 128 : 32;
    constexpr uint32_t B_LBO = DGRAD ? UMMA_SLAB_BYTES : 16;
    const uint64_t bd_base = wgmma_desc_sw128(smem_u32(sB), B_LBO, 1024);
    // ldmatrix row of this lane: tile row 64 cw + 16 warp + (lane & 15) = pixel (h, w) of the 8 x 16
    // tile; k half (lane >> 4).  Its halo row for tap (kh, kw) is hrow0 + kh * 10 + kw.
    const int trow = cw * 64 + 16 * (t >> 5) + (lane & 15);
    const int hrow0 = (trow >> 3) * HALO_PITCH + (trow & 7);
    const int khalf = lane >> 4;
    uint32_t a = 0, aph = 0, bs = 0, bph = 0, eph = 0;
    bool first = true;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      float d[BN / 2];
      for (int c = 0; c < cchunks; ++c) {
        mbar_wait(&a_full[a], aph, 25);
        const uint32_t abase = smem_u32(sA + a * HALO_SLOT);
        const bool steady = resident && !first;
        uint32_t prevb = 0;
        uint32_t af[2][4][4];
#pragma unroll
        for (int tap = 0; tap < 9; ++tap) {
          uint32_t b;
          if (resident) {
            b = c * 9 + tap;
            if (!steady) mbar_wait(&b_full[b], 0, 26);      // first tile of this CTA: weights still arriving
          } else {
            b = bs;
            mbar_wait(&b_full[b], bph, 27);
            if (++bs == NB) { bs = 0; bph ^= 1; }
          }
          const int hr = hrow0 + (tap / 3) * HALO_PITCH + tap % 3;
          uint32_t (&f)[4][4] = af[AFRAG_DB ? (tap & 1) : 0];
#pragma unroll
          for (int ks = 0; ks < 4; ++ks) ldmatrix_x4(f[ks], abase + sw128_offset(hr, 2 * ks + khalf));
          const uint64_t bd = bd_base + b * (B_SLOT >> 4);
          wgmma_fence();
#pragma unroll
          for (int ks = 0; ks < 4; ++ks)
            wgmma_rs<DGRAD ? 1 : 0>(d, f[ks], bd + ks * (B_KSTEP >> 4), (c | tap | ks) != 0 ? 1 : 0);
          wgmma_commit();
          if constexpr (AFRAG_DB) wgmma_wait<1>(); else wgmma_wait<0>();
          if (!resident && tap > 0 && t == 0) mbar_arrive(&b_empty[prevb]);
          prevb = b;
        }
        wgmma_wait<0>();
        if (t == 0) {
          if (!resident) mbar_arrive(&b_empty[prevb]);
          mbar_arrive(&a_empty[a]);
        }
        if (++a == NA) { a = 0; aph ^= 1; }
      }
      first = false;
      wgmma_fence_acc(d);
      stage_put<BN, 23>(d, stage_base, cw, t, stage_full, stage_empty, eph);
    }
  } else {
    set_role_regs<Regs::EPILOGUE>();
    const int t = threadIdx.x & 127;          // row t of the tile
    const int lane = t & 31;
    if constexpr (Epi::EPI_SMEM > 0) {
      Epi::epi_begin(prm, epi_smem, t);
      named_bar_sync(1, UMMA_EPI_THREADS);
    }
    // Fused bias gradient with a single channel tile (the 64-channel layers): every tile of this
    // CTA lands on the same columns, so a thread keeps running sums of what it stored and the
    // warp transpose-reduce runs once per kernel instead of once per tile.
    float keep[2][32];
    const bool keep_on = DGRAD && BN == 64 && (prm.flags & CONV_COLSUM) && prm.Cn <= BN;
#pragma unroll
    for (int i = 0; i < 32; ++i) keep[0][i] = keep[1][i] = 0.f;
    const bool masked = Epi::masked(prm);
    uint32_t fph = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const typename Epi::Ctx ctx = Epi::make_ctx(prm, tile);
      const typename Epi::RowCtx rc = Epi::row_ctx(prm, ctx, t);
#pragma unroll
      for (int c0 = 0; c0 < BN; c0 += 64) {
        // the mask does not depend on the accumulator: fetch it while the MMAs still run
        uint32_t pm[2][16];
        if (masked) {
          Epi::load_mask(prm, ctx, rc, c0, pm[0]);
          Epi::load_mask(prm, ctx, rc, c0 + 32, pm[1]);
        }
        uint32_t acc[2][32];
        stage_take<BN, 24>(stage_base, c0, t, stage_full, stage_empty, fph, acc);
#pragma unroll
        for (int h = 0; h < 2; ++h)
          Epi::epilogue(prm, ctx, rc, t, c0 + 32 * h, acc[h], epi_smem, pm[h], keep[h], keep_on);
      }
    }
    if constexpr (DGRAD) {
      if (keep_on) {
        Epi::colsum_flush(prm, 0, lane, keep[0], epi_smem);
        Epi::colsum_flush(prm, 32, lane, keep[1], epi_smem);
      }
    }
    if constexpr (Epi::EPI_SMEM > 0) {
      named_bar_sync(1, UMMA_EPI_THREADS);
      Epi::epi_end(prm, epi_smem, t);
    }
  }
}

}  // namespace b200
