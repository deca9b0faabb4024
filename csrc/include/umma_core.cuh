// One persistent, warp-specialised wgmma pipeline shared by the GEMM-shaped kernels in this tree
// (FC fwd/dgrad/wgrad, conv fprop/dgrad/wgrad, the layer-0 im2col GEMM).
//
// One CTA per SM loops over output tiles (tile = blockIdx.x, += gridDim.x):
//   warpgroup 0      TMA producer (one warp): runs ahead across tile boundaries; waits "empty[s]",
//                    arms "full[s]" with the stage byte count, issues the policy's
//                    cp.async.bulk.tensor loads.
//   warpgroups 1, 2  consumers: warpgroup c owns rows [64c, 64c+64) of the 128 x BN tile and keeps
//                    its fp32 accumulator in registers.  Per k-block it waits "full[s]", issues four
//                    wgmma.m64nBNk16 (two m64n128k16 per k16 step at BN = 256), and releases the
//                    previous stage once its wgmmas retired (one group stays in flight).  After
//                    the tile's last k-block it writes the accumulator into the shared staging
//                    tile, one chunk of stage_cols<BN>() columns at a time ("stage_empty" ->
//                    write -> "stage_full"), and goes straight on to the next tile's k-blocks.
//   warpgroup 3      epilogue: thread t takes row t of each staged chunk into registers,
//                    releases the chunk and runs the policy's epilogue on it, so the policy sees
//                    the row-major fragments it expects: one row and 32 consecutive columns per
//                    call, a warp holding 32 consecutive rows.  It overlaps the next tile's MMAs.
// setmaxnreg moves registers from the producer to the consumers and the epilogue (RoleRegs).
//
// Tile: 128 (M) x BN (N), BK = 64 bf16 = one 128-byte swizzle row.  Operands are staged in the
// canonical SWIZZLE_128B layouts, K-major (rows = M/N index) or MN-major (rows = K index,
// 64-element slabs) -- see ptx.cuh.  Either way the second consumer's half of A starts 8 KB in.
//
// A Policy provides:
//   static constexpr int  BN, STAGES;  static constexpr bool A_MN, B_MN;
//   struct Params (POD, holds CUtensorMaps and `int num_tiles`; passed __grid_constant__);
//   struct Ctx;
//   __device__ static void prefetch(const Params&);
//   __device__ static Ctx  make_ctx(const Params&, int tile);
//   __device__ static int  num_k_iters(const Params&, const Ctx&);
//   __device__ static void load(const Params&, const Ctx&, int kiter, uint8_t* sA, uint8_t* sB,
//                               uint64_t* full_bar);                                  // one thread
//   struct RowCtx;  __device__ static RowCtx row_ctx(const Params&, const Ctx&, int row);
//                                                   // per-thread, per-tile address arithmetic
//   __device__ static void epilogue(const Params&, const Ctx&, const RowCtx&, int row, int col0,
//                                   const uint32_t (&acc)[32], float* epi_smem);
//                                                                 // row in [0,128), 32 columns
//   static constexpr bool PREMASK;      // true: where masked(prm), load_mask(prm, ctx, rc, col0, m[16])
//                                       // fetches what the epilogue's `const uint32_t* premask` takes
//   static constexpr int EPI_SMEM;                                // bytes of epilogue scratch
//   __device__ static void epi_begin(const Params&, float* epi_smem, int tid);  // tid in [0,128)
//   __device__ static void epi_end(const Params&, float* epi_smem, int tid);    // after all tiles
#pragma once
#include <type_traits>

#include "ptx.cuh"

namespace b200 {

constexpr int UMMA_BM = 128;
constexpr int UMMA_BK = 64;                           // elements per k-block (128 bytes of bf16)
constexpr int UMMA_A_BYTES = UMMA_BM * UMMA_BK * 2;   // 16 KB per stage
constexpr int UMMA_SLAB_BYTES = 64 * 128;             // one MN-major slab: 64 k-rows x 128 B
constexpr int UMMA_CONSUMERS = 2;                     // consumer warpgroups, 64 rows each
constexpr int UMMA_EPI_THREADS = 128;                 // the epilogue warpgroup
constexpr int UMMA_THREADS = 128 * (1 + UMMA_CONSUMERS) + UMMA_EPI_THREADS;
constexpr int UMMA_LAUNCH_REGS = 65536 / UMMA_THREADS;   // __launch_bounds__(UMMA_THREADS, 1): 128
constexpr int UMMA_MAX_SMEM = 227 * 1024;             // H100: opt-in shared memory per block
constexpr int UMMA_BAR_BYTES = 256;                   // full[STAGES], empty[STAGES], stage_full, stage_empty

// Staging tile: each consumer hands its 64 accumulator rows to the epilogue warpgroup one chunk of
// stage_cols columns at a time.  64 columns up to BN = 128.  At BN = 256 the chunk is 32 columns:
// the two 17 KB staging halves of a 64-column chunk would leave room for only three 48 KB stages,
// and the epilogue's 120 registers (RoleRegs<256>) hold one 32-column row, not a 64-column one.
// The row pitch of 4 extra floats makes the epilogue's float4 row reads conflict-free.
template <int BN>
__host__ __device__ constexpr int stage_cols() { return BN >= 256 ? 32 : 64; }
template <int BN>
__host__ __device__ constexpr int stage_ld() { return stage_cols<BN>() + 4; }
template <int BN>
__host__ __device__ constexpr int stage_bytes() { return 64 * stage_ld<BN>() * 4; }   // one consumer's rows

template <int BN>
__host__ __device__ constexpr int umma_b_bytes() { return BN * UMMA_BK * 2; }
// Pipeline depth: as many stages as fit next to the staging tile, the barriers and the epilogue
// scratch, <= 8.
template <int BN, int EPI_SMEM>
__host__ __device__ constexpr int umma_stages() {
  constexpr int room = UMMA_MAX_SMEM - 1024 - UMMA_BAR_BYTES - UMMA_CONSUMERS * stage_bytes<BN>() - EPI_SMEM;
  constexpr int s = room / (UMMA_A_BYTES + umma_b_bytes<BN>());
  return s > 8 ? 8 : s;
}
template <int BN, int STAGES>
__host__ __device__ constexpr int umma_smem_bytes() {
  static_assert((2 * STAGES + 2) * 8 <= UMMA_BAR_BYTES, "mbarriers");
  static_assert(STAGES >= 4, "the operand ring keeps at least four stages at every tile width");
  return STAGES * (UMMA_A_BYTES + umma_b_bytes<BN>()) + UMMA_CONSUMERS * stage_bytes<BN>() +
         1024 /*alignment slack*/ + UMMA_BAR_BYTES;
}

// Registers per thread of each warpgroup role (setmaxnreg; multiples of 8 that add up to the launch
// allocation of 4 x 128).  The producer is one converged warp with a few counters.  A consumer holds
// BN / 2 accumulator registers (plus, in the halo kernel, two sets of A fragments) and nothing else.
// The epilogue warpgroup gets the rest: it holds one staged row (64 registers up to BN = 128, 32 at
// BN = 256), the prefetched ReLU mask and, in the 64-channel halo dgrad, 64 running column sums.
// At BN = 256 the producer drops to the minimum so that a consumer can hold its 128 accumulator
// registers with room for descriptors and counters.
template <int BN>
struct RoleRegs {
  static constexpr int PRODUCER = BN >= 256 ? 24 : 40;
  static constexpr int CONSUMER = BN >= 256 ? 184 : (BN >= 128 ? 152 : 128);
  static constexpr int EPILOGUE = 4 * UMMA_LAUNCH_REGS - PRODUCER - UMMA_CONSUMERS * CONSUMER;
  static_assert(EPILOGUE % 8 == 0 && EPILOGUE >= 24 && EPILOGUE <= 256, "register budgets");
};
template <int N>
__device__ __forceinline__ void set_role_regs() {
  if constexpr (N > UMMA_LAUNCH_REGS) setmaxnreg_inc<N>();
  else if constexpr (N < UMMA_LAUNCH_REGS) setmaxnreg_dec<N>();
}

// Accumulator columns [c0, c0 + COLS) of a warpgroup (wgmma fragment layout) -> stage[64][COLS + 4].
// Fragment: d[i] is row 16 * warp + lane / 4 + 8 * ((i >> 1) & 1), column 8 * (i >> 2) + 2 * (lane & 3) + (i & 1).
template <int NACC, int COLS>
__device__ __forceinline__ void stage_acc_chunk(const float (&d)[NACC], int c0, float* stage, int t) {
  constexpr int LD = COLS + 4;
  const int w = t >> 5, l = t & 31;
  const int r = 16 * w + (l >> 2);
  const int cq = 2 * (l & 3);
#pragma unroll
  for (int i = 0; i < NACC; i += 4) {
    const int col = 8 * (i >> 2);
    if (col >= c0 && col < c0 + COLS) {
      *reinterpret_cast<float2*>(stage + r * LD + col - c0 + cq) = make_float2(d[i], d[i + 1]);
      *reinterpret_cast<float2*>(stage + (r + 8) * LD + col - c0 + cq) = make_float2(d[i + 2], d[i + 3]);
    }
  }
}
template <int LD>
__device__ __forceinline__ void stage_read_row(const float* stage, int row_local, int col, uint32_t (&acc)[32]) {
  const float4* src = reinterpret_cast<const float4*>(stage + row_local * LD + col);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float4 v = src[j];
    acc[4 * j] = __float_as_uint(v.x); acc[4 * j + 1] = __float_as_uint(v.y);
    acc[4 * j + 2] = __float_as_uint(v.z); acc[4 * j + 3] = __float_as_uint(v.w);
  }
}

// Consumer side of the hand-off: warpgroup `cw`'s accumulator into its half of the staging tile,
// one chunk after the other.  `eph` counts the chunks handed over (parity of stage_empty).
template <int BN, int TAG>
__device__ __forceinline__ void stage_put(const float (&d)[BN / 2], float* stage_base, int cw, int t,
                                          uint64_t* stage_full, uint64_t* stage_empty, uint32_t& eph) {
  constexpr int COLS = stage_cols<BN>();
  float* stage = stage_base + cw * (stage_bytes<BN>() / 4);
#pragma unroll
  for (int c0 = 0; c0 < BN; c0 += COLS) {
    mbar_wait(stage_empty, eph ^ 1, TAG);     // the epilogue has read the previous chunk
    eph ^= 1;
    stage_acc_chunk<BN / 2, COLS>(d, c0, stage, t);
    __syncwarp();
    if ((t & 31) == 0) mbar_arrive(stage_full);   // one arrival per consumer warp
  }
}
// Epilogue side: row t of the staged chunk, in 32-column halves (a 64-column chunk's second half
// only when the tile is that wide), into registers; then the chunk is released.  `fph` is
// stage_full's parity.
template <int BN, int TAG>
__device__ __forceinline__ void stage_take(const float* stage_base, int c0, int t, uint64_t* stage_full,
                                           uint64_t* stage_empty, uint32_t& fph,
                                           uint32_t (&acc)[stage_cols<BN>() / 32][32]) {
  constexpr int LD = stage_ld<BN>();
  mbar_wait_outlined_timeout(stage_full, fph, TAG);
  fph ^= 1;
  const float* stage = stage_base + (t >> 6) * (stage_bytes<BN>() / 4);
#pragma unroll
  for (int h = 0; h < stage_cols<BN>() / 32; ++h)
    if (c0 + 32 * h < BN) stage_read_row<LD>(stage, t & 63, 32 * h, acc[h]);
  __syncwarp();
  if ((t & 31) == 0) mbar_arrive(stage_empty);    // one arrival per epilogue warp
}
constexpr uint32_t STAGE_FULL_ARRIVALS = UMMA_CONSUMERS * 4;
constexpr uint32_t STAGE_EMPTY_ARRIVALS = UMMA_EPI_THREADS / 32;

// A policy whose A box may hold fewer than UMMA_BM rows (ConvPolicy<..., FILL = true>) declares
// FILL_BOX = true and carries the bytes one A box delivers in Params::a_tx; every other policy's
// stage transaction is the constant UMMA_A_BYTES + B bytes.
template <class P, class = void>
struct umma_fill_box : std::false_type {};
template <class P>
struct umma_fill_box<P, std::enable_if_t<P::FILL_BOX>> : std::true_type {};

template <class P>
__global__ void __launch_bounds__(UMMA_THREADS, 1)
umma_kernel(const __grid_constant__ typename P::Params prm) {
  constexpr int BN = P::BN;
  constexpr int STAGES = P::STAGES;
  constexpr int B_BYTES = umma_b_bytes<BN>();
  constexpr uint32_t STAGE_TX = UMMA_A_BYTES + B_BYTES;
  using Regs = RoleRegs<BN>;
  static_assert(BN % 32 == 0 && BN >= 32 && BN <= 256, "tile N must be a multiple of 32 in [32,256]");
  static_assert(!P::B_MN || BN % 64 == 0, "MN-major B is staged in 64-wide slabs");

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* sA = smem;
  uint8_t* sB = smem + STAGES * UMMA_A_BYTES;
  float* stage_base = reinterpret_cast<float*>(sB + STAGES * B_BYTES);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(stage_base) + UMMA_CONSUMERS * stage_bytes<BN>());
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* stage_full = empty_bar + STAGES;
  uint64_t* stage_empty = stage_full + 1;
  float* epi_smem = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(full_bar) + UMMA_BAR_BYTES);

  const int wg = threadIdx.x >> 7;
  const int warp = threadIdx.x >> 5;

  if (threadIdx.x == 0) {
    P::prefetch(prm);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], UMMA_CONSUMERS);   // one arrival per consumer warpgroup
    }
    mbar_init(stage_full, STAGE_FULL_ARRIVALS);
    mbar_init(stage_empty, STAGE_EMPTY_ARRIVALS);
    fence_mbar_init();
  }
  __syncthreads();
  const int num_tiles = prm.num_tiles;

  if (wg == 0) {
    set_role_regs<Regs::PRODUCER>();
    // The producer warp runs CONVERGED (all 32 lanes execute the loop and poll the barriers); only
    // the TMA instructions themselves are predicated on elect.sync, so addresses stay warp-uniform.
    if (warp == 0) {
      uint32_t s = 0, ph = 0;                 // ring position / phase kept as counters (no div/mod)
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const typename P::Ctx ctx = P::make_ctx(prm, tile);
        const int nk = P::num_k_iters(prm, ctx);
        for (int i = 0; i < nk; ++i) {
          mbar_wait(&empty_bar[s], ph ^ 1, 1);
          if (elect_one()) {
            if constexpr (umma_fill_box<P>::value)
              mbar_arrive_expect_tx(&full_bar[s], prm.a_tx + B_BYTES);
            else
              mbar_arrive_expect_tx(&full_bar[s], STAGE_TX);
            P::load(prm, ctx, i, sA + s * UMMA_A_BYTES, sB + s * B_BYTES, &full_bar[s]);
          }
          __syncwarp();
          if (++s == STAGES) { s = 0; ph ^= 1; }
        }
      }
    }
  } else if (wg <= UMMA_CONSUMERS) {
    set_role_regs<Regs::CONSUMER>();
    const int cw = wg - 1;                    // consumer index: rows [64 cw, 64 cw + 64) of the tile
    const int t = threadIdx.x & 127;
    // byte step per k16: K-major -> 32 B inside the swizzle row; MN-major -> 16 k-rows.
    constexpr uint32_t A_KSTEP = P::A_MN ? 16 * 128 : 32;
    constexpr uint32_t B_KSTEP = P::B_MN ? 16 * 128 : 32;
    constexpr uint32_t A_LBO = P::A_MN ? UMMA_SLAB_BYTES : 16;
    constexpr uint32_t B_LBO = P::B_MN ? UMMA_SLAB_BYTES : 16;
    // Stage descriptors are base + s * stage size: the address field is addr >> 4 and shared
    // memory is < 256 KB, so the add never carries out of the 14-bit field.
    const uint64_t ad_base = wgmma_desc_sw128(smem_u32(sA) + cw * 8192, A_LBO, 1024);
    const uint64_t bd_base = wgmma_desc_sw128(smem_u32(sB), B_LBO, 1024);
    uint32_t s = 0, ph = 0, prev = 0, eph = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const typename P::Ctx ctx = P::make_ctx(prm, tile);
      const int nk = P::num_k_iters(prm, ctx);
      float d[BN / 2];
      for (int i = 0; i < nk; ++i) {
        mbar_wait(&full_bar[s], ph, 2);
        const uint64_t ad0 = ad_base + s * (UMMA_A_BYTES >> 4);
        const uint64_t bd0 = bd_base + s * (B_BYTES >> 4);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < UMMA_BK / 16; ++k) {   // start-address field is in 16-byte units
          const uint64_t ad = ad0 + k * (A_KSTEP >> 4), bd = bd0 + k * (B_KSTEP >> 4);
          const int acc = (i | k) != 0 ? 1 : 0;
          if constexpr (BN == 256) {
            // Two m64n128 halves: ptxas needs 154 registers for one m64n256 instruction and checks
            // that against the 128-register launch allocation, whatever setmaxnreg raised it to.
            // Columns 128..255 of B start 16 KB in, both K-major (rows) and MN-major (slabs 2, 3);
            // d[64 + i] is then column 128 + the column of d[i], the m64n256 fragment layout.
            constexpr uint32_t B_HALF = (128 * 128) >> 4;
            wgmma_ss<P::A_MN ? 1 : 0, P::B_MN ? 1 : 0>(*reinterpret_cast<float(*)[64]>(d), ad, bd, acc);
            wgmma_ss<P::A_MN ? 1 : 0, P::B_MN ? 1 : 0>(*reinterpret_cast<float(*)[64]>(d + 64), ad, bd + B_HALF, acc);
          } else {
            wgmma_ss<P::A_MN ? 1 : 0, P::B_MN ? 1 : 0>(d, ad, bd, acc);
          }
        }
        wgmma_commit();
        wgmma_wait<1>();                      // the previous k-block's wgmmas have retired
        if (i > 0 && t == 0) mbar_arrive(&empty_bar[prev]);
        prev = s;
        if (++s == STAGES) { s = 0; ph ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_fence_acc(d);
      if (nk > 0) {
        if (t == 0) mbar_arrive(&empty_bar[prev]);
        stage_put<BN, 3>(d, stage_base, cw, t, stage_full, stage_empty, eph);
      }
    }
  } else {
    set_role_regs<Regs::EPILOGUE>();
    const int t = threadIdx.x & 127;          // row t of the tile
    if constexpr (P::EPI_SMEM > 0) {
      P::epi_begin(prm, epi_smem, t);
      named_bar_sync(1, UMMA_EPI_THREADS);
    }
    constexpr int COLS = stage_cols<BN>();
    constexpr int HALVES = COLS / 32;
    uint32_t fph = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const typename P::Ctx ctx = P::make_ctx(prm, tile);
      if (P::num_k_iters(prm, ctx) == 0) continue;
      const typename P::RowCtx rc = P::row_ctx(prm, ctx, t);
#pragma unroll
      for (int c0 = 0; c0 < BN; c0 += COLS) {
        uint32_t acc[HALVES][32];
        if constexpr (P::PREMASK) {
          // the mask does not depend on the accumulator: fetch it while the MMAs still run
          uint32_t pm[HALVES][16];
          const bool masked = P::masked(prm);
          if (masked) {
#pragma unroll
            for (int h = 0; h < HALVES; ++h)
              if (c0 + 32 * h < BN) P::load_mask(prm, ctx, rc, c0 + 32 * h, pm[h]);
          }
          stage_take<BN, 4>(stage_base, c0, t, stage_full, stage_empty, fph, acc);
#pragma unroll
          for (int h = 0; h < HALVES; ++h)
            if (c0 + 32 * h < BN) P::epilogue(prm, ctx, rc, t, c0 + 32 * h, acc[h], epi_smem, pm[h]);
        } else {
          stage_take<BN, 4>(stage_base, c0, t, stage_full, stage_empty, fph, acc);
#pragma unroll
          for (int h = 0; h < HALVES; ++h)
            if (c0 + 32 * h < BN) P::epilogue(prm, ctx, rc, t, c0 + 32 * h, acc[h], epi_smem);
        }
      }
    }
    if constexpr (P::EPI_SMEM > 0) {
      named_bar_sync(1, UMMA_EPI_THREADS);
      P::epi_end(prm, epi_smem, t);
    }
  }
}

}  // namespace b200
