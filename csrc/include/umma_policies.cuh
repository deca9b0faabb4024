// Policies for umma_core.cuh: where each k-block's operand tiles come from and what happens to
// the accumulator.  Three families:
//   GemmPolicy   2-D operands (FC fwd / dgrad / wgrad, layer-0 im2col GEMM), optional split-K.
//   ConvPolicy   3x3/s1/p1 convolution as implicit GEMM: the A tile of tap (kh,kw) is a 4-D TMA
//                box of the NHWC activation shifted by (kh-1, kw-1); TMA's out-of-bounds zero fill
//                *is* the padding.  fprop: B = W[Cout][9*Cin] K-major.  dgrad: the same weight
//                tensor read MN-major with the taps mirrored (no transposed weight copy).
//   WgradPolicy  dW[cout][tap][cin] = sum_pixels dZ[p][cout] * X[p+tap][cin]: both operands are
//                MN-major 4-D boxes (K = 64 pixels per k-block), split-K over pixel tiles,
//                fp32 red.add epilogue straight into the gradient arena.
// The split-K epilogues (GemmPolicy's ATOMIC kinds, WgradPolicy) each have a PARTIAL form for
// bit-reproducible training: plain stores into slice `split` of a workspace, which splitk_reduce
// (elementwise.cu) then adds up in split order.
#pragma once
#include "umma_core.cuh"

namespace b200 {

// Division by a runtime constant as multiply-high + shift (host computes the magic number).  The
// epilogue warps of a small-tile layer spend a third of their instructions on `tile / tiles_m`
// style divisions otherwise (ncu: 392 warp instructions per 128x64 tile before, 8 epilogue warps).
struct FastDiv {
  uint32_t mul, shift, div;
};
inline FastDiv make_fastdiv(uint32_t d) {
  FastDiv f;
  f.div = d;
  if (d <= 1) { f.mul = 0; f.shift = 0; return f; }
  uint32_t l = 0;
  while ((1u << l) < d) ++l;                        // ceil(log2(d))
  const uint64_t m = ((1ull << (32 + l)) + d - 1) / d;   // ceil(2^(32+l) / d), fits 33 bits
  f.mul = static_cast<uint32_t>(m - (1ull << 32));  // low 32 bits of (m - 2^32); exact for n < 2^31
  f.shift = l;
  return f;
}
__device__ __forceinline__ void fast_divmod(const FastDiv& f, uint32_t n, uint32_t& q, uint32_t& r) {
  if (f.div <= 1) { q = n; r = 0; return; }
  const uint32_t t = __umulhi(n, f.mul);
  q = (t + ((n - t) >> 1)) >> (f.shift - 1);        // classic round-up method (Granlund-Montgomery)
  r = n - q * f.div;
}

// ---------------------------------------------------------------------------------------------
// Epilogue kinds for GemmPolicy
enum GemmEpi : int {
  EPI_F32_STORE = 0,      // out[row*ldo + col] = acc                      (fp32)
  EPI_F32_ATOMIC = 1,     // out[row*ldo + col] += acc                     (fp32, split-K)
  EPI_F32_ATOMIC_T = 2,   // out[col*ldo + row] += acc                     (swap-AB FC, split-K)
  EPI_BF16_BIAS_RELU = 3, // out[row*ldo + col] = bf16(relu(acc + bias[col]))
  EPI_F32_STORE_T = 4,    // out[col*ldo + row] = acc
  EPI_BF16_STORE = 5,     // out[row*ldo + col] = bf16(alpha * acc)   (FC wgrad straight into the bf16 wire)
  EPI_F32_PARTIAL = 6,    // out[split*slice + row*ldo + col] = acc        (fp32, split-K without atomics)
  EPI_F32_PARTIAL_T = 7,  // out[split*slice + col*ldo + row] = acc
};

struct GemmParams {
  CUtensorMap mapA;
  CUtensorMap mapB;
  int num_tiles;          // tiles_m * tiles_n * ksplit
  int tiles_m, tiles_n;
  int M, N;               // valid output extent (rows of A-side, rows of B-side)
  int k_iters_total;      // ceil(K / 64)
  int k_iters_per_split;
  void* out;
  long long ldo;
  const float* bias;
  float alpha;
  long long slice;        // PARTIAL epilogues: elements between the workspace slices of two splits
};

template <int BN_, int STAGES_, bool A_MN_, bool B_MN_, int EPI>
struct GemmPolicy {
  static constexpr int BN = BN_;
  static constexpr int STAGES = STAGES_;
  static constexpr bool A_MN = A_MN_;
  static constexpr bool B_MN = B_MN_;
  using Params = GemmParams;
  static constexpr bool PREMASK = false;
  static constexpr int EPI_SMEM = 0;
  __device__ static void epi_begin(const Params&, float*, int) {}
  __device__ static void epi_end(const Params&, float*, int) {}
  static constexpr bool PARTIAL = EPI == EPI_F32_PARTIAL || EPI == EPI_F32_PARTIAL_T;
  struct Ctx {
    int m0, n0, k_begin, nk;
    int split;            // set for the PARTIAL epilogues only
  };
  struct RowCtx {};
  __device__ static RowCtx row_ctx(const Params&, const Ctx&, int) { return RowCtx{}; }

  __device__ static void prefetch(const Params& p) {
    tma_prefetch_desc(&p.mapA);
    tma_prefetch_desc(&p.mapB);
  }
  __device__ static Ctx make_ctx(const Params& p, int tile) {
    Ctx c;
    const int tm = tile % p.tiles_m;
    const int rest = tile / p.tiles_m;
    const int tn = rest % p.tiles_n;
    const int tz = rest / p.tiles_n;
    if constexpr (PARTIAL) c.split = tz;
    c.m0 = tm * UMMA_BM;
    c.n0 = tn * BN;
    c.k_begin = tz * p.k_iters_per_split;
    int rem = p.k_iters_total - c.k_begin;
    c.nk = rem < 0 ? 0 : (rem < p.k_iters_per_split ? rem : p.k_iters_per_split);
    return c;
  }
  __device__ static int num_k_iters(const Params&, const Ctx& c) { return c.nk; }

  __device__ static void load(const Params& p, const Ctx& c, int i, uint8_t* sA, uint8_t* sB,
                              uint64_t* bar) {
    const int k0 = (c.k_begin + i) * UMMA_BK;
    if constexpr (A_MN) {
#pragma unroll
      for (int j = 0; j < UMMA_BM / 64; ++j)
        tma_load_2d(sA + j * UMMA_SLAB_BYTES, &p.mapA, bar, c.m0 + 64 * j, k0);
    } else {
      tma_load_2d(sA, &p.mapA, bar, k0, c.m0);
    }
    if constexpr (B_MN) {
#pragma unroll
      for (int j = 0; j < BN / 64; ++j)
        tma_load_2d(sB + j * UMMA_SLAB_BYTES, &p.mapB, bar, c.n0 + 64 * j, k0);
    } else {
      tma_load_2d(sB, &p.mapB, bar, k0, c.n0);
    }
  }

  __device__ static void epilogue(const Params& p, const Ctx& c, const RowCtx&, int row, int col0,
                                  const uint32_t (&acc)[32], float*) {
    const int r = c.m0 + row;
    const int cb = c.n0 + col0;
    if (r >= p.M || cb >= p.N) return;
    const float alpha = p.alpha;
    float* out32 = reinterpret_cast<float*>(p.out);
    if constexpr (PARTIAL) out32 += c.split * p.slice;
    constexpr bool STORE = EPI == EPI_F32_STORE || EPI == EPI_F32_PARTIAL;
    if constexpr (STORE || EPI == EPI_F32_ATOMIC) {
      float* o = out32 + static_cast<long long>(r) * p.ldo + cb;
      const bool vec = (cb + 32 <= p.N) && ((reinterpret_cast<uintptr_t>(o) & 15) == 0);
      if (STORE && vec && (reinterpret_cast<uintptr_t>(o) & 31) == 0) {
        // a thread owns one 128-byte line of the output: four full-sector 32-byte stores
#pragma unroll
        for (int j = 0; j < 32; j += 8) {
          uint32_t v[8];
#pragma unroll
          for (int u = 0; u < 8; ++u) v[u] = __float_as_uint(__uint_as_float(acc[j + u]) * alpha);
          st_global_v8(o + j, v);
        }
      } else if (vec) {
#pragma unroll
        for (int j = 0; j < 32; j += 4) {
          float4 v = make_float4(__uint_as_float(acc[j]) * alpha, __uint_as_float(acc[j + 1]) * alpha,
                                 __uint_as_float(acc[j + 2]) * alpha, __uint_as_float(acc[j + 3]) * alpha);
          if constexpr (STORE) {
            *reinterpret_cast<float4*>(o + j) = v;
          } else {
            asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(o + j), "f"(v.x),
                         "f"(v.y), "f"(v.z), "f"(v.w)
                         : "memory");
          }
        }
      } else {
        for (int j = 0; j < 32 && cb + j < p.N; ++j) {
          if constexpr (STORE) o[j] = __uint_as_float(acc[j]) * alpha;
          else atomicAdd(o + j, __uint_as_float(acc[j]) * alpha);
        }
      }
    } else if constexpr (EPI == EPI_F32_ATOMIC_T || EPI == EPI_F32_STORE_T || EPI == EPI_F32_PARTIAL_T) {
      float* o = out32 + static_cast<long long>(cb) * p.ldo + r;
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        if (cb + j < p.N) {
          if constexpr (EPI == EPI_F32_ATOMIC_T) atomicAdd(o + static_cast<long long>(j) * p.ldo, __uint_as_float(acc[j]) * alpha);
          else o[static_cast<long long>(j) * p.ldo] = __uint_as_float(acc[j]) * alpha;
        }
      }
    } else if constexpr (EPI == EPI_BF16_STORE) {
      __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(p.out) + static_cast<long long>(r) * p.ldo + cb;
      if ((cb + 32 <= p.N) && ((reinterpret_cast<uintptr_t>(o) & 31) == 0)) {
#pragma unroll
        for (int j = 0; j < 32; j += 16) {
          uint32_t pk[8];
#pragma unroll
          for (int u = 0; u < 8; ++u)
            pk[u] = pack_bf16x2(__uint_as_float(acc[j + 2 * u]) * alpha, __uint_as_float(acc[j + 2 * u + 1]) * alpha);
          st_global_v8(o + j, pk);
        }
      } else if ((cb + 32 <= p.N) && ((reinterpret_cast<uintptr_t>(o) & 15) == 0)) {
#pragma unroll
        for (int j = 0; j < 32; j += 8) {
          const uint4 pk = make_uint4(
              pack_bf16x2(__uint_as_float(acc[j]) * alpha, __uint_as_float(acc[j + 1]) * alpha),
              pack_bf16x2(__uint_as_float(acc[j + 2]) * alpha, __uint_as_float(acc[j + 3]) * alpha),
              pack_bf16x2(__uint_as_float(acc[j + 4]) * alpha, __uint_as_float(acc[j + 5]) * alpha),
              pack_bf16x2(__uint_as_float(acc[j + 6]) * alpha, __uint_as_float(acc[j + 7]) * alpha));
          *reinterpret_cast<uint4*>(o + j) = pk;
        }
      } else {
        for (int j = 0; j < 32 && cb + j < p.N; ++j) o[j] = __float2bfloat16(__uint_as_float(acc[j]) * alpha);
      }
    } else if constexpr (EPI == EPI_BF16_BIAS_RELU) {
      __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(p.out) + static_cast<long long>(r) * p.ldo + cb;
      if ((cb + 32 <= p.N) && ((reinterpret_cast<uintptr_t>(o) & 15) == 0)) {
#pragma unroll
        for (int j = 0; j < 32; j += 8) {
          float v[8];
#pragma unroll
          for (int t = 0; t < 8; ++t) {
            float b = p.bias ? __ldg(p.bias + cb + j + t) : 0.f;
            v[t] = fmaxf(__uint_as_float(acc[j + t]) + b, 0.f);
          }
          uint4 pk = make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]),
                                pack_bf16x2(v[4], v[5]), pack_bf16x2(v[6], v[7]));
          *reinterpret_cast<uint4*>(o + j) = pk;
        }
      } else {   // ragged last chunk or unaligned row: neither the bias nor the output past N is touched
        for (int j = 0; j < 32 && cb + j < p.N; ++j) {
          const float b = p.bias ? __ldg(p.bias + cb + j) : 0.f;
          o[j] = __float2bfloat16(fmaxf(__uint_as_float(acc[j]) + b, 0.f));
        }
      }
    }
  }
};

// ---------------------------------------------------------------------------------------------
struct ConvTile {
  int N, H, W;            // activation extent
  int Wb, Hb, Nb;         // pixel box of one tile (Wb*Hb*Nb = 128 for fprop/dgrad, 64 for wgrad)
  int tiles_w, tiles_h;   // ceil(W/Wb), ceil(H/Hb)
  int wb_shift, hb_shift; // log2(Wb), log2(Hb): the box sides are powers of two
  FastDiv div_tw, div_th; // fast division by tiles_w / tiles_h
};

enum ConvFlags : int {
  CONV_BIAS = 1,          // add bias[channel]
  CONV_RELU = 2,          // clamp at 0
  CONV_MASK = 4,          // zero where mask_src <= 0 (ReLU backward fused into dgrad)
  CONV_COLSUM = 8,        // colsum[channel] += sum over pixels of the stored (bf16-rounded) output:
                          // the bias gradient of the previous layer, for free in the dgrad epilogue
  CONV_POOL = 16,         // fprop only, on by default (B200_FUSE_POOL=0 turns it off): 2x2/2 max-pool inside
                          // the epilogue -- writes pool_out + pool_mask, never the un-pooled tensor
};

struct ConvParams {
  CUtensorMap mapA;       // activation, dims {Ca, W, H, N}, box {64, Wb, Hb, Nb}
  CUtensorMap mapB;       // weights as 2-D [Cout][9*Cin]
  int num_tiles;          // pixel tiles * channel tiles
  int tiles_m;            // pixel tiles (fastest: neighbouring CTAs share halos and the weight tile in L2)
  FastDiv div_tm;         // fast division by tiles_m
  ConvTile t;
  int Ca;                 // channels of the A activation (GEMM K per tap)
  int Cn;                 // channels of the output (GEMM N)
  int wcols_per_tap;      // Cin of the weight tensor (column block per tap)
  __nv_bfloat16* out;     // NHWC [N][H][W][Cn]
  const float* bias;
  const __nv_bfloat16* mask_src;
  float* colsum;          // [Cn] fp32, accumulated with atomics (CONV_COLSUM)
  __nv_bfloat16* pool_out;  // CONV_POOL: NHWC [N][H/2][W/2][Cn]
  uint32_t* pool_mask;      // CONV_POOL: [N][H/2][W/2][Cn/32][4] = {argmax bit 0, argmax bit 1, max > 0, 0}
  int flags;
  int resident;           // halo kernel: all weight tiles stay in shared memory for the CTA lifetime
  // FILL instantiations only (a box of any Wb x Hb x Nb <= 128 pixels): row -> (w, h, n) by division
  FastDiv div_wb, div_hb;
  uint32_t a_tx;          // bytes one A box delivers: Wb * Hb * Nb * 64 channels * 2
};

__device__ __forceinline__ void conv_tile_origin(const ConvTile& t, int tile, int& n0, int& h0,
                                                 int& w0) {
  uint32_t rest, tw, tn, th;
  fast_divmod(t.div_tw, static_cast<uint32_t>(tile), rest, tw);
  fast_divmod(t.div_th, rest, tn, th);
  w0 = static_cast<int>(tw) * t.Wb;
  h0 = static_cast<int>(th) * t.Hb;
  n0 = static_cast<int>(tn) * t.Nb;
}

// POOL (fprop only): a separate instantiation, so the un-pooled fprop kernels carry none of its code.
// FILL: the pixel box is any Wb x Hb x Nb <= 128 pixels (conv_fill_tile; 11 x 11 x 1 on an 11^2 map), not
// power-of-two sides: a row is decoded with fastdiv, rows past the box are neither stored nor summed, and
// the A box delivers a_tx bytes.  The power-of-two instantiations keep their shift decode.
template <int BN_, int STAGES_, bool DGRAD, bool POOL = false, bool FILL = false>
struct ConvPolicy {
  static_assert(!(DGRAD && POOL), "the fused pool is an fprop epilogue");
  static_assert(!(POOL && FILL), "the fused pool needs the power-of-two boxes of make_tile");
  static constexpr bool FILL_BOX = FILL;
  static constexpr int BN = BN_;
  static constexpr int STAGES = STAGES_;
  static constexpr bool A_MN = false;
  static constexpr bool B_MN = DGRAD;
  using Params = ConvParams;
  // epilogue scratch [512] floats: dgrad = per-CTA channel sums (fused bias gradient);
  // fprop = the bias vector, staged once per CTA and read back as broadcast float4 loads
  static constexpr int EPI_MAXC = 512;
  static constexpr int EPI_SMEM = EPI_MAXC * 4;
  static constexpr bool PREMASK = DGRAD;
  __device__ static void epi_begin(const Params& p, float* sm, int tid) {
    if constexpr (DGRAD) {
      if (p.flags & CONV_COLSUM)
        for (int i = tid; i < EPI_MAXC; i += UMMA_EPI_THREADS) sm[i] = 0.f;
    } else {
      if (p.flags & CONV_BIAS)
        for (int i = tid; i < p.Cn && i < EPI_MAXC; i += UMMA_EPI_THREADS) sm[i] = p.bias[i];
    }
  }
  __device__ static void epi_end(const Params& p, float* sm, int tid) {
    if constexpr (DGRAD) {
      if (p.flags & CONV_COLSUM)
        for (int i = tid; i < p.Cn; i += UMMA_EPI_THREADS) {
          const float v = sm[i];
          if (v != 0.f) atomicAdd(p.colsum + i, v);
        }
    }
  }
  struct Ctx {
    int n0, h0, w0, c0, cchunks;
  };
  struct RowCtx {
    long long pix_off;      // element offset of this thread's pixel (channel 0) in the NHWC output
    bool valid;
  };
  __device__ static RowCtx row_ctx(const Params& p, const Ctx& c, int row) {
    const ConvTile& t = p.t;
    int ww, hh, nn;
    if constexpr (FILL) {
      uint32_t r2, r3, rw, rh;
      fast_divmod(p.div_wb, static_cast<uint32_t>(row), r2, rw);
      fast_divmod(p.div_hb, r2, r3, rh);
      ww = static_cast<int>(rw); hh = static_cast<int>(rh); nn = static_cast<int>(r3);
    } else {
      ww = row & (t.Wb - 1);
      const int r2 = row >> t.wb_shift;
      hh = r2 & (t.Hb - 1);
      nn = r2 >> t.hb_shift;
    }
    const int n = c.n0 + nn, h = c.h0 + hh, w = c.w0 + ww;
    RowCtx rc;
    rc.valid = n < t.N && h < t.H && w < t.W;
    if constexpr (FILL) rc.valid = rc.valid && nn < t.Nb;      // rows past the box: stale shared memory
    rc.pix_off = ((static_cast<long long>(n) * t.H + h) * t.W + w) * p.Cn;
    return rc;
  }
  __device__ static void prefetch(const Params& p) {
    tma_prefetch_desc(&p.mapA);
    tma_prefetch_desc(&p.mapB);
  }
  __device__ static Ctx make_ctx(const Params& p, int tile) {
    Ctx c;
    uint32_t tn, tm;
    fast_divmod(p.div_tm, static_cast<uint32_t>(tile), tn, tm);
    conv_tile_origin(p.t, static_cast<int>(tm), c.n0, c.h0, c.w0);
    c.c0 = static_cast<int>(tn) * BN;
    c.cchunks = p.Ca / UMMA_BK;
    return c;
  }
  __device__ static int num_k_iters(const Params&, const Ctx& c) { return 9 * c.cchunks; }

  __device__ static void load(const Params& p, const Ctx& c, int i, uint8_t* sA, uint8_t* sB,
                              uint64_t* bar) {
    const int tap = i / c.cchunks;
    const int ck = (i - tap * c.cchunks) * UMMA_BK;
    const int dh = tap / 3 - 1, dw = tap % 3 - 1;
    tma_load_4d(sA, &p.mapA, bar, ck, c.w0 + dw, c.h0 + dh, c.n0);
    if constexpr (!DGRAD) {
      tma_load_2d(sB, &p.mapB, bar, tap * p.wcols_per_tap + ck, c.c0);
    } else {
      const int wt = 8 - tap;          // mirrored tap: dX[q] = sum dZ[q + (kh'-1, kw'-1)] W[2-kh'][2-kw']
#pragma unroll
      for (int j = 0; j < BN / 64; ++j)
        tma_load_2d(sB + j * UMMA_SLAB_BYTES, &p.mapB, bar, wt * p.wcols_per_tap + c.c0 + 64 * j, ck);
    }
  }

  // The ReLU mask of a dgrad chunk (the previous layer's activations at this thread's pixel)
  // depends only on the tile, not on the accumulator: the epilogue warpgroup fetches it BEFORE it
  // waits for the staged accumulator, so the global-load latency overlaps the MMAs.
  __device__ static bool masked(const Params& p) { return DGRAD && (p.flags & CONV_MASK) != 0; }
  __device__ static void load_mask(const Params& p, const Ctx& c, const RowCtx& rc, int col0, uint32_t (&m)[16]) {
    const int ch = c.c0 + col0;
    if (rc.valid && ch < p.Cn) {
      const __nv_bfloat16* src = p.mask_src + rc.pix_off + ch;
      ld_global_nc_v8(src, m);
      ld_global_nc_v8(src + 16, m + 8);
    } else {
#pragma unroll
      for (int j = 0; j < 16; ++j) m[j] = 0u;
    }
  }

  // One 32-column chunk of one pixel: 64 contiguous bytes, written as two 32-byte stores.
  __device__ static void epilogue(const Params& p, const Ctx& c, const RowCtx& rc, int row, int col0,
                                  const uint32_t (&acc)[32], float* sm, const uint32_t* premask = nullptr,
                                  float* keep = nullptr, bool keep_on = false) {
    if constexpr (POOL) {
      epilogue_pool(p, c, rc, row, col0, acc, sm);
      return;
    }
    const int ch = c.c0 + col0;
    const bool valid = rc.valid && ch < p.Cn;
    const long long off = rc.pix_off + ch;
    __nv_bfloat16* o = p.out + off;
    const bool colsum = DGRAD && (p.flags & CONV_COLSUM);
    const int lane = row & 31;
    float cs[32];                                           // what this thread stored (bf16-rounded)
#pragma unroll
    for (int j = 0; j < 32; j += 16) {
      float v[16];
#pragma unroll
      for (int u = 0; u < 16; ++u) v[u] = __uint_as_float(acc[j + u]);
      if (valid) {
        if (!DGRAD && (p.flags & CONV_BIAS)) {
#pragma unroll
          for (int u = 0; u < 16; u += 4) {
            const float4 b = *reinterpret_cast<const float4*>(sm + ch + j + u);     // smem broadcast
            v[u] += b.x; v[u + 1] += b.y; v[u + 2] += b.z; v[u + 3] += b.w;
          }
        }
        if (p.flags & CONV_RELU) {
#pragma unroll
          for (int u = 0; u < 16; ++u) v[u] = fmaxf(v[u], 0.f);
        }
        if (DGRAD && (p.flags & CONV_MASK)) {    // premask: load_mask of this chunk
#pragma unroll
          for (int u = 0; u < 8; ++u) {
            const float2 f = unpack_bf16x2(premask[(j >> 1) + u]);
            if (!(f.x > 0.f)) v[2 * u] = 0.f;
            if (!(f.y > 0.f)) v[2 * u + 1] = 0.f;
          }
        }
        uint32_t pk[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) pk[u] = pack_bf16x2(v[2 * u], v[2 * u + 1]);
        st_global_v8(o + j, pk);
        if (colsum) {        // sum exactly what was stored, like a separate pass over dz would
#pragma unroll
          for (int u = 0; u < 8; ++u) {
            const float2 f = unpack_bf16x2(pk[u]);
            cs[j + 2 * u] = f.x;
            cs[j + 2 * u + 1] = f.y;
          }
        }
      } else if (colsum) {
#pragma unroll
        for (int u = 0; u < 16; ++u) cs[j + u] = 0.f;
      }
    }
    if (colsum) {
      if (keep_on) {         // caller keeps per-thread running sums and flushes once (colsum_flush)
#pragma unroll
        for (int i = 0; i < 32; ++i) keep[i] += cs[i];
      } else {
        colsum_flush(p, c.c0 + col0, lane, cs, sm);
      }
    }
  }

  // CONV_POOL: bias + ReLU + 2x2/2 max-pool of one 32-channel chunk.  The epilogue row
  // is the pixel, a warp holds 32 consecutive tile rows = (32 / Wb) image rows of Wb pixels, so the
  // four pixels of a pool window are lanes {l, l^1, l^Wb, l^Wb^1} (Wb <= 16, tile origin and image
  // extent even: the launcher checks).  The top-left lane of each window stores the pooled bf16
  // values and three bit masks per 32 channels: argmax position (2 bits, first maximum in the order
  // (0,0) (0,1) (1,0) (1,1), like maxpool2x2_relu_bwd) and "max > 0" (the ReLU mask) -- everything
  // the backward pass needs, so the un-pooled activation is never written.
  __device__ static void epilogue_pool(const Params& p, const Ctx& c, const RowCtx& rc, int row, int col0,
                                       const uint32_t (&acc)[32], float* sm) {
    const ConvTile& t = p.t;
    const int ch = c.c0 + col0;
    const bool chan_ok = ch < p.Cn;                        // warp-uniform
    uint32_t pk[16], m[16];
#pragma unroll
    for (int u = 0; u < 16; ++u) {
      float lo = __uint_as_float(acc[2 * u]), hi = __uint_as_float(acc[2 * u + 1]);
      if (chan_ok && (p.flags & CONV_BIAS)) { lo += sm[ch + 2 * u]; hi += sm[ch + 2 * u + 1]; }
      pk[u] = pack_bf16x2(fmaxf(lo, 0.f), fmaxf(hi, 0.f));
    }
#pragma unroll
    for (int u = 0; u < 16; ++u) m[u] = max_bf16x2(pk[u], __shfl_xor_sync(0xffffffffu, pk[u], 1));
#pragma unroll
    for (int u = 0; u < 16; ++u) m[u] = max_bf16x2(m[u], __shfl_xor_sync(0xffffffffu, m[u], t.Wb));
    uint32_t e = 0, pos = 0;                               // bit ch: my value is the window maximum / max > 0
#pragma unroll
    for (int u = 0; u < 16; ++u) {
      const uint32_t d = pk[u] ^ m[u];
      e |= ((d & 0xffffu) == 0u ? 1u : 0u) << (2 * u);
      e |= ((d >> 16) == 0u ? 1u : 0u) << (2 * u + 1);
      pos |= ((m[u] & 0x7fffu) != 0u ? 1u : 0u) << (2 * u);
      pos |= ((m[u] & 0x7fff0000u) != 0u ? 1u : 0u) << (2 * u + 1);
    }
    const uint32_t e1 = __shfl_xor_sync(0xffffffffu, e, 1);          // (0,1) as seen from the top-left lane
    const uint32_t e2 = __shfl_xor_sync(0xffffffffu, e, t.Wb);       // (1,0)
    const int ww = row & (t.Wb - 1);
    const int r2 = row >> t.wb_shift;
    const int hh = r2 & (t.Hb - 1);
    const int nn = r2 >> t.hb_shift;
    if (((ww | hh) & 1) == 0 && rc.valid && chan_ok) {
      const int n = c.n0 + nn, h = c.h0 + hh, w = c.w0 + ww;
      const long long ppix = (static_cast<long long>(n) * (t.H >> 1) + (h >> 1)) * (t.W >> 1) + (w >> 1);
      __nv_bfloat16* o = p.pool_out + ppix * p.Cn + ch;
      const uint32_t lo8[8] = {m[0], m[1], m[2], m[3], m[4], m[5], m[6], m[7]};
      const uint32_t hi8[8] = {m[8], m[9], m[10], m[11], m[12], m[13], m[14], m[15]};
      st_global_v8(o, lo8);
      st_global_v8(o + 16, hi8);
      // first maximum: 0 if e, else 1 if e1, else 2 if e2, else 3
      const uint32_t b0 = ~e & (e1 | ~e2);
      const uint32_t b1 = ~e & ~e1;
      *reinterpret_cast<uint4*>(p.pool_mask + (ppix * (p.Cn >> 5) + (ch >> 5)) * 4) = make_uint4(b0, b1, pos, 0u);
    }
  }

  // Transpose-reduce across the warp with shuffles (recursive halving, 31 SHFL): afterwards lane l
  // holds the sum over the warp's 32 pixels of column l, added to the per-CTA sums in shared
  // memory.  No shared-memory traffic for the reduction itself -- operand staging saturates it.
  // Both loops have constant trip counts so that they unroll completely: with `i < s` as the bound
  // ptxas kept a partly unrolled loop that indexed cs[] at run time, which put cs[] -- and the
  // epilogue's column sums -- in local memory (a 128-byte stack frame, ~100 local loads and stores).
  __device__ static void colsum_flush(const Params& p, int ch0, int lane, float (&cs)[32], float* sm) {
    __syncwarp();
#pragma unroll
    for (int level = 0; level < 5; ++level) {
      const int s = 16 >> level;
      const bool upper = (lane & s) != 0;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        if (i >= s) continue;
        const float keep = upper ? cs[i + s] : cs[i];
        const float send = upper ? cs[i] : cs[i + s];
        cs[i] = keep + __shfl_xor_sync(0xffffffffu, send, s);
      }
    }
    const int cc = ch0 + lane;
    if (cc < p.Cn && cc < EPI_MAXC) atomicAdd(sm + cc, cs[0]);
  }
};

// ---------------------------------------------------------------------------------------------
struct WgradParams {
  CUtensorMap mapA;       // dZ, dims {Cout, W, H, N}, box {64, Wb, Hb, Nb} (64 pixels)
  CUtensorMap mapB;       // X,  dims {Cin,  W, H, N}, same box
  int num_tiles;          // tiles_m * tiles_n * 9 * ksplit
  int tiles_m, tiles_n;
  ConvTile t;
  int Cout, Cin;
  int total_tiles;        // pixel tiles = tiles_w * tiles_h * tiles_n
  int tiles_per_split;
  int ksplit;
  float* dW;              // [Cout][9][Cin] fp32, accumulated with red.add; PARTIAL: [ksplit][Cout][9][Cin], stored
  float scale;
};

template <int BN_, int STAGES_, bool PARTIAL = false>
struct WgradPolicy {
  static constexpr int BN = BN_;
  static constexpr int STAGES = STAGES_;
  static constexpr bool A_MN = true;
  static constexpr bool B_MN = true;
  using Params = WgradParams;
  static constexpr bool PREMASK = false;
  static constexpr int EPI_SMEM = 0;
  __device__ static void epi_begin(const Params&, float*, int) {}
  __device__ static void epi_end(const Params&, float*, int) {}
  struct Ctx {
    int m0, c0, tap, tile_begin, nk;
    int split;            // set for PARTIAL only
  };
  struct RowCtx {};
  __device__ static RowCtx row_ctx(const Params&, const Ctx&, int) { return RowCtx{}; }
  __device__ static void prefetch(const Params& p) {
    tma_prefetch_desc(&p.mapA);
    tma_prefetch_desc(&p.mapB);
  }
  __device__ static Ctx make_ctx(const Params& p, int tile) {
    Ctx c;
    // tap fastest, then the channel tiles, pixel split slowest: the CTAs that run together read
    // the SAME pixel range of dZ / X for different taps and channel tiles, so it comes from DRAM
    // once and from L2 for everybody else (ncu: split-fastest order re-streamed both tensors from
    // DRAM once per tap -- 89 % DRAM utilisation on features.2).
    c.tap = tile % 9;
    int rest = tile / 9;
    c.m0 = (rest % p.tiles_m) * UMMA_BM;
    rest /= p.tiles_m;
    c.c0 = (rest % p.tiles_n) * BN;
    const int split = rest / p.tiles_n;
    if constexpr (PARTIAL) c.split = split;
    c.tile_begin = split * p.tiles_per_split;
    int rem = p.total_tiles - c.tile_begin;
    c.nk = rem < 0 ? 0 : (rem < p.tiles_per_split ? rem : p.tiles_per_split);
    return c;
  }
  __device__ static int num_k_iters(const Params&, const Ctx& c) { return c.nk; }

  __device__ static void load(const Params& p, const Ctx& c, int i, uint8_t* sA, uint8_t* sB,
                              uint64_t* bar) {
    int n0, h0, w0;
    conv_tile_origin(p.t, c.tile_begin + i, n0, h0, w0);
    const int dh = c.tap / 3 - 1, dw = c.tap % 3 - 1;
#pragma unroll
    for (int j = 0; j < UMMA_BM / 64; ++j)
      tma_load_4d(sA + j * UMMA_SLAB_BYTES, &p.mapA, bar, c.m0 + 64 * j, w0, h0, n0);
#pragma unroll
    for (int j = 0; j < BN / 64; ++j)
      tma_load_4d(sB + j * UMMA_SLAB_BYTES, &p.mapB, bar, c.c0 + 64 * j, w0 + dw, h0 + dh, n0);
  }

  __device__ static void epilogue(const Params& p, const Ctx& c, const RowCtx&, int row, int col0,
                                  const uint32_t (&acc)[32], float*) {
    const int co = c.m0 + row;
    const int ci = c.c0 + col0;
    if (co >= p.Cout || ci >= p.Cin) return;
    float* o = p.dW + (static_cast<long long>(co) * 9 + c.tap) * p.Cin + ci;
    const float s = p.scale;
    if constexpr (PARTIAL) {     // this split's own slice: every element has one writer
      o += static_cast<long long>(c.split) * p.Cout * 9 * p.Cin;
#pragma unroll
      for (int j = 0; j < 32; j += 4)
        *reinterpret_cast<float4*>(o + j) = make_float4(__uint_as_float(acc[j]) * s, __uint_as_float(acc[j + 1]) * s,
                                                        __uint_as_float(acc[j + 2]) * s, __uint_as_float(acc[j + 3]) * s);
      return;
    }
#pragma unroll
    for (int j = 0; j < 32; j += 4) {
      asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(o + j),
                   "f"(__uint_as_float(acc[j]) * s), "f"(__uint_as_float(acc[j + 1]) * s),
                   "f"(__uint_as_float(acc[j + 2]) * s), "f"(__uint_as_float(acc[j + 3]) * s)
                   : "memory");
    }
  }
};

}  // namespace b200
