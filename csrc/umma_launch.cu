// Host side of the wgmma GEMM / convolution family: builds the TMA tensor maps
// (cuTensorMapEncodeTiled through the runtime's driver entry point, so nothing links libcuda),
// picks the tile width and launches umma_kernel<Policy>.
#include <cudaTypedefs.h>

#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <stdexcept>
#include <string>

#include "api.h"
#include "conv0.cuh"
#include "conv_halo.cuh"
#include "wgrad_halo.cuh"
#include "umma_policies.cuh"

namespace b200 {

static std::atomic<long long> g_launches{0};
long long launch_count() { return g_launches.load(); }
void count_launch(int n) { g_launches.fetch_add(n); }
void check_last(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess)
    throw std::runtime_error(std::string("[b200] ") + what + ": " + cudaGetErrorString(e));
}

static PFN_cuTensorMapEncodeTiled_v12000 encode_fn() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
    if (e != cudaSuccess || q != cudaDriverEntryPointSuccess || !p)
      throw std::runtime_error("[b200] cuTensorMapEncodeTiled entry point not available");
    fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
  }
  return fn;
}

static void encode(CUtensorMap* map, const void* ptr, int rank, const cuuint64_t* dims,
                   const cuuint64_t* strides_bytes, const cuuint32_t* box) {
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) != 0)
    throw std::runtime_error("[b200] TMA base pointer must be 16-byte aligned");
  for (int i = 0; i < rank - 1; ++i)
    if (strides_bytes[i] % 16 != 0)
      throw std::runtime_error("[b200] TMA strides must be multiples of 16 bytes");
  CUresult r = encode_fn()(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank, const_cast<void*>(ptr),
                           dims, strides_bytes, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                           CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                           CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char buf[256];
    snprintf(buf, sizeof buf,
             "[b200] cuTensorMapEncodeTiled failed (%d): rank %d dims %llu %llu box %u %u", (int)r,
             rank, (unsigned long long)dims[0], (unsigned long long)dims[1], box[0], box[1]);
    throw std::runtime_error(buf);
  }
}

// 2-D row-major matrix [rows][cols] (row stride ld elements); box = {box_cols, box_rows}.
static void map_2d(CUtensorMap* m, const bf16* p, long long rows, long long cols, long long ld,
                   int box_cols, int box_rows) {
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t str[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
  encode(m, p, 2, dims, str, box);
}
// NHWC activation as {C, W, H, N}; box = {64, Wb, Hb, Nb}.
static void map_nhwc(CUtensorMap* m, const bf16* p, int N, int H, int W, int C, int Wb, int Hb,
                     int Nb) {
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
  cuuint64_t str[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
  cuuint32_t box[4] = {64, (cuuint32_t)Wb, (cuuint32_t)Hb, (cuuint32_t)Nb};
  encode(m, p, 4, dims, str, box);
}

int sm_count() {
  static int n = 0;
  if (!n) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) throw std::runtime_error("[b200] cannot query the SM count of the current device");
  }
  return n;
}
static int num_sms() { return sm_count(); }

bool comm_carveout_enabled() {
  static const bool on = [] {
    const char* e = getenv("B200_COMM_CARVEOUT");
    return !(e && e[0] == '0');
  }();
  return on;
}
void prefer_max_shared_carveout(const void* kernel) {
  if (!comm_carveout_enabled()) return;
  const cudaError_t err = cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout,
                                               cudaSharedmemCarveoutMaxShared);
  if (err != cudaSuccess)
    throw std::runtime_error(std::string("[b200] cudaFuncSetAttribute(carveout): ") + cudaGetErrorString(err));
}

// Switches of two variants that exist only in the tcgen05 version of this library: the dynamic tile
// scheduler (B200_DYNAMIC_TILES) and the TMA-store halo epilogue (B200_HALO_TMA_EPI).  Both were off
// by default and measured no faster than the default kernels; they are not provided for sm_90a, and
// asking for them is an error rather than a silent fall-back.
static void reject_removed_variants() {
  static const bool checked = [] {
    for (const char* name : {"B200_DYNAMIC_TILES", "B200_HALO_TMA_EPI"}) {
      const char* e = getenv(name);
      if (e && e[0] == '1')
        throw std::runtime_error(std::string("[b200] ") + name +
                                 "=1: this kernel variant is not available in the sm_90a build (docs/EXPERIMENTAL.md)");
    }
    return true;
  }();
  (void)checked;
}

// Persistent launch: one CTA per SM (or fewer when there are fewer tiles).
template <class P>
static void launch(const typename P::Params& prm, cudaStream_t stream) {
  reject_removed_variants();
  if (prm.num_tiles <= 0) return;
  dim3 grid(prm.num_tiles < num_sms() ? prm.num_tiles : num_sms());
  constexpr int smem = umma_smem_bytes<P::BN, P::STAGES>() + P::EPI_SMEM;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(umma_kernel<P>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess)
      throw std::runtime_error(std::string("[b200] cudaFuncSetAttribute: ") + cudaGetErrorString(e));
    configured = true;
  }
  umma_kernel<P><<<grid, UMMA_THREADS, smem, stream>>>(prm);
  count_launch();
  check_last("umma_kernel launch");
}

static int largest_pow2_divisor(int x, int cap) {
  int p = 1;
  while (p * 2 <= cap && x % (p * 2) == 0) p *= 2;
  return p;
}
// Pixel box {Wb, Hb, Nb} with Wb*Hb*Nb == pixels, following the power-of-two factors of W and H
// (224 = 7*32 -> 32x4x1, 112 -> 16x8x1, 56 -> 8x8x2, 28 -> 4x4x8, 14 -> 2x2x32).
static ConvTile make_tile(int N, int H, int W, int pixels) {
  ConvTile t;
  t.N = N; t.H = H; t.W = W;
  t.Wb = largest_pow2_divisor(W, pixels < 32 ? pixels : 32);
  t.Hb = largest_pow2_divisor(H, pixels / t.Wb);
  t.Nb = pixels / (t.Wb * t.Hb);
  t.tiles_w = (W + t.Wb - 1) / t.Wb;
  t.tiles_h = (H + t.Hb - 1) / t.Hb;
  t.wb_shift = 0; while ((1 << t.wb_shift) < t.Wb) ++t.wb_shift;
  t.hb_shift = 0; while ((1 << t.hb_shift) < t.Hb) ++t.hb_shift;
  t.div_tw = make_fastdiv(t.tiles_w);
  t.div_th = make_fastdiv(t.tiles_h);
  return t;
}

static long long conv_tile_count(const ConvTile& t) {
  return static_cast<long long>(t.tiles_w) * t.tiles_h * ((t.N + t.Nb - 1) / t.Nb);
}
// Maps without a large power-of-two factor (11^2, 25^2) leave make_tile's 1 x 1 x 128 box half empty at
// batch 64: 121 tiles do the work of 61.  conv_fill_tile searches every box Wb x Hb x Nb <= 128 pixels for
// the fewest tiles (ties: the most pixels per box, then the widest rows) and returns true only where that
// beats make_tile -- never where make_tile's tiles are already full, so those shapes keep their box and
// their kernels.  11^2 at batch 64 -> 11 x 11 x 1 (64 tiles), 25^2 -> 25 x 5 x 1 (320 tiles instead of 625).
static bool conv_fill_tile(int N, int H, int W, ConvTile* out) {
  const ConvTile base = make_tile(N, H, W, UMMA_BM);
  long long best = conv_tile_count(base);
  int bw = 0, bh = 0, bn = 0, bpix = 0;
  for (int wb = 1; wb <= W && wb <= UMMA_BM; ++wb)
    for (int hb = 1; hb <= H && wb * hb <= UMMA_BM; ++hb) {
      const int nb = std::min(N, UMMA_BM / (wb * hb));
      const long long tiles = static_cast<long long>((W + wb - 1) / wb) * ((H + hb - 1) / hb) * ((N + nb - 1) / nb);
      const int pix = wb * hb * nb;
      if (tiles < best || (bw && tiles == best && (pix > bpix || (pix == bpix && wb > bw)))) {
        best = tiles; bw = wb; bh = hb; bn = nb; bpix = pix;
      }
    }
  if (!bw) return false;
  ConvTile& t = *out;
  t = base;
  t.Wb = bw; t.Hb = bh; t.Nb = bn;
  t.tiles_w = (W + bw - 1) / bw;
  t.tiles_h = (H + bh - 1) / bh;
  t.wb_shift = t.hb_shift = -1;             // not powers of two: the FILL kernels divide
  t.div_tw = make_fastdiv(t.tiles_w);
  t.div_th = make_fastdiv(t.tiles_h);
  return true;
}
static void set_fill(ConvParams& prm) {
  prm.div_wb = make_fastdiv(prm.t.Wb);
  prm.div_hb = make_fastdiv(prm.t.Hb);
  prm.a_tx = static_cast<uint32_t>(prm.t.Wb * prm.t.Hb * prm.t.Nb * UMMA_BK * 2);
}

// NHWC activation with an explicit pixel box {64, bw, bh, bn} (the halo kernel's (8+2) x (16+2)).
static void map_nhwc_box(CUtensorMap* m, const bf16* p, int N, int H, int W, int C, int bw, int bh, int bn) {
  map_nhwc(m, p, N, H, W, C, bw, bh, bn);
}

static bool halo_enabled() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("B200_CONV_HALO");
    v = (e && e[0] == '0') ? 0 : 1;
  }
  return v != 0;
}
// The halo kernel tiles the image in 8 x 16 pixel blocks: use it where that wastes nothing.
static bool halo_applicable(int H, int W) { return halo_enabled() && W % HALO_WT == 0 && H % HALO_HT == 0 && W >= 32; }

template <int BN, bool DGRAD, bool POOL = false>
static void conv_halo_launch(ConvParams& prm, const bf16* act, cudaStream_t stream) {
  reject_removed_variants();
  using Cfg = HaloCfg<BN>;
  ConvTile& t = prm.t;
  t.Wb = HALO_WT; t.Hb = HALO_HT; t.Nb = 1; t.wb_shift = 3; t.hb_shift = 4;
  t.tiles_w = t.W / HALO_WT; t.tiles_h = t.H / HALO_HT;
  t.div_tw = make_fastdiv(t.tiles_w); t.div_th = make_fastdiv(t.tiles_h);
  prm.tiles_m = t.tiles_w * t.tiles_h * t.N;
  prm.div_tm = make_fastdiv(prm.tiles_m);
  const int tiles_n = (prm.Cn + BN - 1) / BN;
  prm.num_tiles = prm.tiles_m * tiles_n;
  map_nhwc_box(&prm.mapA, act, t.N, t.H, t.W, prm.Ca, HALO_PITCH, HALO_HT + 2, 1);
  constexpr int smem = Cfg::SMEM + ConvPolicy<BN, 1, DGRAD, POOL>::EPI_SMEM;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(conv_halo_kernel<BN, DGRAD, POOL>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess)
      throw std::runtime_error(std::string("[b200] cudaFuncSetAttribute(halo): ") + cudaGetErrorString(e));
    configured = true;
  }
  dim3 grid(prm.num_tiles < num_sms() ? prm.num_tiles : num_sms());
  conv_halo_kernel<BN, DGRAD, POOL><<<grid, UMMA_THREADS, smem, stream>>>(prm);
  count_launch();
  check_last("conv_halo_kernel launch");
}

// ------------------------------------------------------------------------- first conv (no im2col)
template <bool WGRAD, bool PARTIAL = false>
static void conv0_launch(Conv0Params& prm, int grid, cudaStream_t stream) {
  constexpr int stage = C0_TILE_BYTES + (WGRAD ? UMMA_SLAB_BYTES : 0);
  constexpr int smem = C0_STAGES * stage + 8192 + 512 + 1024;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(conv0_kernel<WGRAD, PARTIAL>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess)
      throw std::runtime_error(std::string("[b200] cudaFuncSetAttribute(conv0): ") + cudaGetErrorString(e));
    configured = true;
  }
  conv0_kernel<WGRAD, PARTIAL><<<grid, C0_THREADS, smem, stream>>>(prm);
  count_launch();
  check_last("conv0_kernel launch");
}

void conv0_fprop(const bf16* x4, const bf16* w0, const float* bias, bf16* y, int N, int H, int W,
                 cudaStream_t stream) {
  Conv0Params prm;
  prm.x4 = x4; prm.out = y; prm.bias = bias; prm.dW = nullptr;
  prm.N = N; prm.H = H; prm.W = W; prm.pixels = static_cast<long long>(N) * H * W;
  prm.num_tiles = static_cast<int>((prm.pixels + 127) / 128);
  prm.blocks_per_cta = 0;
  map_2d(&prm.mapW, w0, 64, 64, 64, 64, 64);
  prm.mapZ = prm.mapW;
  conv0_launch<false>(prm, prm.num_tiles < num_sms() ? prm.num_tiles : num_sms(), stream);
}

// CTAs of the layer-0 wgrad and the 64-pixel k-blocks each takes.
static int conv0_wgrad_grid(int N, int H, int W, int sms, int* num_tiles, int* blocks_per_cta) {
  const long long pixels = static_cast<long long>(N) * H * W;
  *num_tiles = static_cast<int>((pixels + 63) / 64);
  int grid = *num_tiles < sms ? *num_tiles : sms;
  *blocks_per_cta = (*num_tiles + grid - 1) / grid;
  return (*num_tiles + *blocks_per_cta - 1) / *blocks_per_cta;
}
int conv0_wgrad_splits(int N, int H, int W, int sms) {
  int tiles, per_cta;
  return 2 * conv0_wgrad_grid(N, H, W, sms, &tiles, &per_cta);   // one slice per (CTA, consumer warpgroup)
}

// A split-K workspace must hold `splits` slices of `elems` floats (each padded to whole float4s).
static void check_workspace(const char* what, const float* ws, long long ws_elems, int splits, long long elems) {
  if (!ws || (reinterpret_cast<uintptr_t>(ws) & 15) != 0)
    throw std::runtime_error(std::string("[b200] ") + what + ": the split-K workspace must be a 16-byte aligned buffer");
  if (ws_elems < splits * workspace_slice(elems))
    throw std::runtime_error(std::string("[b200] ") + what + ": the split-K workspace holds " + std::to_string(ws_elems) +
                             " floats, this launch writes " + std::to_string(splits) + " slices of " +
                             std::to_string(workspace_slice(elems)));
}

static void conv0_wgrad_impl(const bf16* dz, const bf16* x4, float* dw0, long long ws_elems, bool partial, int N,
                             int H, int W, cudaStream_t stream) {
  Conv0Params prm;
  prm.x4 = x4; prm.out = nullptr; prm.bias = nullptr; prm.dW = dw0;
  prm.N = N; prm.H = H; prm.W = W; prm.pixels = static_cast<long long>(N) * H * W;
  const int grid = conv0_wgrad_grid(N, H, W, num_sms(), &prm.num_tiles, &prm.blocks_per_cta);
  if (partial) check_workspace("conv0_wgrad_partial", dw0, ws_elems, 2 * grid, 64 * 64);
  map_2d(&prm.mapZ, dz, prm.pixels, 64, 64, 64, 64);
  prm.mapW = prm.mapZ;
  if (partial) conv0_launch<true, true>(prm, grid, stream);
  else conv0_launch<true>(prm, grid, stream);
}
void conv0_wgrad(const bf16* dz, const bf16* x4, float* dw0, int N, int H, int W, cudaStream_t stream) {
  conv0_wgrad_impl(dz, x4, dw0, 0, false, N, H, W, stream);
}
int conv0_wgrad_partial(const bf16* dz, const bf16* x4, float* ws, long long ws_elems, int N, int H, int W,
                        cudaStream_t stream) {
  conv0_wgrad_impl(dz, x4, ws, ws_elems, true, N, H, W, stream);
  return conv0_wgrad_splits(N, H, W, num_sms());
}

// ---------------------------------------------------------------------------------------- GEMM
template <int BN, bool A_MN, bool B_MN, int EPI>
static void gemm_launch(GemmParams& prm, const bf16* A, long long lda, const bf16* B, long long ldb,
                        int M, int N, int K, int ksplit, cudaStream_t stream) {
  using P = GemmPolicy<BN, umma_stages<BN, 0>(), A_MN, B_MN, EPI>;
  if (A_MN) map_2d(&prm.mapA, A, K, M, lda, 64, 64); else map_2d(&prm.mapA, A, M, K, lda, 64, UMMA_BM);
  if (B_MN) map_2d(&prm.mapB, B, K, N, ldb, 64, 64); else map_2d(&prm.mapB, B, N, K, ldb, 64, BN);
  prm.tiles_m = (M + UMMA_BM - 1) / UMMA_BM;
  prm.tiles_n = (N + BN - 1) / BN;
  prm.num_tiles = prm.tiles_m * prm.tiles_n * ksplit;
  launch<P>(prm, stream);
}

#define GEMM_BN_SWITCH(AMN, BMN, EPI)                                                       \
  switch (bn) {                                                                             \
    case 64:  gemm_launch<64,  AMN, BMN, EPI>(prm, A, lda, B, ldb, M, N, K, ksplit, stream); return; \
    case 128: gemm_launch<128, AMN, BMN, EPI>(prm, A, lda, B, ldb, M, N, K, ksplit, stream); return; \
    default: break;                                                                         \
  }
#define GEMM_BN_SWITCH_32(AMN, BMN, EPI)                                                    \
  if (bn == 32) { gemm_launch<32, AMN, BMN, EPI>(prm, A, lda, B, ldb, M, N, K, ksplit, stream); return; } \
  GEMM_BN_SWITCH(AMN, BMN, EPI)

// Splits a GEMM over K really makes when asked for `ksplit`: whole 64-wide k-blocks, none empty.
int gemm_splits(int K, int ksplit) {
  const int total = (K + UMMA_BK - 1) / UMMA_BK;
  if (ksplit < 1) ksplit = 1;
  const int per_split = (total + ksplit - 1) / ksplit;
  return (total + per_split - 1) / per_split;
}

// `ws_elems` > 0: `out` is a split-K workspace of that many floats (the PARTIAL epilogues).
static void gemm_impl(const bf16* A, long long lda, bool a_mn, const bf16* B, long long ldb, bool b_mn,
                      int M, int N, int K, void* out, long long ldo, int epi, const float* bias,
                      float alpha, int ksplit, int bn, long long ws_elems, cudaStream_t stream) {
  // Tiles are at most 128 wide here: the FC forward and dgrad have the batch as N (swap-AB), and
  // the FC wgrad has it as K -- one k-block per tile, bound by storing its output, which a wider
  // tile does not shorten.  256-wide tiles are built for the convolutions only (conv_bn).
  if (bn == 0) bn = N <= 32 && !b_mn ? 32 : (N <= 64 ? 64 : 128);
  if (ksplit < 1) ksplit = 1;
  GemmParams prm;
  prm.M = M; prm.N = N;
  prm.k_iters_total = (K + UMMA_BK - 1) / UMMA_BK;
  prm.k_iters_per_split = (prm.k_iters_total + ksplit - 1) / ksplit;
  ksplit = (prm.k_iters_total + prm.k_iters_per_split - 1) / prm.k_iters_per_split;
  prm.out = out; prm.ldo = ldo; prm.bias = bias; prm.alpha = alpha;
  const bool partial = epi == EPI_F32_PARTIAL || epi == EPI_F32_PARTIAL_T;
  // a slice is the output as the matching ATOMIC epilogue addresses it: [M][ldo], transposed [N][ldo]
  const long long slice_elems = static_cast<long long>(epi == EPI_F32_PARTIAL_T ? N : M) * ldo;
  prm.slice = partial ? workspace_slice(slice_elems) : 0;
  if (partial) check_workspace("gemm_bf16_partial", static_cast<const float*>(out), ws_elems, ksplit, slice_elems);
  if (ksplit > 1 && !(epi == EPI_F32_ATOMIC || epi == EPI_F32_ATOMIC_T || partial))
    throw std::runtime_error("[b200] gemm_bf16: split-K needs an atomic or a partial epilogue");
  if (!a_mn && !b_mn) {
    if (epi == EPI_F32_PARTIAL_T) { GEMM_BN_SWITCH_32(false, false, EPI_F32_PARTIAL_T) }
    if (epi == EPI_F32_ATOMIC_T) { GEMM_BN_SWITCH_32(false, false, EPI_F32_ATOMIC_T) }
    if (epi == EPI_F32_STORE_T) { GEMM_BN_SWITCH_32(false, false, EPI_F32_STORE_T) }
    if (epi == EPI_BF16_BIAS_RELU) { GEMM_BN_SWITCH(false, false, EPI_BF16_BIAS_RELU) }
    if (epi == EPI_F32_STORE) { GEMM_BN_SWITCH(false, false, EPI_F32_STORE) }
  } else if (a_mn && !b_mn) {
    if (epi == EPI_F32_PARTIAL_T) { GEMM_BN_SWITCH_32(true, false, EPI_F32_PARTIAL_T) }
    if (epi == EPI_F32_ATOMIC_T) { GEMM_BN_SWITCH_32(true, false, EPI_F32_ATOMIC_T) }
    if (epi == EPI_F32_STORE_T) { GEMM_BN_SWITCH_32(true, false, EPI_F32_STORE_T) }
  } else if (a_mn && b_mn) {
    if (epi == EPI_F32_STORE) { GEMM_BN_SWITCH(true, true, EPI_F32_STORE) }
    if (epi == EPI_F32_ATOMIC) { GEMM_BN_SWITCH(true, true, EPI_F32_ATOMIC) }
    if (epi == EPI_F32_PARTIAL) { GEMM_BN_SWITCH(true, true, EPI_F32_PARTIAL) }
    if (epi == EPI_BF16_STORE) { GEMM_BN_SWITCH(true, true, EPI_BF16_STORE) }
  }
  throw std::runtime_error("[b200] gemm_bf16: unsupported (layout, epilogue, bn) combination");
}

void gemm_bf16(const bf16* A, long long lda, bool a_mn, const bf16* B, long long ldb, bool b_mn,
               int M, int N, int K, void* out, long long ldo, int epi, const float* bias,
               float alpha, int ksplit, int bn, cudaStream_t stream) {
  if (epi == EPI_F32_PARTIAL || epi == EPI_F32_PARTIAL_T)
    throw std::runtime_error("[b200] gemm_bf16: the partial epilogues take a workspace (gemm_bf16_partial)");
  gemm_impl(A, lda, a_mn, B, ldb, b_mn, M, N, K, out, ldo, epi, bias, alpha, ksplit, bn, 0, stream);
}
int gemm_bf16_partial(const bf16* A, long long lda, bool a_mn, const bf16* B, long long ldb, bool b_mn, int M,
                      int N, int K, float* ws, long long ws_elems, long long ldo, bool transposed, float alpha,
                      int ksplit, int bn, cudaStream_t stream) {
  const int splits = gemm_splits(K, ksplit);
  gemm_impl(A, lda, a_mn, B, ldb, b_mn, M, N, K, ws, ldo, transposed ? EPI_F32_PARTIAL_T : EPI_F32_PARTIAL, nullptr,
            alpha, splits, bn, ws_elems, stream);
  return splits;
}

// ---------------------------------------------------------------------------------------- conv
static void check_channels(int c, const char* what) {
  if (c % 64 != 0) throw std::runtime_error(std::string("[b200] ") + what + " must be a multiple of 64");
}

template <int BN, bool DGRAD, bool POOL = false, bool FILL = false>
static void conv_launch(ConvParams& prm, cudaStream_t stream) {
  using P = ConvPolicy<BN, umma_stages<BN, ConvPolicy<BN, 1, DGRAD, POOL>::EPI_SMEM>(), DGRAD, POOL, FILL>;
  const ConvTile& t = prm.t;
  const int tiles_n = (t.N + t.Nb - 1) / t.Nb;
  prm.tiles_m = t.tiles_w * t.tiles_h * tiles_n;
  prm.div_tm = make_fastdiv(prm.tiles_m);
  prm.num_tiles = prm.tiles_m * ((prm.Cn + BN - 1) / BN);
  launch<P>(prm, stream);
}

// Channel-tile width of a convolution with `cn` output channels, from the tile counts at 128 and
// 256 columns.  A 256-wide tile does twice the work of a 128-wide one but reads the activation tile
// once instead of twice, and takes 1.67-1.77x as long (the 56^2, 28^2 and 14^2 layers at batch 64,
// per wave; H100 80GB HBM3, 700 W): 7/4.  It is taken where the number of waves over the SMs times
// that cost is no worse than at 128 -- at batch 64 on 132 SMs every 56^2 and 28^2 layer, not the
// 14^2 ones, whose 196 wide tiles take 2 waves x 7/4 against 392 narrow tiles in 3 waves x 1.
static int conv_bn(int cn, long long tiles128, long long tiles256, long long sms) {
  if (cn <= 64) return 64;
  if (cn < 256) return 128;
  return ((tiles256 + sms - 1) / sms) * 7 <= ((tiles128 + sms - 1) / sms) * 4 ? 256 : 128;
}

// Pixel-tile splits of the halo wgrad: one work item per SM, none empty.
static int wgrad_halo64_splits(int total_tiles, int tiles_n, int sms, int* tiles_per_split) {
  int ksplit = sms / tiles_n;
  if (ksplit < 1) ksplit = 1;
  if (ksplit > total_tiles) ksplit = total_tiles;
  *tiles_per_split = (total_tiles + ksplit - 1) / ksplit;
  return (total_tiles + *tiles_per_split - 1) / *tiles_per_split;
}
static bool wgrad_halo64_applicable(int H, int W, int Cin) {
  return Cin == 64 && H % WH_T == 0 && W % WH_T == 0 && W >= 16 && halo_enabled();
}

// Pixel-tile splits of the generic wgrad when every split stores a slice of partials that a second
// kernel adds up.  A slice costs a write and a read of Cout*9*Cin floats, so the 4096-pixel work
// items of the atomic path (196 splits, 115 MB of partials at 128 -> 128 channels, 112^2, batch 64)
// are too fine.  Of the counts that give at most ~4 work items per SM, take the one with the least
// modelled time: waves over the SMs x k-blocks per item, plus the slices' traffic in the same unit
// (WS_ELEMS_PER_KBLOCK floats written and read back in the time one SM takes for a k-block:
// ~0.5 us against ~2.5 TB/s; a model, see DESIGN 2.9 for what was measured).  Ties: fewer splits.
constexpr long long WS_ELEMS_PER_KBLOCK = 160000;
static int wgrad_partial_ksplit(int total_tiles, int base, long long slice_elems, int sms) {
  int kmax = (4 * sms + base - 1) / base;
  if (kmax > total_tiles) kmax = total_tiles;
  int best = 1;
  long long best_cost = -1;
  for (int k = 1; k <= kmax; ++k) {
    const long long waves = (static_cast<long long>(base) * k + sms - 1) / sms;
    const long long depth = (total_tiles + k - 1) / k;
    const long long cost = waves * depth * WS_ELEMS_PER_KBLOCK + k * slice_elems;
    if (best_cost < 0 || cost < best_cost) { best = k; best_cost = cost; }
  }
  return best;
}

// conv_plan with the launchers' explicit choices: a tile width `bn` (0: chosen here) and a wgrad split
// `ksplit` (<= 0: chosen here); either one takes the wgrad off the halo64 kernel.  `tile` (optional)
// receives the pixel tile of the implicit-GEMM and generic wgrad paths.
static ConvPlan plan_conv(int kind, int N, int H, int W, int Cin, int Cout, int sms, int bn, int ksplit,
                          ConvTile* tile) {
  ConvPlan p{};
  if (kind == CONV_KIND_WGRAD || kind == CONV_KIND_WGRAD_PARTIAL) {
    if (bn == 0 && ksplit <= 0 && wgrad_halo64_applicable(H, W, Cin)) {
      p.path = CONV_PATH_WGRAD_HALO64;
      p.bn = 64; p.Wb = WH_T; p.Hb = WH_T; p.Nb = 1;
      p.tiles = static_cast<long long>(N) * (W / WH_T) * (H / WH_T);
      p.ksplit = wgrad_halo64_splits(static_cast<int>(p.tiles), (Cout + 63) / 64, sms, &p.tiles_per_split);
      return p;
    }
    const ConvTile t = make_tile(N, H, W, 64);
    const int total = static_cast<int>(conv_tile_count(t));
    // The split is chosen for the width asked for, or for the narrow tile when the width is chosen
    // here; a 256-wide tile then keeps that split, so it has half as many work items of the same depth.
    const int split_bn = bn ? bn : (Cin <= 64 ? 64 : 128);
    if (ksplit <= 0) {     // work items of <= ~64 k-blocks (4096 pixels), and at least ~4 per SM
      const int base = ((Cout + UMMA_BM - 1) / UMMA_BM) * ((Cin + split_bn - 1) / split_bn) * 9;
      if (kind == CONV_KIND_WGRAD_PARTIAL) {
        ksplit = wgrad_partial_ksplit(total, base, static_cast<long long>(Cout) * 9 * Cin, sms);
      } else {
        ksplit = (total + 63) / 64;
        const int min_split = (4 * sms + base - 1) / base;
        if (ksplit < min_split) ksplit = min_split;
      }
    }
    if (ksplit > total) ksplit = total;
    p.path = CONV_PATH_WGRAD;
    p.Wb = t.Wb; p.Hb = t.Hb; p.Nb = t.Nb;
    p.tiles = total;
    p.tiles_per_split = (total + ksplit - 1) / ksplit;
    p.ksplit = (total + p.tiles_per_split - 1) / p.tiles_per_split;
    if (bn == 0) {
      const long long items = static_cast<long long>((Cout + UMMA_BM - 1) / UMMA_BM) * 9 * p.ksplit;
      bn = conv_bn(Cin, items * ((Cin + 127) / 128), items * ((Cin + 255) / 256), sms);
    }
    p.bn = bn;
    if (tile) *tile = t;
    return p;
  }
  const bool dgrad = kind == CONV_KIND_DGRAD;
  const int cn = dgrad ? Cin : Cout;          // output channels (GEMM N)
  const int ca = dgrad ? Cout : Cin;          // channels of the A activation (GEMM K per tap)
  p.ksplit = 1;
  if (halo_applicable(H, W)) {                // the halo kernel's own 8 x 16 x 1 tiles
    p.path = CONV_PATH_HALO;
    p.bn = bn ? bn : (cn <= 64 ? 64 : 128);
    p.Wb = HALO_WT; p.Hb = HALO_HT; p.Nb = 1;
    p.tiles = static_cast<long long>(W / HALO_WT) * (H / HALO_HT) * N;
    p.tiles_per_split = static_cast<int>(p.tiles);
    const int nb = p.bn == 64 ? HaloCfg<64>::NB : HaloCfg<128>::NB;
    p.resident = ((cn + p.bn - 1) / p.bn == 1 && 9 * (ca / UMMA_BK) <= nb) ? 1 : 0;
    return p;
  }
  ConvTile t = make_tile(N, H, W, UMMA_BM);
  const bool fill = kind != CONV_KIND_FPROP_POOL && conv_fill_tile(N, H, W, &t);
  p.path = fill ? CONV_PATH_FILL : CONV_PATH_POW2;
  p.Wb = t.Wb; p.Hb = t.Hb; p.Nb = t.Nb;
  p.tiles = conv_tile_count(t);
  p.tiles_per_split = static_cast<int>(p.tiles);
  // the pixel tiles are the same at both widths
  p.bn = bn ? bn : conv_bn(cn, p.tiles * ((cn + 127) / 128), p.tiles * ((cn + 255) / 256), sms);
  if (tile) *tile = t;
  return p;
}

ConvPlan conv_plan(int kind, int N, int H, int W, int Cin, int Cout, int sms, int bn) {
  if (kind < CONV_KIND_FPROP || kind > CONV_KIND_WGRAD_PARTIAL) throw std::runtime_error("[b200] conv_plan: unknown kind");
  if (N < 1 || H < 1 || W < 1 || Cin < 1 || Cout < 1 || sms < 1)
    throw std::runtime_error("[b200] conv_plan: extents and the SM count must be positive");
  if (bn != 0 && bn != 64 && bn != 128 && bn != 256)
    throw std::runtime_error("[b200] conv_plan: bn must be 0 (chosen), 64, 128 or 256");
  return plan_conv(kind, N, H, W, Cin, Cout, sms, bn, 0, nullptr);
}

void conv_pixel_box(int N, int H, int W, int* box) {
  const ConvPlan p = conv_plan(CONV_KIND_FPROP, N, H, W, 64, 64, num_sms());
  box[0] = p.Wb; box[1] = p.Hb; box[2] = p.Nb; box[3] = p.path == CONV_PATH_FILL ? 1 : 0;
}

int conv_bn_choice(int N, int H, int W, int cn) { return conv_plan(CONV_KIND_FPROP, N, H, W, 64, cn, num_sms()).bn; }

static void fprop_impl(const bf16* x, const bf16* w, const float* bias, bf16* y, bf16* pool_out,
                       uint32_t* pool_mask, int N, int H, int W, int Cin, int Cout, bool relu, int bn,
                       cudaStream_t stream) {
  check_channels(Cin, "conv3x3_fprop Cin");
  check_channels(Cout, "conv3x3_fprop Cout");
  // the epilogue stages the bias in a 512-float shared-memory scratch (ConvPolicy::EPI_MAXC)
  if (bias && Cout > 512) throw std::runtime_error("[b200] conv3x3_fprop: a bias supports Cout <= 512");
  const bool pool = pool_out != nullptr;
  ConvParams prm;
  const ConvPlan plan = plan_conv(pool ? CONV_KIND_FPROP_POOL : CONV_KIND_FPROP, N, H, W, Cin, Cout, num_sms(), bn,
                                  0, &prm.t);
  bn = plan.bn;
  prm.t.N = N; prm.t.H = H; prm.t.W = W;
  prm.Ca = Cin; prm.Cn = Cout; prm.wcols_per_tap = Cin;
  prm.out = y; prm.bias = bias; prm.mask_src = nullptr; prm.colsum = nullptr;
  prm.pool_out = pool_out; prm.pool_mask = pool_mask;
  prm.flags = (bias ? CONV_BIAS : 0) | (relu ? CONV_RELU : 0) | (pool_out ? CONV_POOL : 0);
  prm.resident = plan.resident;
  map_2d(&prm.mapB, w, Cout, 9LL * Cin, 9LL * Cin, 64, bn);
  if (plan.path == CONV_PATH_HALO) {
    switch (bn) {
      case 64: pool ? conv_halo_launch<64, false, true>(prm, x, stream) : conv_halo_launch<64, false>(prm, x, stream); return;
      case 128: pool ? conv_halo_launch<128, false, true>(prm, x, stream) : conv_halo_launch<128, false>(prm, x, stream); return;
      default: throw std::runtime_error("[b200] conv3x3_fprop: bn must be 64 or 128");
    }
  }
  map_nhwc(&prm.mapA, x, N, H, W, Cin, prm.t.Wb, prm.t.Hb, prm.t.Nb);
  if (plan.path == CONV_PATH_FILL) {
    set_fill(prm);
    switch (bn) {
      case 64: conv_launch<64, false, false, true>(prm, stream); return;
      case 128: conv_launch<128, false, false, true>(prm, stream); return;
      case 256: conv_launch<256, false, false, true>(prm, stream); return;
      default: throw std::runtime_error("[b200] conv3x3_fprop: bn must be 64, 128 or 256");
    }
  }
  switch (bn) {
    case 64: pool ? conv_launch<64, false, true>(prm, stream) : conv_launch<64, false>(prm, stream); break;
    case 128: pool ? conv_launch<128, false, true>(prm, stream) : conv_launch<128, false>(prm, stream); break;
    case 256: pool ? conv_launch<256, false, true>(prm, stream) : conv_launch<256, false>(prm, stream); break;
    default: throw std::runtime_error("[b200] conv3x3_fprop: bn must be 64, 128 or 256");
  }
}

void conv3x3_fprop(const bf16* x, const bf16* w, const float* bias, bf16* y, int N, int H, int W,
                   int Cin, int Cout, bool relu, int bn, cudaStream_t stream) {
  fprop_impl(x, w, bias, y, nullptr, nullptr, N, H, W, Cin, Cout, relu, bn, stream);
}

// The pool windows must lie inside one epilogue warp (see ConvPolicy::epilogue_pool).
bool conv3x3_pool_fusable(int N, int H, int W) {
  if (H % 2 || W % 2) return false;
  if (halo_applicable(H, W)) return true;               // 8 x 16 tiles
  const ConvTile t = make_tile(N, H, W, UMMA_BM);
  return t.Wb <= 16 && t.Hb >= 2 && W % t.Wb == 0 && H % t.Hb == 0;
}

void conv3x3_fprop_pool(const bf16* x, const bf16* w, const float* bias, bf16* pool_out, uint32_t* pool_mask,
                        int N, int H, int W, int Cin, int Cout, int bn, cudaStream_t stream) {
  if (!conv3x3_pool_fusable(N, H, W))
    throw std::runtime_error("[b200] conv3x3_fprop_pool: this image size cannot fuse the 2x2 pool");
  if (!pool_out || !pool_mask) throw std::runtime_error("[b200] conv3x3_fprop_pool: missing outputs");
  fprop_impl(x, w, bias, nullptr, pool_out, pool_mask, N, H, W, Cin, Cout, true, bn, stream);
}

void conv3x3_dgrad(const bf16* dz, const bf16* w, const bf16* mask_src, bf16* dx, float* colsum, int N,
                   int H, int W, int Cin, int Cout, int bn, cudaStream_t stream) {
  check_channels(Cin, "conv3x3_dgrad Cin");
  check_channels(Cout, "conv3x3_dgrad Cout");
  if (colsum && Cin > 512) throw std::runtime_error("[b200] conv3x3_dgrad: fused column sum supports Cin <= 512");
  ConvParams prm;
  const ConvPlan plan = plan_conv(CONV_KIND_DGRAD, N, H, W, Cin, Cout, num_sms(), bn, 0, &prm.t);
  bn = plan.bn;
  prm.t.N = N; prm.t.H = H; prm.t.W = W;
  prm.Ca = Cout; prm.Cn = Cin; prm.wcols_per_tap = Cin;
  prm.out = dx; prm.bias = nullptr; prm.mask_src = mask_src; prm.colsum = colsum;
  prm.pool_out = nullptr; prm.pool_mask = nullptr;
  prm.flags = (mask_src ? CONV_MASK : 0) | (colsum ? CONV_COLSUM : 0);
  prm.resident = plan.resident;
  map_2d(&prm.mapB, w, Cout, 9LL * Cin, 9LL * Cin, 64, 64);   // MN-major: 64 ci x 64 co boxes
  if (plan.path == CONV_PATH_HALO) {
    switch (bn) {
      case 64: conv_halo_launch<64, true>(prm, dz, stream); return;
      case 128: conv_halo_launch<128, true>(prm, dz, stream); return;
      default: throw std::runtime_error("[b200] conv3x3_dgrad: bn must be 64 or 128");
    }
  }
  map_nhwc(&prm.mapA, dz, N, H, W, Cout, prm.t.Wb, prm.t.Hb, prm.t.Nb);
  if (plan.path == CONV_PATH_FILL) {
    set_fill(prm);
    switch (bn) {
      case 64: conv_launch<64, true, false, true>(prm, stream); return;
      case 128: conv_launch<128, true, false, true>(prm, stream); return;
      case 256: conv_launch<256, true, false, true>(prm, stream); return;
      default: throw std::runtime_error("[b200] conv3x3_dgrad: bn must be 64, 128 or 256");
    }
  }
  switch (bn) {
    case 64: conv_launch<64, true>(prm, stream); break;
    case 128: conv_launch<128, true>(prm, stream); break;
    case 256: conv_launch<256, true>(prm, stream); break;
    default: throw std::runtime_error("[b200] conv3x3_dgrad: bn must be 64, 128 or 256");
  }
}

template <int BN, bool PARTIAL = false>
static void wgrad_launch(WgradParams& prm, cudaStream_t stream) {
  using P = WgradPolicy<BN, umma_stages<BN, 0>(), PARTIAL>;
  prm.tiles_m = (prm.Cout + UMMA_BM - 1) / UMMA_BM;
  prm.tiles_n = (prm.Cin + BN - 1) / BN;
  prm.num_tiles = prm.tiles_m * prm.tiles_n * 9 * prm.ksplit;
  launch<P>(prm, stream);
}

// 64-input-channel layers on 8-divisible maps: nine tap views of one X halo per pixel tile.
template <bool PARTIAL = false>
static int wgrad_halo64_launch(const ConvPlan& plan, const bf16* dz, const bf16* x, float* dw, long long ws_elems,
                               int N, int H, int W, int Cout, float scale, cudaStream_t stream) {
  WgradHaloParams prm;
  prm.tiles_n = (Cout + 63) / 64;
  prm.tiles_w = W / WH_T; prm.tiles_h = H / WH_T;
  prm.total_tiles = static_cast<int>(plan.tiles);
  prm.tiles_per_split = plan.tiles_per_split;
  if (PARTIAL) check_workspace("conv3x3_wgrad_partial", dw, ws_elems, plan.ksplit, static_cast<long long>(Cout) * 9 * 64);
  prm.num_items = prm.tiles_n * plan.ksplit;
  prm.Cout = Cout; prm.dW = dw; prm.scale = scale;
  map_nhwc(&prm.mapX, x, N, H, W, 64, WH_PITCH, WH_PITCH, 1);
  map_nhwc(&prm.mapZ, dz, N, H, W, Cout, WH_T, WH_T, 1);
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(wgrad_halo64_kernel<PARTIAL>, cudaFuncAttributeMaxDynamicSharedMemorySize, WH_SMEM);
    if (e != cudaSuccess)
      throw std::runtime_error(std::string("[b200] cudaFuncSetAttribute(wgrad halo): ") + cudaGetErrorString(e));
    configured = true;
  }
  dim3 grid(prm.num_items < num_sms() ? prm.num_items : num_sms());
  wgrad_halo64_kernel<PARTIAL><<<grid, WH_THREADS, WH_SMEM, stream>>>(prm);
  count_launch();
  check_last("wgrad_halo64_kernel launch");
  return plan.ksplit;
}

int conv_wgrad_splits(int N, int H, int W, int Cin, int Cout, int sms) {
  return conv_plan(CONV_KIND_WGRAD_PARTIAL, N, H, W, Cin, Cout, sms).ksplit;
}

static int wgrad_impl(const bf16* dz, const bf16* x, float* dw, long long ws_elems, bool partial, int N, int H,
                      int W, int Cin, int Cout, float scale, int ksplit, int bn, cudaStream_t stream) {
  check_channels(Cin, "conv3x3_wgrad Cin");
  check_channels(Cout, "conv3x3_wgrad Cout");
  WgradParams prm;
  const ConvPlan plan = plan_conv(partial ? CONV_KIND_WGRAD_PARTIAL : CONV_KIND_WGRAD, N, H, W, Cin, Cout, num_sms(),
                                  bn, ksplit, &prm.t);
  if (plan.path == CONV_PATH_WGRAD_HALO64) {
    if (partial) return wgrad_halo64_launch<true>(plan, dz, x, dw, ws_elems, N, H, W, Cout, scale, stream);
    return wgrad_halo64_launch(plan, dz, x, dw, 0, N, H, W, Cout, scale, stream);
  }
  prm.Cout = Cout; prm.Cin = Cin;
  prm.total_tiles = static_cast<int>(plan.tiles);
  prm.tiles_per_split = plan.tiles_per_split;
  prm.ksplit = plan.ksplit;
  if (partial) check_workspace("conv3x3_wgrad_partial", dw, ws_elems, prm.ksplit, static_cast<long long>(Cout) * 9 * Cin);
  prm.dW = dw; prm.scale = scale;
  map_nhwc(&prm.mapA, dz, N, H, W, Cout, prm.t.Wb, prm.t.Hb, prm.t.Nb);
  map_nhwc(&prm.mapB, x, N, H, W, Cin, prm.t.Wb, prm.t.Hb, prm.t.Nb);
  switch (plan.bn) {
    case 64: partial ? wgrad_launch<64, true>(prm, stream) : wgrad_launch<64>(prm, stream); break;
    case 128: partial ? wgrad_launch<128, true>(prm, stream) : wgrad_launch<128>(prm, stream); break;
    case 256: partial ? wgrad_launch<256, true>(prm, stream) : wgrad_launch<256>(prm, stream); break;
    default: throw std::runtime_error("[b200] conv3x3_wgrad: bn must be 64, 128 or 256");
  }
  return prm.ksplit;
}

void conv3x3_wgrad(const bf16* dz, const bf16* x, float* dw, int N, int H, int W, int Cin,
                   int Cout, float scale, int ksplit, int bn, cudaStream_t stream) {
  wgrad_impl(dz, x, dw, 0, false, N, H, W, Cin, Cout, scale, ksplit, bn, stream);
}
int conv3x3_wgrad_partial(const bf16* dz, const bf16* x, float* ws, long long ws_elems, int N, int H, int W,
                          int Cin, int Cout, float scale, cudaStream_t stream) {
  return wgrad_impl(dz, x, ws, ws_elems, true, N, H, W, Cin, Cout, scale, 0, 0, stream);
}

}  // namespace b200
