// Host-callable entry points of the native library (raw pointers + stream; no torch types so the
// .cu files compile in seconds).  bindings.cpp adapts torch tensors onto these.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <cstdint>
#include <vector>

namespace b200 {

typedef __nv_bfloat16 bf16;

// Number of kernels launched by this library since load (bench.py reports it as gpu_launches).
long long launch_count();
void count_launch(int n = 1);
void check_last(const char* what);
// multiProcessorCount of the current device (cached; grids are sized from it, never from a literal)
int sm_count();
// Kernels that run on the comm stream UNDER the persistent conv kernels must ask for the same L1 /
// shared-memory split as those (maximum shared memory): an SM only changes its carve-out when it is
// empty, so a resident CTA of a kernel with the default (L1-heavy) preference keeps every conv CTA --
// which needs > 200 KB of shared memory -- off that SM until it exits (bench/interference.py: a
// background kernel that only sleeps slowed the convolutions by 1.3-1.6x).  Call once per kernel.
void prefer_max_shared_carveout(const void* kernel);
bool comm_carveout_enabled();   // B200_COMM_CARVEOUT=0 switches the above off (A/B measurements)

// ---- wgmma GEMM family (umma_launch.cu) -------------------------------------------------------
// D[M,N] = alpha * sum_k A[m,k] * B[n,k].  a_mn: A is stored [K][M] (row stride lda) instead of
// [M][K]; same for b_mn.  epi: GemmEpi.  ksplit > 1 needs an ATOMIC epilogue and a zeroed output.
void gemm_bf16(const bf16* A, long long lda, bool a_mn, const bf16* B, long long ldb, bool b_mn,
               int M, int N, int K, void* out, long long ldo, int epi, const float* bias,
               float alpha, int ksplit, int bn, cudaStream_t stream);

// First convolution (3 -> 64 channels) straight from NHWC4 pixels: the im2col operand tile is built
// in shared memory by producer warps (conv0.cuh).  w0 is [64][64] bf16 (k = (kh*3+kw)*3+c, zero tail).
void conv0_fprop(const bf16* x4, const bf16* w0, const float* bias, bf16* y, int N, int H, int W,
                 cudaStream_t stream);
void conv0_wgrad(const bf16* dz, const bf16* x4, float* dw0, int N, int H, int W, cudaStream_t stream);

// 3x3 / stride 1 / pad 1 convolution, NHWC bf16, weights [Cout][3][3][Cin] bf16.
void conv3x3_fprop(const bf16* x, const bf16* w, const float* bias, bf16* y, int N, int H, int W,
                   int Cin, int Cout, bool relu, int bn, cudaStream_t stream);
// EXPERIMENTAL (B200_FUSE_POOL=1): conv + bias + ReLU + 2x2/2 max-pool in one kernel.  Writes the
// pooled activation [N,H/2,W/2,Cout] and, per pooled pixel and 32 channels, four words {argmax bit 0,
// argmax bit 1, max > 0, 0}; the un-pooled activation is never materialised.  unpool2x2 is the
// matching backward (elementwise.cu).
bool conv3x3_pool_fusable(int N, int H, int W);
// What a 3x3 convolution launch runs, as the launchers choose it for `sms` SMs: pure host code, so it
// can be asked where no GPU is present.  conv3x3_fprop / _fprop_pool / _dgrad / _wgrad / _wgrad_partial
// with their default tile width and split take every choice from here.
enum ConvKind { CONV_KIND_FPROP, CONV_KIND_FPROP_POOL, CONV_KIND_DGRAD, CONV_KIND_WGRAD, CONV_KIND_WGRAD_PARTIAL };
enum ConvPath {
  CONV_PATH_HALO,          // conv_halo_kernel: 8 x 16 pixel halos
  CONV_PATH_POW2,          // implicit GEMM, make_tile's power-of-two pixel box
  CONV_PATH_FILL,          // implicit GEMM, a box of any sides (conv_fill_tile; the FILL kernels)
  CONV_PATH_WGRAD_HALO64,  // wgrad_halo64_kernel: 64 input channels, 8 x 8 pixel tiles
  CONV_PATH_WGRAD,         // WgradPolicy: 64-pixel power-of-two boxes
};
struct ConvPlan {
  int path;                // ConvPath
  int bn;                  // channel-tile width (wgrad_halo64: 64)
  int Wb, Hb, Nb;          // pixel box of one tile
  long long tiles;         // pixel tiles: fprop / dgrad per channel tile, wgrad over the whole reduction
  int ksplit;              // wgrad: splits of the pixel tiles (fprop / dgrad: 1)
  int tiles_per_split;     // wgrad: pixel tiles of every split but possibly the last (fprop / dgrad: tiles)
  int resident;            // halo: every weight tile stays in shared memory
};
// bn: a tile width the caller asks for (0: chosen here), as the launchers' bn argument; an explicit width
// also takes a wgrad off the halo64 kernel, and its split is then chosen for that width.
ConvPlan conv_plan(int kind, int N, int H, int W, int Cin, int Cout, int sms, int bn = 0);
// Views of conv_plan at the device's own SM count: the fprop box {Wb, Hb, Nb, fill} (fill = 1: the FILL
// path), and the fprop channel-tile width (64, 128 or 256) for cn output channels.  Both query the
// device; where none is present, ask conv_plan with an explicit SM count.
void conv_pixel_box(int N, int H, int W, int* box);
int conv_bn_choice(int N, int H, int W, int cn);
void conv3x3_fprop_pool(const bf16* x, const bf16* w, const float* bias, bf16* pool_out, uint32_t* pool_mask,
                        int N, int H, int W, int Cin, int Cout, int bn, cudaStream_t stream);
// dx[N,H,W,Cin] = conv_transpose(dz[N,H,W,Cout], w); optional mask: zero where mask_src <= 0;
// optional colsum[Cin] += sum over pixels of dx (the previous layer's bias gradient, fused).
void conv3x3_dgrad(const bf16* dz, const bf16* w, const bf16* mask_src, bf16* dx, float* colsum, int N,
                   int H, int W, int Cin, int Cout, int bn, cudaStream_t stream);
// dw[Cout][3][3][Cin] (fp32) += scale * sum_pixels dz * shifted x.
void conv3x3_wgrad(const bf16* dz, const bf16* x, float* dw, int N, int H, int W, int Cin,
                   int Cout, float scale, int ksplit, int bn, cudaStream_t stream);

// ---- split-K without atomics (bit-reproducible training) --------------------------------------
// Each split-K kernel has a `_partial` form that stores every split's tile into its own slice of a
// workspace, ws[split][output elements] (plain stores, one writer per element), and returns the number
// of slices it wrote; splitk_reduce then adds the slices in split order.  The `_splits` queries are the
// launchers' own split arithmetic as pure host functions of the shape and an SM count, for sizing the
// workspace (also where no GPU is present).  A launch refuses a workspace that is null, misaligned or
// too small before anything is enqueued.
inline long long workspace_slice(long long elems) { return (elems + 3) / 4 * 4; }   // slices start on float4s
int conv_wgrad_splits(int N, int H, int W, int Cin, int Cout, int sms);   // conv_plan(WGRAD_PARTIAL).ksplit
int conv0_wgrad_splits(int N, int H, int W, int sms);      // 2 per CTA: one per consumer warpgroup
int gemm_splits(int K, int ksplit);
int colsum_partial_blocks(long long rows, int C, int sms);
// ws[splits][Cout][9][Cin].  The split count differs from conv3x3_wgrad's: see wgrad_partial_ksplit.
int conv3x3_wgrad_partial(const bf16* dz, const bf16* x, float* ws, long long ws_elems, int N, int H, int W,
                          int Cin, int Cout, float scale, cudaStream_t stream);
// ws[splits][64][64]; a consumer warpgroup that had no k-block stores zeros.
int conv0_wgrad_partial(const bf16* dz, const bf16* x4, float* ws, long long ws_elems, int N, int H, int W,
                        cudaStream_t stream);
// gemm_bf16 with split-K into ws[splits][workspace_slice(M * ldo)] ([N * ldo] when `transposed`), each
// slice addressed as EPI_F32_ATOMIC (_T) addresses the output.
int gemm_bf16_partial(const bf16* A, long long lda, bool a_mn, const bf16* B, long long ldb, bool b_mn, int M,
                      int N, int K, float* ws, long long ws_elems, long long ldo, bool transposed, float alpha,
                      int ksplit, int bn, cudaStream_t stream);
// bias_grad's per-block sums as rows ws[blocks][C] (C % 8 == 0); returns blocks.
int colsum_partial(const bf16* dz, float* ws, long long ws_elems, long long rows, int C, float scale, cudaStream_t s);
// dst[i] = (accumulate ? dst[i] : 0) + alpha * (((ws[0][i] + ws[1][i]) + ws[2][i]) + ...) for i < n, slices
// `slice` floats apart, every operation rounded to fp32 on its own.
void splitk_reduce(const float* ws, long long ws_elems, float* dst, long long n, long long slice, int splits,
                   float alpha, bool accumulate, cudaStream_t s);

// ---- element-wise / reduction kernels (elementwise.cu) ----------------------------------------
void maxpool2x2_fwd(const bf16* x, bf16* y, int N, int H, int W, int C, cudaStream_t s);
// dz[N,H,W,C] = (y == pooled(y) first match && y > 0) ? dp[N,H/2,W/2,C] : 0
// optional colsum[C] += sum over pixels of dz (the layer's bias gradient, fused).
void maxpool2x2_relu_bwd(const bf16* y, const bf16* dp, bf16* dz, float* colsum, int N, int H, int W,
                         int C, cudaStream_t s);
// EXPERIMENTAL: backward of conv3x3_fprop_pool's pooling: dz[N,H,W,C] gets dp[N,H/2,W/2,C] at the
// recorded argmax where the maximum was positive, zero elsewhere; optional colsum as above.
void unpool2x2(const bf16* dp, const uint32_t* mask, bf16* dz, float* colsum, int N, int H, int W, int C,
               cudaStream_t s);
void adaptive_avgpool_fwd(const bf16* x, bf16* y, int N, int H, int W, int C, int OH, int OW,
                          cudaStream_t s);
void adaptive_avgpool_bwd(const bf16* dy, bf16* dx, int N, int H, int W, int C, int OH, int OW,
                          cudaStream_t s);
// db[c] += scale * sum_rows dz[row][c]      (rows = N*H*W for conv, batch for FC)
void bias_grad(const bf16* dz, float* db, long long rows, int C, float scale, cudaStream_t s);
// same for C % 8 != 0 (row stride ld), e.g. the 3-class logits gradient
void bias_grad_ld(const bf16* dz, float* db, long long rows, int C, int ld, float scale,
                  cudaStream_t s);
// FC epilogue: y = dropout(relu(acc + bias)) -> bf16; acc (fp32 [B][N]) is cleared for the next use.
void fc_bias_act(float* acc, const float* bias, bf16* y, float* y_f32, int B, int N, bool relu,
                 float drop_p, unsigned long long seed, unsigned long long offset, bool clear,
                 cudaStream_t s);
// FC backward epilogue: dz = acc * (act > 0) * dropmask/(1-p) -> bf16; acc cleared.
void fc_grad_act(float* acc, const bf16* act, bf16* dz, int B, int N, bool relu, float drop_p,
                 unsigned long long seed, unsigned long long offset, bool clear, cudaStream_t s);
// co-residency probe (bench/interference.py): thin background kernel exercising one SM resource
void probe_background(float* buf, long long n, int mode, int ctas, int reps, float* sink, cudaStream_t s);
void cast_f32_to_bf16(const float* x, bf16* y, long long n, cudaStream_t s);
void cast_bf16_to_f32(const bf16* x, float* y, long long n, cudaStream_t s);

// Fused cross-entropy forward+backward+metrics over fp32 logits [B][C].
// dlogits = (softmax - onehot) * grad_scale (bf16, ld = C rounded up to `ldd`);
// meter += {sum loss, #correct, B}; loss_out (optional) = mean loss of this batch.
void cross_entropy_fused(const float* logits, const long long* target, bf16* dlogits, int ldd,
                         float* meter, float* loss_out, int B, int C, float grad_scale,
                         const float* class_weights, cudaStream_t s);

// Soft targets of the loss (label smoothing eps, and MixUp / CutMix's probability targets).
// Row r's target is t = (lam_a e_{y_r} + lam_b e_{y_(r-1) mod B}) (1 - eps) + eps / C when `mix`, else
// (1 - eps) e_{y_r} + eps / C; the loss is sum_c w_c t_c (-log p_c) over rows, divided by sum_r w_{y_r}
// for integer targets (B without class weights) and by B for probability targets (torch's rules).
// A row is correct when argmax(logits) == argmax(lam_a e_{y_r} + lam_b e_{y_(r-1)}) (first maximum).
struct SoftTargets {
  float eps, lam_a, lam_b;
  int mix;
};
void cross_entropy_soft(const float* logits, const long long* target, bf16* dlogits, int ldd, float* meter,
                        float* loss_out, int B, int C, float grad_scale, const float* class_weights,
                        const SoftTargets& st, cudaStream_t s);

// Knowledge distillation against teacher logits u [B][C] fp32, weight alpha and temperature T:
//   L = (1 - alpha) CE + alpha T^2 / B sum_r KL(softmax(u_r / T) || softmax(z_r / T))
//   dL/dz[r][c] = (1 - alpha) (the cross-entropy gradient) + alpha T / B (softmax(z_r / T)_c - softmax(u_r / T)_c)
// CE is the loss of cross_entropy_fused / cross_entropy_soft (class weights and soft targets apply to it alone);
// meter / loss_out receive L.  kd_params(alpha, T, B) = {1 - alpha, alpha T / B, alpha T^2, 1 / T}.
struct KdParams {
  float ce, g, l, inv_t;
};
KdParams kd_params(double alpha, double temperature, int B);
void cross_entropy_kd(const float* logits, const long long* target, bf16* dlogits, int ldd, float* meter,
                      float* loss_out, int B, int C, float grad_scale, const float* class_weights,
                      const SoftTargets* soft, const float* teacher, const KdParams& kd, cudaStream_t s);

// K-FUN2+CE: last Linear(K -> C) + cross-entropy + metrics + the layer's whole backward in one launch
// (C <= 8, K <= 1024, B <= 256).  h [B][K] bf16 (the previous FC layer's output), W [C][K] bf16.
// Writes logits [B][C] fp32, meter / loss_out as cross_entropy_fused, optional dlogits (bf16, ld ldd);
// with dW != nullptr also dW [C][K] (fp32, stored; added to with `accumulate`), db [C] (fp32, accumulated) and
// dh [B][K] = (h > 0 or !relu) * drop_scale * dlogits W  (bf16: the previous layer's dz).
bool head_ce_supported(int B, int C, int K);
void head_ce_fused(const bf16* h, const bf16* W, const float* bias, const long long* target, float* logits,
                   bf16* dlogits, int ldd, float* dW, float* db, bf16* dh, float drop_scale, bool relu, float* meter,
                   float* loss_out, int B, int C, int K, const float* class_weights, bool accumulate,
                   cudaStream_t s, const SoftTargets* soft = nullptr);
// head_ce_fused with the distillation loss (see cross_entropy_kd): the dlogits it rounds to bf16 and feeds to the
// layer's backward are those of L.
void head_ce_kd_fused(const bf16* h, const bf16* W, const float* bias, const long long* target, float* logits,
                      bf16* dlogits, int ldd, float* dW, float* db, bf16* dh, float drop_scale, bool relu, float* meter,
                      float* loss_out, int B, int C, int K, const float* class_weights, bool accumulate,
                      const SoftTargets* soft, const float* teacher, const KdParams& kd, cudaStream_t s);

// Weight decay of one optimizer launch, per segment of its range: segment k covers the float4s
// [start4[k], start4[k + 1]) (the last one runs to the end of the range) and takes value[k].  start4[0]
// = 0 and the starts increase; a uniform decay is one segment.  value is the L2 decay wd (Adam, SGD) or,
// for AdamW, keep = fp32(1 - lr * wd) with the product taken in double.  Passed by value
// (__grid_constant__), so a bucket whose tensors decay differently (biases) still takes one launch.
constexpr int WD_MAX_SEGMENTS = 16;
struct WdSegments {
  int n;
  long long start4[WD_MAX_SEGMENTS];
  float value[WD_MAX_SEGMENTS];
};

// One update of the weights' exponential moving average (ema_update in adam.cuh): d = fp32(decay) and
// a = fp32(1 - decay) with 1 - decay taken in double; `first`: AveragedModel's first update, ema = p.
struct EmaCoef {
  float d, a;
  int first;
};
EmaCoef ema_coef(double decay, bool first);

// The scalars of one optimizer launch, in the form the kernels consume.  Built by make_opt_step only.
// The field order matters to the kernels' register allocation: in some orders nvcc loads neighbouring
// fields as pairs, which costs adam_kernel spills at its 40-register cap.
enum OptKind : int { OPT_ADAM = 0, OPT_ADAMW = 1, OPT_SGD = 2, OPT_LAMB = 3, OPT_LARS = 4 };
struct OptStep {
  float lr, beta1, beta2, eps;   // beta1, beta2, eps: Adam / AdamW
  float bc1_inv, bc2_inv_sqrt;   // 1 / (1 - beta1^step), 1 / sqrt(1 - beta2^step): double, rounded once
  float grad_scale;
  float momentum;                // SGD
  OptKind kind;
  int first;                     // SGD's first step: the momentum buffer starts as the gradient
  EmaCoef ema;                   // used by the launches that are given an `ema` arena
  WdSegments wd;                 // L2 decays (Adam, SGD) or AdamW keep factors
};
// Validates the weight-decay table and refuses a bad one naming `op`.  Without `wd_starts` the decay is
// `wd` everywhere; otherwise segment k covers elements [wd_starts[k], wd_starts[k + 1]) of the n-element
// range with decay wd_values[k] (and `wd` is not used).  Starts must begin at 0, increase, be multiples of
// 4 and lie inside the range; decays must be finite and >= 0.  AdamW's keep factors 1 - lr * wd are
// taken in double, as torch computes the Python scalar.
OptStep make_opt_step(const char* op, OptKind kind, long long n, double lr, double beta1, double beta2, double eps,
                      double momentum, int step, bool first, double grad_scale, double wd,
                      const std::vector<int64_t>& wd_starts, const std::vector<double>& wd_values, double ema_decay,
                      bool ema_first);

// Fused optimizer over flat arenas of n elements (n % 4 == 0): reads grad (fp32 g32, local, or bf16 g16,
// the reduced wire), updates the fp32 master p and the state (Adam: moments m and v; SGD: momentum
// buffer m, v null), writes the bf16 shadow and clears gzero when given.  With `ema`, the same pass
// also updates the weights' moving average from the new p.
void optimizer_fused(const OptStep& o, float* p, float* m, float* v, const float* g32, const bf16* g16,
                     bf16* shadow, float* gzero, float* ema, long long n, cudaStream_t s);
// The EMA update of the optimizers alone, for weights no optimizer launch covers (frozen layers):
// ema[i] = decay * ema[i] + (1 - decay) * p[i] with each operation rounded to fp32, or p[i] when `first`.
// n elements, any n >= 0; p and ema 16-byte aligned.
void ema_fused(const float* p, float* ema, long long n, double decay, bool first, cudaStream_t s);

// ---- layer-wise adaptive optimizers: LAMB and LARS (loss_optim.cu) -----------------------------
// The trust ratio of a tensor needs norms over the whole tensor, which the gradient buckets cut apart, so
// each step of these optimizers takes two passes.  Phase 1 runs per bucket once its gradient is final
// (LAMB: moments, and the partial sums of p^2 and u^2; LARS: the partial sums of p^2 and (g gscale)^2) and
// stores one pair of partial sums per CTA at a slot the host assigned.  Phase 2 runs once per group of
// tensors whose last piece that bucket held: it adds each tensor's partials in a fixed order, forms the
// ratio and applies the update, the bf16 shadow, the EMA and (LARS) the gradient zeroing.  No atomics:
// a ratio is the same bits on every run and every rank.
//
// One launch covers a range of n4 float4s cut into segments, segment k being float4s [start4[k],
// start4[k + 1]) of one tensor and CTAs [cta0[k], cta0[k + 1]).  Phase 1: the segment's CTA j stores its
// partials at ws[2 (slot[k] + j)], ws[2 (slot[k] + j) + 1].  Phase 2: the tensor's partials are slots
// [slot[k], slot[k] + nslots[k]); its ratio goes to ratio[tensor[k]] when `ratio` is given.
constexpr int LW_MAX_SEGMENTS = 16;
struct LayerwiseLaunch {
  int n;                                   // segments
  int cta0[LW_MAX_SEGMENTS + 1];           // cta0[0] = 0, increasing; cta0[n] = the grid
  long long start4[LW_MAX_SEGMENTS + 1];   // start4[0] = 0, increasing; start4[n] = the range's float4s
  int slot[LW_MAX_SEGMENTS];
  int nslots[LW_MAX_SEGMENTS];             // phase 2
  int tensor[LW_MAX_SEGMENTS];             // phase 2
  float wd[LW_MAX_SEGMENTS];               // the tensor's decay; 0 leaves it unadapted (ratio 1)
  float trust_coeff, trust_eps;            // LARS: ratio = coeff |p| / (|g| + wd |p| + eps)
};
// Validates the table (naming `op`) and fills a LayerwiseLaunch: starts in elements of the range
// (multiples of 4, the first 0, increasing, inside n), CTAs per segment >= 1 and at most `max_grid` in all.
LayerwiseLaunch make_layerwise_launch(const char* op, long long n, const std::vector<int64_t>& starts,
                                      const std::vector<int64_t>& ctas, const std::vector<int64_t>& slots,
                                      const std::vector<int64_t>& nslots, const std::vector<int64_t>& tensors,
                                      const std::vector<double>& wds, double trust_coeff, double trust_eps,
                                      long long max_grid);
// CTAs a layer-wise launch may use in all: the optimizer launches' cap, 4 per SM.
long long layerwise_max_grid();
// o.kind OPT_LAMB (m, v: the moments) or OPT_LARS (m: the momentum buffer, v unused).  Exactly one of g32
// and g16.  Phase 1 of LAMB clears gzero when given; phase 1 of LARS only reads.
void layerwise_phase1(const OptStep& o, const LayerwiseLaunch& L, float* p, float* m, float* v, const float* g32,
                      const bf16* g16, float* gzero, float* ws, cudaStream_t s);
// LAMB reads no gradient (g32 = g16 = null); LARS reads it and clears gzero when given.
void layerwise_phase2(const OptStep& o, const LayerwiseLaunch& L, float* p, float* m, float* v, const float* g32,
                      const bf16* g16, bf16* shadow, float* gzero, float* ema, const float* ws, float* ratio,
                      cudaStream_t s);

// ---- PowerSGD gradient compression (powersgd.cu) ----------------------------------------------
// A compressed tensor is an n x m row-major fp32 matrix (m % 4 == 0); P is [n][rank], Q is [m][rank],
// 1 <= rank <= PSGD_MAX_RANK; every operand 16-byte aligned.
constexpr int PSGD_MAX_RANK = 8;
// e = g * scale + e (M, stored over e); p = M q.
void psgd_project(const float* g, float* e, const float* q, float* p, int n, int m, int rank, float scale,
                  cudaStream_t s);
// q = M^T p, from per-row-split partial sums in ws[splits][workspace_slice(m * rank)] added in split order.
void psgd_backproject(const float* M, const float* p, float* q, float* ws, long long ws_elems, int n, int m, int rank,
                      cudaStream_t s);
int psgd_backproject_splits(int n, int m, int sms);
long long psgd_workspace_elems(int n, int m, int rank, int sms);
// Modified Gram-Schmidt of `count` consecutive [rows][rank] matrices, one per CTA; zero columns stay zero.
void psgd_orthogonalize(float* x, int rows, int count, int rank, cudaStream_t s);
// g = alpha * p q^T, e = e - g (e held M).
void psgd_decompress(const float* p, const float* q, float* g, float* e, int n, int m, int rank, float alpha,
                     cudaStream_t s);

// Fused input transform: uint8 HWC source -> normalised bf16.  mode 0: NHWC with C padded to
// `cpad`; mode 1: layer-0 im2col matrix [N*OH*OW][kpad] (k = (kh*3+kw)*3 + c, zero padded).
void augment_fused(const uint8_t* src, const float* params, bf16* out, int N, int SH, int SW,
                   int RH, int RW, int OH, int OW, int mode, int pad, const float* mean,
                   const float* stdv, cudaStream_t s);
// MixUp / CutMix of one batch (data/transforms.py::MixDraw).  Sample n's partner is n - 1 mod N.
// MixUp: lam * x_n + lam_b * x_partner in fp32 (lam_b = 1 - lam, rounded once on the host).  CutMix:
// output pixels with x1 <= ox < x2 and y1 <= oy < y2 are the partner's.
enum MixKind { MixNone = 0, MixMixUp = 1, MixCutMix = 2 };
struct MixParams {
  int kind;
  float lam, lam_b;
  int x1, y1, x2, y2;
};
// augment_fused mode 0 (NHWC, C padded to `pad`) with the batch mixed as `mix` says.
void augment_mixed(const uint8_t* src, const float* params, bf16* out, int N, int SH, int SW, int RH, int RW,
                   int OH, int OW, int pad, const float* mean, const float* stdv, const MixParams& mix,
                   cudaStream_t s);
// The same transform for a batch of images of any sizes, resampled exactly as Pillow's BILINEAR
// resize does.  src: the images back to back; geom [N][5] int64 rows (byte offset, H, W, RH, RW);
// params [N][8] as for augment_fused; inter: uint8 scratch of at least ragged_inter_bytes; out:
// NHWC bf16 with 4 channels (the 4th written as 0).  grid_x: blocks per image of each launch.
// Pass 1 filters the crop box horizontally into inter; pass 2 filters vertically, follows the
// rotation / flip / centre-crop chain and normalises (and mixes the batch when `mix` says so).
void augment_ragged(const uint8_t* src, const long long* geom, const float* params, uint8_t* inter,
                    bf16* out, int N, int OH, int OW, int grid_x, const float* mean,
                    const float* stdv, cudaStream_t s, const MixParams* mix = nullptr);
// ---- test-time augmentation views (--val-tta) --------------------------------------------------
// A view is an OH x OW crop of the RH x RW resized image: its position (torchvision's five_crop order, then the
// centre crop's mirror image), or'ed with TtaFlip to take the crop from the image's horizontal mirror.
enum TtaPosition { TtaTopLeft = 0, TtaTopRight = 1, TtaBottomLeft = 2, TtaBottomRight = 3, TtaCentre = 4,
                   TtaCentreMirror = 5 };
constexpr int TtaFlip = 8;
constexpr int kTtaMaxViews = 10;
struct TtaViews {                 // view v's code in bits [4v, 4v + 4)
  unsigned long long codes;
  int n;
};
// augment_fused mode 0 (NHWC4) for one view; the view's flip is combined with each sample's flip bit.
void augment_view(const uint8_t* src, const float* params, bf16* out, int N, int SH, int SW, int RH, int RW, int OH,
                  int OW, int view, const float* mean, const float* stdv, cudaStream_t s);
// augment_ragged for one view: with `pass1`, first pass 1 over the union of the columns and rows those views read
// (the batch's other views then run pass 2 alone on the same inter); then pass 2 at `view`.
void augment_ragged_view(const uint8_t* src, const long long* geom, const float* params, uint8_t* inter, bf16* out,
                         int N, int OH, int OW, int grid_x, const float* mean, const float* stdv, int view,
                         const TtaViews* pass1, cudaStream_t s);
// The view-mean reduction of one view's fp32 logits [B][C] into acc [B][C]: acc = softmax at
// view 0, acc += softmax at the later ones.  At view V - 1 it adds the batch's -log(acc[y] / V) sum, the count
// of argmax(acc / V) == y (lowest index on ties) and B into meter, and writes the mean loss to loss_out.
void tta_accumulate(const float* logits, const long long* target, float* acc, float* meter,
                    float* loss_out, int B, int C, int view, int views, cudaStream_t s);
// ---- per-class evaluation counts (--val-metrics) -------------------------------------------------
// For each row of the fp32 scores [B][C] divided by `views` (logits: 1; tta_accumulate's acc: V), add 1 to
// confusion[y][first maximum] (int64 [C][C], rows labels) and, when the label ranks among the first five
// (#{c : s_c > s_y} + #{c < y : s_c == s_y} < 5), 1 to *top5.  Integer atomics only.
void class_metrics(const float* scores, const long long* target, long long* confusion, long long* top5, int B, int C,
                   int views, cudaStream_t s);
// ---- streaming JPEG decode (jpeg.cu, --pipeline stream) ------------------------------------------
// A batch of k images described by desc [k][kJpegDesc] (jpeg.h) and geom [k][5] rows as augment_ragged's:
// dequantise + IDCT the total_blocks coefficient blocks into planes (total_blocks x 64 bytes), then write each
// image's RGB at out + geom offset (raw members copied from raw).  grid_x: blocks per image of the second launch.
void jpeg_decode(const int16_t* coef, const int* quant, const int* desc, const long long* geom, const uint8_t* raw,
                 uint8_t* planes, uint8_t* out, int k, long long total_blocks, int grid_x, cudaStream_t s);

// im2col of an NHWC(3, padded to cpad) bf16 image for layer 0 (used when the input is given as a
// float tensor instead of uint8 + params).
void im2col3x3_c3(const bf16* x, bf16* out, int N, int H, int W, int cpad, int kpad,
                  cudaStream_t s);
void nchw_f32_to_nhwc_bf16(const float* x, bf16* y, int N, int C, int H, int W, int cpad,
                           cudaStream_t s);

// ---- cross-GPU (allreduce.cu) ------------------------------------------------------------------
constexpr int AR_MAX_WORLD = 16;   // ranks of one CommCtx (the signal pad has a word per source rank)
struct CommCtx {
  int rank, world;
  void* const* wire_ptrs;        // device array [world]: peers' wire buffers (bf16 or fp32)
  uint32_t* const* signal_ptrs;  // device array [world]: peers' signal pads
  void* wire_mc;                 // multicast alias of the wire buffer (NVLS) or nullptr
  uint32_t* signal_mc;           // multicast alias of the signal pad or nullptr
  unsigned long long timeout_ns; // wall-clock bound of every cross-GPU wait (B200_BARRIER_TIMEOUT_S)
};
enum AllreduceAlgo : int { AR_ONESHOT = 0, AR_TWOSHOT = 1, AR_NVLS = 2 };
// Fused gradient all-reduce of arena range [start, start+n):
//   pack:   wire[i] = bf16(grad_f32[i] * inv_world)            (skipped when grad_f32 == nullptr)
//   reduce: every rank ends with wire[i] = sum over ranks (fp32 accumulation, bf16 on the wire)
//   unpack: optional fp32 write-back of the averaged gradient into grad_out_f32.
// `slot` selects one of the signal-pad barrier groups; `epoch` is incremented by the caller.
void allreduce_fused(const CommCtx& ctx, const float* grad_f32, float* grad_out_f32,
                     long long start, long long n, float inv_world, int algo, bool wire_fp32,
                     int slot, uint32_t epoch, int max_ctas, cudaStream_t s);
// CTAs allreduce_fused / zero1_step use for a range of n elements (the cell decomposition follows).
int allreduce_grid(long long n, int world, int max_ctas, bool wire_fp32);
// EXPERIMENTAL: ZeRO-1 step of arena range [start, start+n) in one kernel -- reduce-scatter, Adam on
// the cells this rank owns, all-gather of the new bf16 weights into every rank's shadow (allreduce.cu).
// The update is optimizer_fused's at grad_scale 1: Adam or AdamW with one decay for the whole range.
// With `ema`, the owner also updates the moving average of its cells.
void zero1_step(const CommCtx& ctx, const OptStep& o, float* grad_f32, float* p, float* m, float* v, bf16* shadow,
                float* ema, long long start, long long n, float inv_world, int algo, int slot, uint32_t epoch,
                int max_ctas, cudaStream_t s);
// Parameter broadcast rank `root` -> all through the wire buffer (K-BCAST).
void broadcast_fused(const CommCtx& ctx, float* data_f32, long long n, int root, int slot,
                     uint32_t epoch, cudaStream_t s);
void device_barrier(const CommCtx& ctx, int slot, uint32_t epoch, cudaStream_t s);
// uint32 words of signal pad needed for `slots` barrier groups
int allreduce_signal_words(int slots);

}  // namespace b200
