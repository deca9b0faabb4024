// pybind11 surface of the native library: adapts torch tensors to the raw-pointer API of api.h.
// Every op runs on torch's current CUDA stream of the tensor's device.
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include "api.h"
#include "jpeg.h"

namespace py = pybind11;
using b200::bf16;

static cudaStream_t cur_stream() { return at::cuda::getCurrentCUDAStream().stream(); }

static const bf16* bfp(const at::Tensor& t) {
  TORCH_CHECK(t.is_cuda() && t.scalar_type() == at::kBFloat16, "expected a CUDA bf16 tensor");
  return reinterpret_cast<const bf16*>(t.data_ptr());
}
static bf16* bfp_mut(at::Tensor& t) { return const_cast<bf16*>(bfp(t)); }
static float* f32p(const at::Tensor& t) {
  TORCH_CHECK(t.is_cuda() && t.scalar_type() == at::kFloat, "expected a CUDA fp32 tensor");
  return reinterpret_cast<float*>(t.data_ptr());
}
static const bf16* bfp_opt(const c10::optional<at::Tensor>& t) { return t.has_value() ? bfp(*t) : nullptr; }
static float* f32p_opt(const c10::optional<at::Tensor>& t) { return t.has_value() ? f32p(*t) : nullptr; }
// The element-wise kernels move 16-byte (8 x bf16 / 4 x fp32) or 8-byte vectors: refuse a tensor they
// would read or write out of bounds or misaligned before anything is launched.
static void check_vec(const at::Tensor& t, at::ScalarType dt, int64_t align, const char* op, const char* name) {
  TORCH_CHECK(t.is_cuda() && t.scalar_type() == dt && t.is_contiguous(), op, ": ", name, " must be a contiguous CUDA ",
              dt == at::kFloat ? "fp32" : "bf16", " tensor");
  TORCH_CHECK(reinterpret_cast<uintptr_t>(t.data_ptr()) % align == 0, op, ": ", name, " must be ", align,
              "-byte aligned");
}
static void check_nhwc(const at::Tensor& t, int64_t N, int64_t H, int64_t W, int64_t C, const char* op, const char* name) {
  TORCH_CHECK(t.dim() == 4 && t.size(0) == N && t.size(1) == H && t.size(2) == W && t.size(3) == C, op, ": ", name,
              " must be [", N, ", ", H, ", ", W, ", ", C, "], got ", t.sizes());
}

// ------------------------------------------------------------------------------------- GEMM / conv
static void gemm(const at::Tensor& A, bool a_mn, const at::Tensor& B, bool b_mn, int64_t M, int64_t N,
                 int64_t K, at::Tensor out, int64_t ldo, int64_t epi, c10::optional<at::Tensor> bias,
                 double alpha, int64_t ksplit, int64_t bn) {
  c10::cuda::CUDAGuard g(A.device());
  TORCH_CHECK(A.dim() == 2 && B.dim() == 2 && A.stride(1) == 1 && B.stride(1) == 1, "gemm: 2-D row-major operands");
  TORCH_CHECK(epi >= 0 && epi <= 5, "gemm: unknown epilogue ", epi);
  TORCH_CHECK(M > 0 && N > 0 && K > 0, "gemm: M, N and K must be positive");
  // the tensor maps span the operand's own rows and columns: A is [M][K] or [K][M] (a_mn), B [N][K] or [K][N]
  TORCH_CHECK(A.size(0) >= (a_mn ? K : M) && A.size(1) >= (a_mn ? M : K), "gemm: A must be at least ",
              a_mn ? "[K, M]" : "[M, K]", ", got ", A.sizes());
  TORCH_CHECK(B.size(0) >= (b_mn ? K : N) && B.size(1) >= (b_mn ? N : K), "gemm: B must be at least ",
              b_mn ? "[K, N]" : "[N, K]", ", got ", B.sizes());
  // the epilogue writes rows x cols elements at row stride ldo: [M][N], or [N][M] for the transposed ones
  const bool bf_out = epi == 3 || epi == 5, t_out = epi == 2 || epi == 4;
  const int64_t rows = t_out ? N : M, cols = t_out ? M : N;
  TORCH_CHECK(out.is_cuda() && out.is_contiguous() && out.scalar_type() == (bf_out ? at::kBFloat16 : at::kFloat),
              "gemm: out must be a contiguous ", bf_out ? "bf16" : "fp32", " tensor for this epilogue");
  TORCH_CHECK(ldo >= cols && out.numel() >= (rows - 1) * ldo + cols, "gemm: out must hold ", rows, " rows of ",
              cols, " elements at ldo = ", ldo, ", got ", out.numel(), " elements");
  TORCH_CHECK(epi != 3 || bias.has_value(), "gemm: the bias + ReLU epilogue needs a bias");
  TORCH_CHECK(!bias.has_value() || bias->numel() >= N, "gemm: bias must have N = ", N, " elements");
  b200::gemm_bf16(bfp(A), A.stride(0), a_mn, bfp(B), B.stride(0), b_mn, (int)M, (int)N, (int)K, out.data_ptr(),
                  ldo, (int)epi, f32p_opt(bias), (float)alpha, (int)ksplit, (int)bn, cur_stream());
}

static void conv_fprop(const at::Tensor& x, const at::Tensor& w, c10::optional<at::Tensor> bias, at::Tensor y,
                       bool relu, int64_t bn) {
  c10::cuda::CUDAGuard g(x.device());
  TORCH_CHECK(x.dim() == 4 && x.is_contiguous() && w.is_contiguous() && y.is_contiguous(), "conv_fprop: contiguous NHWC");
  const int N = x.size(0), H = x.size(1), W = x.size(2), Cin = x.size(3), Cout = w.size(0);
  TORCH_CHECK(w.numel() == (int64_t)Cout * 9 * Cin && y.numel() == (int64_t)N * H * W * Cout, "conv_fprop: shape mismatch");
  TORCH_CHECK(!bias.has_value() || bias->numel() >= Cout, "conv_fprop: bias must have Cout = ", Cout, " elements");
  b200::conv3x3_fprop(bfp(x), bfp(w), f32p_opt(bias), bfp_mut(y), N, H, W, Cin, Cout, relu, (int)bn, cur_stream());
}
// Fused conv + pool (default; B200_FUSE_POOL=0 turns it off): pooled activation + int32 mask words [N,H/2,W/2,Cout/32,4]
static void conv_fprop_pool(const at::Tensor& x, const at::Tensor& w, c10::optional<at::Tensor> bias,
                            at::Tensor pooled, at::Tensor mask, int64_t bn) {
  c10::cuda::CUDAGuard g(x.device());
  TORCH_CHECK(x.dim() == 4 && x.is_contiguous() && w.is_contiguous() && pooled.is_contiguous() && mask.is_contiguous(),
              "conv_fprop_pool: contiguous NHWC");
  const int N = x.size(0), H = x.size(1), W = x.size(2), Cin = x.size(3), Cout = w.size(0);
  TORCH_CHECK(w.numel() == (int64_t)Cout * 9 * Cin && pooled.numel() == (int64_t)N * (H / 2) * (W / 2) * Cout &&
                  pooled.scalar_type() == at::kBFloat16,
              "conv_fprop_pool: shape mismatch");
  TORCH_CHECK(mask.scalar_type() == at::kInt && mask.numel() == (int64_t)N * (H / 2) * (W / 2) * (Cout / 32) * 4,
              "conv_fprop_pool: mask must be int32 [N,H/2,W/2,Cout/32,4]");
  TORCH_CHECK(!bias.has_value() || bias->numel() >= Cout, "conv_fprop_pool: bias must have Cout = ", Cout, " elements");
  b200::conv3x3_fprop_pool(bfp(x), bfp(w), f32p_opt(bias), bfp_mut(pooled),
                           reinterpret_cast<uint32_t*>(mask.data_ptr<int>()), N, H, W, Cin, Cout, (int)bn, cur_stream());
}
static bool conv_pool_fusable(int64_t N, int64_t H, int64_t W) { return b200::conv3x3_pool_fusable((int)N, (int)H, (int)W); }
static std::vector<int64_t> conv_pixel_box(int64_t N, int64_t H, int64_t W) {
  int b[4];
  b200::conv_pixel_box((int)N, (int)H, (int)W, b);
  return {b[0], b[1], b[2], b[3]};
}
static int64_t conv_bn_choice(int64_t N, int64_t H, int64_t W, int64_t cn) {
  return b200::conv_bn_choice((int)N, (int)H, (int)W, (int)cn);
}
// conv_plan(kind, N, H, W, Cin, Cout, sms, bn=0): what a conv launch runs (pure host code, no GPU needed);
// bn: the tile width a caller passes to the launcher (0: the launcher's own choice).
static py::dict conv_plan(const std::string& kind, int64_t N, int64_t H, int64_t W, int64_t Cin, int64_t Cout,
                          int64_t sms, int64_t bn) {
  static const char* kinds[] = {"fprop", "fprop_pool", "dgrad", "wgrad", "wgrad_partial"};
  static const char* paths[] = {"halo", "pow2", "fill", "wgrad_halo64", "wgrad"};
  int k = -1;
  for (int i = 0; i < 5; ++i)
    if (kind == kinds[i]) k = i;
  TORCH_CHECK(k >= 0, "conv_plan: kind must be fprop, fprop_pool, dgrad, wgrad or wgrad_partial, got ", kind);
  const b200::ConvPlan p = b200::conv_plan(k, (int)N, (int)H, (int)W, (int)Cin, (int)Cout, (int)sms, (int)bn);
  py::dict d;
  d["path"] = paths[p.path];
  d["bn"] = p.bn;
  d["box"] = py::make_tuple(p.Wb, p.Hb, p.Nb);
  d["tiles"] = p.tiles;
  d["ksplit"] = p.ksplit;
  d["tiles_per_split"] = p.tiles_per_split;
  d["resident"] = bool(p.resident);
  return d;
}
static void unpool(const at::Tensor& dp, const at::Tensor& mask, at::Tensor dz, c10::optional<at::Tensor> colsum) {
  c10::cuda::CUDAGuard g(dp.device());
  TORCH_CHECK(dp.dim() == 4 && dz.dim() == 4 && dp.is_contiguous() && dz.is_contiguous() && mask.is_contiguous() &&
                  mask.scalar_type() == at::kInt,
              "unpool2x2: contiguous NHWC bf16 + int32 mask");
  const int N = dz.size(0), H = dz.size(1), W = dz.size(2), C = dz.size(3);
  TORCH_CHECK(dp.size(0) == N && dp.size(1) == H / 2 && dp.size(2) == W / 2 && dp.size(3) == C &&
                  mask.numel() == (int64_t)N * (H / 2) * (W / 2) * (C / 32) * 4,
              "unpool2x2: shape mismatch");
  b200::unpool2x2(bfp(dp), reinterpret_cast<const uint32_t*>(mask.data_ptr<int>()), bfp_mut(dz), f32p_opt(colsum), N, H,
                  W, C, cur_stream());
}

static void conv_dgrad(const at::Tensor& dz, const at::Tensor& w, c10::optional<at::Tensor> mask, at::Tensor dx,
                       c10::optional<at::Tensor> colsum, int64_t bn) {
  c10::cuda::CUDAGuard g(dz.device());
  TORCH_CHECK(dz.dim() == 4 && dz.is_contiguous() && w.is_contiguous() && dx.is_contiguous(), "conv_dgrad: contiguous NHWC");
  const int N = dz.size(0), H = dz.size(1), W = dz.size(2), Cout = dz.size(3), Cin = dx.size(3);
  TORCH_CHECK(w.numel() == (int64_t)Cout * 9 * Cin, "conv_dgrad: weight shape mismatch");
  check_nhwc(dx, N, H, W, Cin, "conv_dgrad", "dx");
  if (mask.has_value()) {
    TORCH_CHECK(mask->is_contiguous(), "conv_dgrad: mask_src must be contiguous");
    check_nhwc(*mask, N, H, W, Cin, "conv_dgrad", "mask_src");
  }
  TORCH_CHECK(!colsum.has_value() || colsum->numel() >= Cin, "conv_dgrad: colsum must have Cin = ", Cin, " elements");
  b200::conv3x3_dgrad(bfp(dz), bfp(w), bfp_opt(mask), bfp_mut(dx), f32p_opt(colsum), N, H, W, Cin, Cout, (int)bn, cur_stream());
}
static void conv_wgrad(const at::Tensor& dz, const at::Tensor& x, at::Tensor dw, double scale, int64_t ksplit,
                       int64_t bn) {
  c10::cuda::CUDAGuard g(dz.device());
  TORCH_CHECK(dz.dim() == 4 && dz.is_contiguous() && x.is_contiguous(), "conv_wgrad: contiguous NHWC");
  const int N = dz.size(0), H = dz.size(1), W = dz.size(2), Cout = dz.size(3), Cin = x.size(3);
  TORCH_CHECK(dw.numel() == (int64_t)Cout * 9 * Cin && dw.is_contiguous(), "conv_wgrad: dw shape mismatch");
  check_nhwc(x, N, H, W, Cin, "conv_wgrad", "x");
  b200::conv3x3_wgrad(bfp(dz), bfp(x), f32p(dw), N, H, W, Cin, Cout, (float)scale, (int)ksplit, (int)bn, cur_stream());
}

static void conv0_fprop(const at::Tensor& x4, const at::Tensor& w0, const at::Tensor& bias, at::Tensor y) {
  c10::cuda::CUDAGuard g(x4.device());
  TORCH_CHECK(x4.dim() == 4 && x4.size(3) == 4 && x4.is_contiguous() && w0.numel() == 64 * 64 && y.is_contiguous(),
              "conv0_fprop: x4 [N,H,W,4], w0 [64,64]");
  TORCH_CHECK(w0.is_contiguous(), "conv0_fprop: w0 must be contiguous");
  check_nhwc(y, x4.size(0), x4.size(1), x4.size(2), 64, "conv0_fprop", "y");
  TORCH_CHECK(bias.numel() >= 64, "conv0_fprop: bias must have 64 elements");
  b200::conv0_fprop(bfp(x4), bfp(w0), f32p(bias), bfp_mut(y), x4.size(0), x4.size(1), x4.size(2), cur_stream());
}
static void conv0_wgrad(const at::Tensor& dz, const at::Tensor& x4, at::Tensor dw0) {
  c10::cuda::CUDAGuard g(x4.device());
  TORCH_CHECK(x4.dim() == 4 && x4.size(3) == 4 && x4.is_contiguous() && dz.is_contiguous() && dw0.numel() == 64 * 64,
              "conv0_wgrad: x4 [N,H,W,4], dw0 [64,64]");
  TORCH_CHECK(dw0.is_contiguous(), "conv0_wgrad: dw0 must be contiguous");
  check_nhwc(dz, x4.size(0), x4.size(1), x4.size(2), 64, "conv0_wgrad", "dz");
  b200::conv0_wgrad(bfp(dz), bfp(x4), f32p(dw0), x4.size(0), x4.size(1), x4.size(2), cur_stream());
}

// ------------------------------------------------------------- split-K without atomics (api.h)
static void check_workspace_tensor(const at::Tensor& ws, const char* op) {
  check_vec(ws, at::kFloat, 16, op, "the workspace");
}
static int64_t gemm_partial(const at::Tensor& A, bool a_mn, const at::Tensor& B, bool b_mn, int64_t M, int64_t N,
                            int64_t K, at::Tensor ws, int64_t ldo, bool transposed, double alpha, int64_t ksplit,
                            int64_t bn) {
  c10::cuda::CUDAGuard g(A.device());
  TORCH_CHECK(A.dim() == 2 && B.dim() == 2 && A.stride(1) == 1 && B.stride(1) == 1, "gemm_partial: 2-D row-major operands");
  TORCH_CHECK(M > 0 && N > 0 && K > 0, "gemm_partial: M, N and K must be positive");
  TORCH_CHECK(A.size(0) >= (a_mn ? K : M) && A.size(1) >= (a_mn ? M : K), "gemm_partial: A must be at least ",
              a_mn ? "[K, M]" : "[M, K]", ", got ", A.sizes());
  TORCH_CHECK(B.size(0) >= (b_mn ? K : N) && B.size(1) >= (b_mn ? N : K), "gemm_partial: B must be at least ",
              b_mn ? "[K, N]" : "[N, K]", ", got ", B.sizes());
  // every element of a slice must be written: the reduction reads whole slices
  TORCH_CHECK(ldo == (transposed ? M : N), "gemm_partial: slices are dense, ldo must be ", transposed ? M : N);
  check_workspace_tensor(ws, "gemm_partial");
  return b200::gemm_bf16_partial(bfp(A), A.stride(0), a_mn, bfp(B), B.stride(0), b_mn, (int)M, (int)N, (int)K, f32p(ws),
                                 ws.numel(), ldo, transposed, (float)alpha, (int)ksplit, (int)bn, cur_stream());
}
static int64_t conv_wgrad_partial(const at::Tensor& dz, const at::Tensor& x, at::Tensor ws, double scale) {
  c10::cuda::CUDAGuard g(dz.device());
  TORCH_CHECK(dz.dim() == 4 && dz.is_contiguous() && x.is_contiguous(), "conv_wgrad_partial: contiguous NHWC");
  const int N = dz.size(0), H = dz.size(1), W = dz.size(2), Cout = dz.size(3), Cin = x.size(3);
  check_nhwc(x, N, H, W, Cin, "conv_wgrad_partial", "x");
  check_workspace_tensor(ws, "conv_wgrad_partial");
  return b200::conv3x3_wgrad_partial(bfp(dz), bfp(x), f32p(ws), ws.numel(), N, H, W, Cin, Cout, (float)scale, cur_stream());
}
static int64_t conv0_wgrad_partial(const at::Tensor& dz, const at::Tensor& x4, at::Tensor ws) {
  c10::cuda::CUDAGuard g(x4.device());
  TORCH_CHECK(x4.dim() == 4 && x4.size(3) == 4 && x4.is_contiguous() && dz.is_contiguous(),
              "conv0_wgrad_partial: x4 [N,H,W,4]");
  check_nhwc(dz, x4.size(0), x4.size(1), x4.size(2), 64, "conv0_wgrad_partial", "dz");
  check_workspace_tensor(ws, "conv0_wgrad_partial");
  return b200::conv0_wgrad_partial(bfp(dz), bfp(x4), f32p(ws), ws.numel(), x4.size(0), x4.size(1), x4.size(2), cur_stream());
}
static int64_t colsum_partial(const at::Tensor& dz, at::Tensor ws, int64_t rows, int64_t C, double scale) {
  c10::cuda::CUDAGuard g(dz.device());
  TORCH_CHECK(C > 0 && C % 8 == 0 && rows > 0 && dz.numel() >= rows * C, "colsum_partial: dz must hold rows x C, C % 8 == 0");
  check_vec(dz, at::kBFloat16, 16, "colsum_partial", "dz");
  check_workspace_tensor(ws, "colsum_partial");
  return b200::colsum_partial(bfp(dz), f32p(ws), ws.numel(), rows, (int)C, (float)scale, cur_stream());
}
static void splitk_reduce(const at::Tensor& ws, at::Tensor dst, int64_t n, int64_t slice, int64_t splits, double alpha,
                          bool accumulate) {
  c10::cuda::CUDAGuard g(ws.device());
  check_workspace_tensor(ws, "splitk_reduce");
  check_vec(dst, at::kFloat, 16, "splitk_reduce", "dst");
  TORCH_CHECK(dst.numel() >= n, "splitk_reduce: dst must hold n = ", n, " elements, got ", dst.numel());
  b200::splitk_reduce(f32p(ws), ws.numel(), f32p(dst), n, slice, (int)splits, (float)alpha, accumulate, cur_stream());
}

// ------------------------------------------------------------------------------------ element-wise
static void maxpool_fwd(const at::Tensor& x, at::Tensor y) {
  c10::cuda::CUDAGuard g(x.device());
  check_vec(x, at::kBFloat16, 16, "maxpool_fwd", "x");
  check_vec(y, at::kBFloat16, 16, "maxpool_fwd", "y");
  TORCH_CHECK(x.dim() == 4, "maxpool_fwd: x must be NHWC");
  check_nhwc(y, x.size(0), x.size(1) / 2, x.size(2) / 2, x.size(3), "maxpool_fwd", "y");
  b200::maxpool2x2_fwd(bfp(x), bfp_mut(y), x.size(0), x.size(1), x.size(2), x.size(3), cur_stream());
}
static void maxpool_relu_bwd(const at::Tensor& y, const at::Tensor& dp, at::Tensor dz,
                             c10::optional<at::Tensor> colsum) {
  c10::cuda::CUDAGuard g(y.device());
  check_vec(y, at::kBFloat16, 16, "maxpool_relu_bwd", "y");
  check_vec(dp, at::kBFloat16, 16, "maxpool_relu_bwd", "dp");
  check_vec(dz, at::kBFloat16, 16, "maxpool_relu_bwd", "dz");
  TORCH_CHECK(y.dim() == 4, "maxpool_relu_bwd: y must be NHWC");
  check_nhwc(dp, y.size(0), y.size(1) / 2, y.size(2) / 2, y.size(3), "maxpool_relu_bwd", "dp");
  check_nhwc(dz, y.size(0), y.size(1), y.size(2), y.size(3), "maxpool_relu_bwd", "dz");
  if (colsum.has_value())
    TORCH_CHECK(colsum->scalar_type() == at::kFloat && colsum->numel() >= y.size(3), "maxpool_relu_bwd: colsum fp32 [C]");
  b200::maxpool2x2_relu_bwd(bfp(y), bfp(dp), bfp_mut(dz), f32p_opt(colsum), y.size(0), y.size(1), y.size(2), y.size(3),
                            cur_stream());
}
static void avgpool_fwd(const at::Tensor& x, at::Tensor y) {
  c10::cuda::CUDAGuard g(x.device());
  check_vec(x, at::kBFloat16, 16, "avgpool_fwd", "x");
  check_vec(y, at::kBFloat16, 16, "avgpool_fwd", "y");
  TORCH_CHECK(x.dim() == 4 && y.dim() == 4, "avgpool_fwd: NHWC x and y");
  check_nhwc(y, x.size(0), y.size(1), y.size(2), x.size(3), "avgpool_fwd", "y");
  b200::adaptive_avgpool_fwd(bfp(x), bfp_mut(y), x.size(0), x.size(1), x.size(2), x.size(3), y.size(1), y.size(2), cur_stream());
}
static void avgpool_bwd(const at::Tensor& dy, at::Tensor dx) {
  c10::cuda::CUDAGuard g(dy.device());
  check_vec(dy, at::kBFloat16, 16, "avgpool_bwd", "dy");
  check_vec(dx, at::kBFloat16, 16, "avgpool_bwd", "dx");
  TORCH_CHECK(dy.dim() == 4 && dx.dim() == 4, "avgpool_bwd: NHWC dy and dx");
  check_nhwc(dy, dx.size(0), dy.size(1), dy.size(2), dx.size(3), "avgpool_bwd", "dy");
  b200::adaptive_avgpool_bwd(bfp(dy), bfp_mut(dx), dx.size(0), dx.size(1), dx.size(2), dx.size(3), dy.size(1), dy.size(2), cur_stream());
}
static void bias_grad(const at::Tensor& dz, at::Tensor db, int64_t rows, int64_t C, int64_t ld, double scale) {
  c10::cuda::CUDAGuard g(dz.device());
  TORCH_CHECK(dz.is_cuda() && dz.scalar_type() == at::kBFloat16 && dz.is_contiguous() && ld >= C && C > 0 &&
                  dz.numel() >= (rows - 1) * ld + C,
              "bias_grad: contiguous bf16 dz of at least rows x ld elements, ld >= C");
  TORCH_CHECK(db.scalar_type() == at::kFloat && db.numel() >= C, "bias_grad: db must be fp32 with C elements");
  if (C % 8 == 0 && ld == C) check_vec(dz, at::kBFloat16, 16, "bias_grad", "dz");
  if (C % 8 == 0 && ld == C) b200::bias_grad(bfp(dz), f32p(db), rows, (int)C, (float)scale, cur_stream());
  else b200::bias_grad_ld(bfp(dz), f32p(db), rows, (int)C, (int)ld, (float)scale, cur_stream());
}
static void fc_bias_act(at::Tensor acc, c10::optional<at::Tensor> bias, c10::optional<at::Tensor> y,
                        c10::optional<at::Tensor> y_f32, int64_t B, int64_t N, bool relu, double drop_p,
                        int64_t seed, int64_t offset, bool clear) {
  c10::cuda::CUDAGuard g(acc.device());
  TORCH_CHECK(acc.is_contiguous() && acc.numel() >= B * N, "fc_bias_act: contiguous acc of B x N");
  TORCH_CHECK(!bias.has_value() || bias->numel() >= N, "fc_bias_act: bias of N");
  TORCH_CHECK(!y.has_value() || (y->is_contiguous() && y->numel() >= B * N), "fc_bias_act: contiguous y of B x N");
  TORCH_CHECK(!y_f32.has_value() || (y_f32->is_contiguous() && y_f32->numel() >= B * N),
              "fc_bias_act: contiguous y_f32 of B x N");
  b200::fc_bias_act(f32p(acc), f32p_opt(bias), y.has_value() ? bfp_mut(*y) : nullptr, f32p_opt(y_f32), (int)B,
                    (int)N, relu, (float)drop_p, (unsigned long long)seed, (unsigned long long)offset, clear,
                    cur_stream());
}
static void fc_grad_act(at::Tensor acc, c10::optional<at::Tensor> act, at::Tensor dz, int64_t B, int64_t N,
                        bool relu, double drop_p, bool clear) {
  c10::cuda::CUDAGuard g(acc.device());
  // the dropout mask is read back from act > 0, which only a ReLU layer's output encodes
  TORCH_CHECK(relu || drop_p == 0.0, "fc_grad_act: dropout without ReLU is not supported");
  TORCH_CHECK(acc.is_contiguous() && acc.numel() >= B * N && dz.is_contiguous() && dz.numel() >= B * N,
              "fc_grad_act: contiguous acc and dz of B x N");
  TORCH_CHECK(!relu || (act.has_value() && act->is_contiguous() && act->numel() >= B * N),
              "fc_grad_act: relu needs a contiguous act of B x N");
  b200::fc_grad_act(f32p(acc), bfp_opt(act), bfp_mut(dz), (int)B, (int)N, relu, (float)drop_p, 0, 0, clear, cur_stream());
}
static void cast_to_bf16(const at::Tensor& x, at::Tensor y) {
  c10::cuda::CUDAGuard g(x.device());
  check_vec(x, at::kFloat, 16, "cast_to_bf16", "x");
  check_vec(y, at::kBFloat16, 8, "cast_to_bf16", "y");
  TORCH_CHECK(y.numel() == x.numel(), "cast_to_bf16: x and y differ in size");
  b200::cast_f32_to_bf16(f32p(x), bfp_mut(y), x.numel(), cur_stream());
}
static void cast_to_f32(const at::Tensor& x, at::Tensor y) {
  c10::cuda::CUDAGuard g(x.device());
  TORCH_CHECK(x.is_contiguous() && y.is_contiguous() && y.numel() == x.numel(), "cast_to_f32: contiguous, same size");
  b200::cast_bf16_to_f32(bfp(x), f32p(y), x.numel(), cur_stream());
}

static void check_cross_entropy(const at::Tensor& logits, const at::Tensor& target,
                                const c10::optional<at::Tensor>& dlogits, int64_t ldd,
                                const c10::optional<at::Tensor>& meter, const c10::optional<at::Tensor>& loss_out,
                                const c10::optional<at::Tensor>& class_weights) {
  TORCH_CHECK(target.scalar_type() == at::kLong && logits.is_contiguous(), "cross_entropy: int64 targets, contiguous logits");
  TORCH_CHECK(logits.dim() == 2, "cross_entropy: logits must be [B, C]");
  const int64_t B = logits.size(0), C = logits.size(1);
  TORCH_CHECK(target.is_contiguous() && target.numel() >= B, "cross_entropy: contiguous targets of B = ", B);
  if (dlogits.has_value())
    TORCH_CHECK(ldd >= C && dlogits->is_contiguous() && dlogits->numel() >= B * ldd,
                "cross_entropy: dlogits must be contiguous, ldd >= C and at least B x ldd elements");
  TORCH_CHECK(!meter.has_value() || meter->numel() >= 3, "cross_entropy: meter must have 3 elements");
  TORCH_CHECK(!loss_out.has_value() || loss_out->numel() >= 1, "cross_entropy: loss_out must have 1 element");
  TORCH_CHECK(!class_weights.has_value() || class_weights->numel() >= C, "cross_entropy: class_weights of C = ", C);
}

// Soft targets (label smoothing eps; with `mix`, row r's target also takes lam_b of row r-1's label):
// the host values are checked here so that a bad draw cannot reach the kernels.
static b200::SoftTargets soft_targets(const char* what, double eps, double lam, bool mix) {
  TORCH_CHECK(eps >= 0.0 && eps < 1.0, what, ": label smoothing must lie in [0, 1), got ", eps);
  TORCH_CHECK(!mix || (lam >= 0.0 && lam <= 1.0), what, ": the mixing weight must lie in [0, 1], got ", lam);
  return b200::SoftTargets{(float)eps, mix ? (float)lam : 1.f, mix ? (float)(1.0 - lam) : 0.f, mix ? 1 : 0};
}

static void cross_entropy(const at::Tensor& logits, const at::Tensor& target, c10::optional<at::Tensor> dlogits,
                          int64_t ldd, c10::optional<at::Tensor> meter, c10::optional<at::Tensor> loss_out,
                          double grad_scale, c10::optional<at::Tensor> class_weights) {
  c10::cuda::CUDAGuard g(logits.device());
  check_cross_entropy(logits, target, dlogits, ldd, meter, loss_out, class_weights);
  b200::cross_entropy_fused(f32p(logits), reinterpret_cast<const long long*>(target.data_ptr()),
                            dlogits.has_value() ? bfp_mut(*dlogits) : nullptr, (int)ldd, f32p_opt(meter),
                            f32p_opt(loss_out), (int)logits.size(0), (int)logits.size(1), (float)grad_scale,
                            f32p_opt(class_weights), cur_stream());
}

static void cross_entropy_soft(const at::Tensor& logits, const at::Tensor& target, c10::optional<at::Tensor> dlogits,
                               int64_t ldd, c10::optional<at::Tensor> meter, c10::optional<at::Tensor> loss_out,
                               double grad_scale, c10::optional<at::Tensor> class_weights, double eps, double lam,
                               bool mix) {
  c10::cuda::CUDAGuard g(logits.device());
  check_cross_entropy(logits, target, dlogits, ldd, meter, loss_out, class_weights);
  const b200::SoftTargets st = soft_targets("cross_entropy_soft", eps, lam, mix);
  b200::cross_entropy_soft(f32p(logits), reinterpret_cast<const long long*>(target.data_ptr()),
                           dlogits.has_value() ? bfp_mut(*dlogits) : nullptr, (int)ldd, f32p_opt(meter),
                           f32p_opt(loss_out), (int)logits.size(0), (int)logits.size(1), (float)grad_scale,
                           f32p_opt(class_weights), st, cur_stream());
}

static void check_head_ce(const char* what, const at::Tensor& h, const at::Tensor& W, const at::Tensor& bias,
                          const at::Tensor& target, const at::Tensor& logits, const c10::optional<at::Tensor>& dlogits,
                          int64_t ldd, const c10::optional<at::Tensor>& dW, const c10::optional<at::Tensor>& db,
                          const c10::optional<at::Tensor>& dh, double drop_scale, bool relu,
                          const c10::optional<at::Tensor>& meter, const c10::optional<at::Tensor>& loss_out,
                          const c10::optional<at::Tensor>& class_weights) {
  TORCH_CHECK(h.dim() == 2 && W.dim() == 2 && h.size(1) == W.size(1) && h.is_contiguous() && W.is_contiguous(),
              what, ": h [B][K], W [C][K], contiguous");
  TORCH_CHECK(target.scalar_type() == at::kLong && logits.is_contiguous() && logits.size(0) == h.size(0) &&
              logits.size(1) == W.size(0), what, ": int64 targets, logits [B][C]");
  TORCH_CHECK(dW.has_value() == db.has_value(), what, ": dW and db come together");
  // dh keeps only the elements with h > 0: that is the dropout mask only after a ReLU
  TORCH_CHECK(relu || drop_scale == 1.0, what, ": dropout without ReLU is not supported");
  const int64_t B = h.size(0), C = W.size(0), K = h.size(1);
  TORCH_CHECK(target.is_contiguous() && target.numel() >= B, what, ": contiguous targets of B = ", B);
  TORCH_CHECK(bias.numel() >= C, what, ": bias must have C = ", C, " elements");
  if (dlogits.has_value())
    TORCH_CHECK(ldd >= C && dlogits->is_contiguous() && dlogits->numel() >= B * ldd,
                what, ": dlogits must be contiguous, ldd >= C and at least B x ldd elements");
  TORCH_CHECK(!dW.has_value() || (dW->is_contiguous() && dW->numel() >= C * K), what, ": contiguous dW of C x K");
  TORCH_CHECK(!db.has_value() || db->numel() >= C, what, ": db must have C elements");
  TORCH_CHECK(!dh.has_value() || (dh->is_contiguous() && dh->numel() >= B * K), what, ": contiguous dh of B x K");
  TORCH_CHECK(!meter.has_value() || meter->numel() >= 3, what, ": meter must have 3 elements");
  TORCH_CHECK(!loss_out.has_value() || loss_out->numel() >= 1, what, ": loss_out must have 1 element");
  TORCH_CHECK(!class_weights.has_value() || class_weights->numel() >= C, what, ": class_weights of C = ", C);
}

// Distillation operands: teacher logits fp32 [B][C], contiguous, on the logits' device; 0 < alpha <= 1; T finite > 0.
static b200::KdParams check_kd(const char* what, const at::Tensor& teacher, const at::Device& dev, int64_t B, int64_t C,
                               double alpha, double temperature) {
  TORCH_CHECK(teacher.device() == dev, what, ": teacher logits must be on ", dev, ", got ", teacher.device());
  TORCH_CHECK(teacher.scalar_type() == at::kFloat && teacher.is_contiguous() && teacher.dim() == 2 &&
              teacher.size(0) == B && teacher.size(1) == C,
              what, ": teacher logits must be contiguous fp32 [", B, "][", C, "], got ", teacher.scalar_type(), " ",
              teacher.sizes());
  TORCH_CHECK(alpha > 0.0 && alpha <= 1.0, what, ": alpha must lie in (0, 1], got ", alpha);
  TORCH_CHECK(std::isfinite(temperature) && temperature > 0.0, what, ": temperature must be finite and > 0, got ",
              temperature);
  return b200::kd_params(alpha, temperature, (int)B);
}

static b200::SoftTargets soft_list(const char* what, const c10::optional<std::vector<double>>& soft) {
  TORCH_CHECK(!soft.has_value() || soft->size() == 3, what, ": soft is (eps, lam, mix)");
  return soft.has_value() ? soft_targets(what, (*soft)[0], (*soft)[1], (*soft)[2] != 0.0) : b200::SoftTargets{};
}

// cross_entropy / cross_entropy_soft with the distillation loss; soft = (eps, lam, mix) or None (integer labels)
static void cross_entropy_kd(const at::Tensor& logits, const at::Tensor& target, c10::optional<at::Tensor> dlogits,
                             int64_t ldd, c10::optional<at::Tensor> meter, c10::optional<at::Tensor> loss_out,
                             double grad_scale, c10::optional<at::Tensor> class_weights, const at::Tensor& teacher,
                             double alpha, double temperature, c10::optional<std::vector<double>> soft) {
  c10::cuda::CUDAGuard g(logits.device());
  check_cross_entropy(logits, target, dlogits, ldd, meter, loss_out, class_weights);
  TORCH_CHECK(logits.scalar_type() == at::kFloat, "cross_entropy_kd: fp32 logits");
  const b200::KdParams kd = check_kd("cross_entropy_kd", teacher, logits.device(), logits.size(0), logits.size(1),
                                     alpha, temperature);
  const b200::SoftTargets st = soft_list("cross_entropy_kd", soft);
  b200::cross_entropy_kd(f32p(logits), reinterpret_cast<const long long*>(target.data_ptr()),
                         dlogits.has_value() ? bfp_mut(*dlogits) : nullptr, (int)ldd, f32p_opt(meter),
                         f32p_opt(loss_out), (int)logits.size(0), (int)logits.size(1), (float)grad_scale,
                         f32p_opt(class_weights), soft.has_value() ? &st : nullptr, f32p(teacher), kd, cur_stream());
}

// The optimizers' optional moving average of the weights: fp32, 16-byte aligned, p's size, decay in [0, 1].
static void check_ema(const c10::optional<at::Tensor>& ema, int64_t n, double decay, const char* op) {
  if (!ema.has_value()) return;
  check_vec(*ema, at::kFloat, 16, op, "ema");
  TORCH_CHECK(ema->numel() == n, op, ": ema must have p's size");
  TORCH_CHECK(decay >= 0.0 && decay <= 1.0, op, ": ema_decay must lie in [0, 1], got ", decay);
}
// The operands of one adam / sgd launch over p's n elements: the fp32 state (p first), exactly one of the
// fp32 and bf16 gradients, and the optional shadow, gradient range to clear and moving average.
static void check_optimizer(const char* op, const char* state_names, std::initializer_list<const at::Tensor*> state,
                            const c10::optional<at::Tensor>& g32, const c10::optional<at::Tensor>& g16,
                            const c10::optional<at::Tensor>& shadow, const c10::optional<at::Tensor>& gzero,
                            const c10::optional<at::Tensor>& ema, double ema_decay) {
  const int64_t n = (*state.begin())->numel();
  for (const at::Tensor* t : state) check_vec(*t, at::kFloat, 16, op, state_names);
  check_ema(ema, n, ema_decay, op);
  if (g32.has_value()) check_vec(*g32, at::kFloat, 16, op, "g32");
  if (gzero.has_value()) check_vec(*gzero, at::kFloat, 16, op, "gzero");
  if (g16.has_value()) check_vec(*g16, at::kBFloat16, 8, op, "g16");
  if (shadow.has_value()) check_vec(*shadow, at::kBFloat16, 8, op, "shadow");
  TORCH_CHECK(g32.has_value() != g16.has_value(), op, ": exactly one of g32 and g16");
  for (const auto* t : {&g32, &g16, &shadow, &gzero})
    TORCH_CHECK(!t->has_value() || (*t)->numel() == n, op, ": every tensor has p's size");
  for (const at::Tensor* t : state) TORCH_CHECK(t->numel() == n, op, ": every tensor has p's size");
}

static void adam(at::Tensor p, at::Tensor m, at::Tensor v, c10::optional<at::Tensor> g32,
                 c10::optional<at::Tensor> g16, c10::optional<at::Tensor> shadow, double lr, double b1, double b2,
                 double eps, double wd, int64_t step, double grad_scale, c10::optional<at::Tensor> gzero,
                 c10::optional<at::Tensor> ema, double ema_decay, bool ema_first, bool decoupled,
                 const std::vector<int64_t>& wd_starts, const std::vector<double>& wd_values) {
  c10::cuda::CUDAGuard g(p.device());
  check_optimizer("adam", "p, m and v", {&p, &m, &v}, g32, g16, shadow, gzero, ema, ema_decay);
  const b200::OptStep o =
      b200::make_opt_step("adam", decoupled ? b200::OPT_ADAMW : b200::OPT_ADAM, p.numel(), lr, b1, b2, eps, 0.0,
                          (int)step, false, grad_scale, wd, wd_starts, wd_values, ema_decay, ema_first);
  b200::optimizer_fused(o, f32p(p), f32p(m), f32p(v), f32p_opt(g32), bfp_opt(g16),
                        shadow.has_value() ? bfp_mut(*shadow) : nullptr, f32p_opt(gzero), f32p_opt(ema), p.numel(),
                        cur_stream());
}
static void sgd(at::Tensor p, at::Tensor mom, c10::optional<at::Tensor> g32, c10::optional<at::Tensor> g16,
                c10::optional<at::Tensor> shadow, double lr, double momentum, double wd, bool first,
                double grad_scale, c10::optional<at::Tensor> gzero, c10::optional<at::Tensor> ema, double ema_decay,
                bool ema_first, const std::vector<int64_t>& wd_starts, const std::vector<double>& wd_values) {
  c10::cuda::CUDAGuard g(p.device());
  check_optimizer("sgd", "p and mom", {&p, &mom}, g32, g16, shadow, gzero, ema, ema_decay);
  const b200::OptStep o = b200::make_opt_step("sgd", b200::OPT_SGD, p.numel(), lr, 0.0, 0.0, 0.0, momentum, 0, first,
                                              grad_scale, wd, wd_starts, wd_values, ema_decay, ema_first);
  b200::optimizer_fused(o, f32p(p), f32p(mom), nullptr, f32p_opt(g32), bfp_opt(g16),
                        shadow.has_value() ? bfp_mut(*shadow) : nullptr, f32p_opt(gzero), f32p_opt(ema), p.numel(),
                        cur_stream());
}
// LAMB / LARS, one phase of one launch over p's n elements (loss_optim.cu).  The segment table comes as six
// equal-length lists; the workspace must hold every slot the table names, the ratio array every tensor.
static void layerwise(int64_t phase, const std::string& kind, at::Tensor p, at::Tensor m, c10::optional<at::Tensor> v,
                      c10::optional<at::Tensor> g32, c10::optional<at::Tensor> g16, c10::optional<at::Tensor> shadow,
                      c10::optional<at::Tensor> gzero, c10::optional<at::Tensor> ema, at::Tensor ws,
                      c10::optional<at::Tensor> ratio, double lr, double b1, double b2, double eps, double momentum,
                      int64_t step, bool first, double grad_scale, double ema_decay, bool ema_first,
                      const std::vector<int64_t>& starts, const std::vector<int64_t>& ctas,
                      const std::vector<int64_t>& slots, const std::vector<int64_t>& nslots,
                      const std::vector<int64_t>& tensors, const std::vector<double>& wds, double trust_coeff,
                      double trust_eps) {
  c10::cuda::CUDAGuard g(p.device());
  TORCH_CHECK(phase == 1 || phase == 2, "layerwise: phase must be 1 or 2");
  TORCH_CHECK(kind == "lamb" || kind == "lars", "layerwise: kind must be lamb or lars, got ", kind);
  const bool lamb = kind == "lamb";
  const char* op = phase == 1 ? "layerwise_phase1" : "layerwise_phase2";
  TORCH_CHECK(!lamb || v.has_value(), op, ": LAMB needs v");
  const bool reads_grad = phase == 1 || !lamb;
  TORCH_CHECK(!reads_grad || g32.has_value() != g16.has_value(), op, ": exactly one of g32 and g16");
  TORCH_CHECK(reads_grad || (!g32.has_value() && !g16.has_value() && !gzero.has_value()), op,
              ": LAMB's phase 2 reads no gradient");
  TORCH_CHECK(phase == 2 || (!shadow.has_value() && !ema.has_value() && !ratio.has_value()), op,
              ": phase 1 writes no shadow, EMA or ratio");
  TORCH_CHECK(!(phase == 1 && !lamb && gzero.has_value()), op, ": LARS clears the gradient in phase 2");
  const int64_t n = p.numel();
  for (const at::Tensor* t : {&p, &m}) check_vec(*t, at::kFloat, 16, op, "p and m");
  if (lamb) check_vec(*v, at::kFloat, 16, op, "v");
  check_ema(ema, n, ema_decay, op);
  if (g32.has_value()) check_vec(*g32, at::kFloat, 16, op, "g32");
  if (gzero.has_value()) check_vec(*gzero, at::kFloat, 16, op, "gzero");
  if (g16.has_value()) check_vec(*g16, at::kBFloat16, 8, op, "g16");
  if (shadow.has_value()) check_vec(*shadow, at::kBFloat16, 8, op, "shadow");
  for (const auto* t : {&g32, &g16, &shadow, &gzero})
    TORCH_CHECK(!t->has_value() || (*t)->numel() == n, op, ": every tensor has p's size");
  TORCH_CHECK(m.numel() == n && (!lamb || v->numel() == n), op, ": every tensor has p's size");
  check_vec(ws, at::kFloat, 16, op, "ws");
  const b200::LayerwiseLaunch L =
      b200::make_layerwise_launch(op, p.numel(), starts, ctas, slots, nslots, tensors, wds, trust_coeff, trust_eps,
                                  b200::layerwise_max_grid());
  int64_t need = 0, tmax = -1;
  for (size_t k = 0; k < starts.size(); ++k) {
    need = std::max<int64_t>(need, slots[k] + (phase == 1 ? ctas[k] : nslots[k]));
    tmax = std::max<int64_t>(tmax, tensors[k]);
    TORCH_CHECK(phase == 1 || nslots[k] >= 1, op, ": every tensor has at least one slot");
  }
  TORCH_CHECK(ws.numel() >= 2 * need, op, ": ws must hold 2 x ", need, " floats, got ", ws.numel());
  if (ratio.has_value()) {
    check_vec(*ratio, at::kFloat, 4, op, "ratio");
    TORCH_CHECK(ratio->numel() > tmax, op, ": ratio must hold tensor ", tmax);
  }
  const b200::OptStep o = b200::make_opt_step(op, lamb ? b200::OPT_LAMB : b200::OPT_LARS, p.numel(), lr,
                                              lamb ? b1 : 0.0, lamb ? b2 : 0.0, lamb ? eps : 0.0, momentum,
                                              lamb ? (int)step : 0, first, grad_scale, 0.0, {}, {}, ema_decay,
                                              ema_first);
  float* vp = lamb ? f32p(*v) : nullptr;
  if (phase == 1)
    b200::layerwise_phase1(o, L, f32p(p), f32p(m), vp, f32p_opt(g32), bfp_opt(g16), f32p_opt(gzero), f32p(ws),
                           cur_stream());
  else
    b200::layerwise_phase2(o, L, f32p(p), f32p(m), vp, f32p_opt(g32), bfp_opt(g16),
                           shadow.has_value() ? bfp_mut(*shadow) : nullptr, f32p_opt(gzero), f32p_opt(ema), f32p(ws),
                           f32p_opt(ratio), cur_stream());
}
static void ema_update(const at::Tensor& p, at::Tensor ema, double decay, bool first) {
  c10::cuda::CUDAGuard g(p.device());
  check_vec(p, at::kFloat, 16, "ema_update", "p");
  check_ema(ema, p.numel(), decay, "ema_update");
  b200::ema_fused(f32p(p), f32p(ema), p.numel(), decay, first, cur_stream());
}

// ---- PowerSGD (powersgd.cu): one n x m fp32 matrix, P [n][rank], Q [m][rank]
static void check_psgd(const char* op, int64_t n, int64_t m, int64_t rank) {
  TORCH_CHECK(rank >= 1 && rank <= b200::PSGD_MAX_RANK, op, ": rank must lie in [1, ", b200::PSGD_MAX_RANK,
              "] (got ", rank, "): each thread keeps rank fp32 accumulators in a 40-register budget");
  TORCH_CHECK(n >= 1 && m >= 4 && m % 4 == 0 && n <= INT32_MAX && m <= INT32_MAX, op,
              ": needs n >= 1 and m >= 4 a multiple of 4 (got ", n, " x ", m, ")");
}
static void check_psgd_operand(const at::Tensor& t, int64_t elems, const char* op, const char* name) {
  check_vec(t, at::kFloat, 16, op, name);
  TORCH_CHECK(t.numel() >= elems, op, ": ", name, " must hold ", elems, " elements, got ", t.numel());
}
static void psgd_project(const at::Tensor& g, at::Tensor e, const at::Tensor& q, at::Tensor p, int64_t n, int64_t m,
                         int64_t rank, double scale) {
  c10::cuda::CUDAGuard guard(g.device());
  check_psgd("psgd_project", n, m, rank);
  check_psgd_operand(g, n * m, "psgd_project", "g");
  check_psgd_operand(e, n * m, "psgd_project", "e");
  check_psgd_operand(q, m * rank, "psgd_project", "q");
  check_psgd_operand(p, n * rank, "psgd_project", "p");
  b200::psgd_project(f32p(g), f32p(e), f32p(q), f32p(p), (int)n, (int)m, (int)rank, (float)scale, cur_stream());
}
static void psgd_backproject(const at::Tensor& M, const at::Tensor& p, at::Tensor q, at::Tensor ws, int64_t n, int64_t m,
                             int64_t rank) {
  c10::cuda::CUDAGuard guard(M.device());
  check_psgd("psgd_backproject", n, m, rank);
  check_psgd_operand(M, n * m, "psgd_backproject", "M");
  check_psgd_operand(p, n * rank, "psgd_backproject", "p");
  check_psgd_operand(q, m * rank, "psgd_backproject", "q");
  check_psgd_operand(ws, b200::psgd_workspace_elems((int)n, (int)m, (int)rank, b200::sm_count()), "psgd_backproject",
                     "the workspace");
  b200::psgd_backproject(f32p(M), f32p(p), f32p(q), f32p(ws), ws.numel(), (int)n, (int)m, (int)rank, cur_stream());
}
static void psgd_orthogonalize(at::Tensor x, int64_t rows, int64_t rank, int64_t count) {
  c10::cuda::CUDAGuard guard(x.device());
  check_psgd("psgd_orthogonalize", 1, 4, rank);
  TORCH_CHECK(count >= 1 && rows >= rank && rows <= INT32_MAX, "psgd_orthogonalize: needs count >= 1 and rows >= rank");
  check_psgd_operand(x, count * rows * rank, "psgd_orthogonalize", "x");
  b200::psgd_orthogonalize(f32p(x), (int)rows, (int)count, (int)rank, cur_stream());
}
static void psgd_decompress(const at::Tensor& p, const at::Tensor& q, at::Tensor g, at::Tensor e, int64_t n, int64_t m,
                            int64_t rank, double alpha) {
  c10::cuda::CUDAGuard guard(g.device());
  check_psgd("psgd_decompress", n, m, rank);
  check_psgd_operand(p, n * rank, "psgd_decompress", "p");
  check_psgd_operand(q, m * rank, "psgd_decompress", "q");
  check_psgd_operand(g, n * m, "psgd_decompress", "g");
  check_psgd_operand(e, n * m, "psgd_decompress", "e");
  b200::psgd_decompress(f32p(p), f32p(q), f32p(g), f32p(e), (int)n, (int)m, (int)rank, (float)alpha, cur_stream());
}

static void check_augment(const at::Tensor& src, const at::Tensor& params, const at::Tensor& out, int64_t OH,
                          int64_t OW, int64_t mode, int64_t pad, const std::vector<double>& mean,
                          const std::vector<double>& stdv) {
  TORCH_CHECK(src.is_cuda() && src.scalar_type() == at::kByte && src.is_contiguous() && src.dim() == 4 && src.size(3) == 3,
              "augment: uint8 [N,H,W,3] CUDA tensor");
  const int64_t N = src.size(0);
  TORCH_CHECK(params.is_contiguous() && params.dim() == 2 && params.size(0) >= N && params.size(1) == 8,
              "augment: params must be contiguous [N, 8]");
  TORCH_CHECK(mode == 0 || mode == 1, "augment: mode is 0 (NHWC) or 1 (im2col)");
  TORCH_CHECK(OH > 0 && OW > 0 && mean.size() == 3 && stdv.size() == 3, "augment: OH, OW > 0, 3 means and deviations");
  // mode 0 writes 3 channels and zeros up to pad (one 8-byte store at pad = 4); mode 1 16-byte stores of pad-wide rows
  TORCH_CHECK(mode == 1 || pad >= 3, "augment: NHWC pad must be >= 3");
  check_vec(out, at::kBFloat16, mode == 1 ? 16 : (pad == 4 ? 8 : 2), "augment", "out");
  TORCH_CHECK(out.numel() >= N * OH * OW * pad, "augment: out must hold N x OH x OW x pad elements");
}

static void augment(const at::Tensor& src, const at::Tensor& params, at::Tensor out, int64_t RH, int64_t RW,
                    int64_t OH, int64_t OW, int64_t mode, int64_t pad, std::vector<double> mean,
                    std::vector<double> stdv) {
  c10::cuda::CUDAGuard g(src.device());
  check_augment(src, params, out, OH, OW, mode, pad, mean, stdv);
  float m[3] = {(float)mean[0], (float)mean[1], (float)mean[2]}, s[3] = {(float)stdv[0], (float)stdv[1], (float)stdv[2]};
  b200::augment_fused(src.data_ptr<uint8_t>(), f32p(params), bfp_mut(out), src.size(0), src.size(1), src.size(2),
                      (int)RH, (int)RW, (int)OH, (int)OW, (int)mode, (int)pad, m, s, cur_stream());
}

// One batch's MixUp (kind 1: lam) or CutMix (kind 2: the box x1, y1, x2, y2 in output pixels) draw.
static b200::MixParams mix_params(const char* what, int64_t kind, double lam, const std::vector<int64_t>& box,
                                  int64_t OH, int64_t OW) {
  TORCH_CHECK(kind == b200::MixMixUp || kind == b200::MixCutMix, what, ": kind is 1 (MixUp) or 2 (CutMix)");
  TORCH_CHECK(lam >= 0.0 && lam <= 1.0, what, ": lam must lie in [0, 1], got ", lam);
  TORCH_CHECK(box.size() == 4, what, ": box is (x1, y1, x2, y2)");
  TORCH_CHECK(kind == b200::MixMixUp || (0 <= box[0] && box[0] <= box[2] && box[2] <= OW && 0 <= box[1] &&
                                         box[1] <= box[3] && box[3] <= OH),
              what, ": CutMix box (", box[0], ", ", box[1], ", ", box[2], ", ", box[3], ") outside ", OH, " x ", OW);
  return b200::MixParams{(int)kind, (float)lam, (float)(1.0 - lam), (int)box[0], (int)box[1], (int)box[2], (int)box[3]};
}

static void augment_mixed(const at::Tensor& src, const at::Tensor& params, at::Tensor out, int64_t RH, int64_t RW,
                          int64_t OH, int64_t OW, int64_t pad, std::vector<double> mean, std::vector<double> stdv,
                          int64_t kind, double lam, std::vector<int64_t> box) {
  c10::cuda::CUDAGuard g(src.device());
  check_augment(src, params, out, OH, OW, 0, pad, mean, stdv);
  TORCH_CHECK(src.size(0) >= 1 && src.size(0) <= (1 << 24), "augment_mixed: 1 to 2^24 images");
  const b200::MixParams mix = mix_params("augment_mixed", kind, lam, box, OH, OW);
  float m[3] = {(float)mean[0], (float)mean[1], (float)mean[2]}, s[3] = {(float)stdv[0], (float)stdv[1], (float)stdv[2]};
  b200::augment_mixed(src.data_ptr<uint8_t>(), f32p(params), bfp_mut(out), src.size(0), src.size(1), src.size(2),
                      (int)RH, (int)RW, (int)OH, (int)OW, (int)pad, m, s, mix, cur_stream());
}
// Bytes of the intermediate augment_ragged needs for these geometry rows: H x RW x 3 per image.
static int64_t ragged_inter_bytes(const at::Tensor& geom) {
  TORCH_CHECK(!geom.is_cuda() && geom.scalar_type() == at::kLong && geom.dim() == 2 && geom.size(1) == 5 &&
                  geom.is_contiguous(), "ragged_inter_bytes: geom must be a CPU int64 [N, 5] tensor");
  const int64_t* g = geom.data_ptr<int64_t>();
  int64_t total = 0;
  for (int64_t i = 0; i < geom.size(0); ++i) total += g[i * 5 + 1] * g[i * 5 + 4] * 3;
  return total;
}

// The kernels read geom and params on the device; the host copies they were made from are checked
// here, so that no row can send a launch outside src, inter or out.
static void augment_ragged_impl(const at::Tensor& src, const at::Tensor& geom, const at::Tensor& params,
                                at::Tensor inter, at::Tensor out, const at::Tensor& geom_host,
                                const at::Tensor& params_host, int64_t OH, int64_t OW, const std::vector<double>& mean,
                                const std::vector<double>& stdv, const b200::MixParams* mix) {
  c10::cuda::CUDAGuard g(src.device());
  TORCH_CHECK(src.is_cuda() && src.scalar_type() == at::kByte && src.is_contiguous(),
              "augment_ragged: src must be a contiguous CUDA uint8 tensor");
  TORCH_CHECK(inter.is_cuda() && inter.scalar_type() == at::kByte && inter.is_contiguous(),
              "augment_ragged: inter must be a contiguous CUDA uint8 tensor");
  TORCH_CHECK(geom.is_cuda() && geom.scalar_type() == at::kLong && geom.is_contiguous() && geom.dim() == 2 &&
                  geom.size(1) == 5, "augment_ragged: geom must be a contiguous CUDA int64 [N, 5] tensor");
  const int64_t N = geom.size(0);
  TORCH_CHECK(N > 0 && N <= 65535, "augment_ragged: 1 to 65535 images");
  TORCH_CHECK(params.is_cuda() && params.scalar_type() == at::kFloat && params.is_contiguous() && params.dim() == 2 &&
                  params.size(0) == N && params.size(1) == 8, "augment_ragged: params must be a contiguous CUDA fp32 [N, 8] tensor");
  TORCH_CHECK(!geom_host.is_cuda() && geom_host.scalar_type() == at::kLong && geom_host.is_contiguous() &&
                  geom_host.sizes() == geom.sizes(), "augment_ragged: geom_host must be the CPU int64 copy of geom");
  TORCH_CHECK(!params_host.is_cuda() && params_host.scalar_type() == at::kFloat && params_host.is_contiguous() &&
                  params_host.sizes() == params.sizes(), "augment_ragged: params_host must be the CPU fp32 copy of params");
  TORCH_CHECK(OH > 0 && OW > 0 && mean.size() == 3 && stdv.size() == 3, "augment_ragged: OH, OW > 0, 3 means and deviations");
  check_vec(out, at::kBFloat16, 8, "augment_ragged", "out");
  TORCH_CHECK(out.numel() >= N * OH * OW * 4, "augment_ragged: out must hold N x OH x OW x 4 elements");
  const int64_t* gh = geom_host.data_ptr<int64_t>();
  const float* ph = params_host.data_ptr<float>();
  int64_t most = 1;
  for (int64_t i = 0; i < N; ++i) {
    const int64_t off = gh[i * 5], H = gh[i * 5 + 1], W = gh[i * 5 + 2], RH = gh[i * 5 + 3], RW = gh[i * 5 + 4];
    TORCH_CHECK(H >= 1 && W >= 1 && H <= 65535 && W <= 65535 && off >= 0 && off + H * W * 3 <= src.numel(),
                "augment_ragged: image ", i, " (offset ", off, ", ", H, " x ", W, ") lies outside src of ",
                src.numel(), " bytes");
    TORCH_CHECK(RH >= 1 && RW >= 1 && RH <= (1 << 24) && RW <= (1 << 24), "augment_ragged: image ", i,
                " has a resized size of ", RH, " x ", RW);
    const int64_t top = (int64_t)ph[i * 8], left = (int64_t)ph[i * 8 + 1];
    const int64_t ch = (int64_t)ph[i * 8 + 2], cw = (int64_t)ph[i * 8 + 3];
    TORCH_CHECK(top >= 0 && left >= 0 && ch >= 1 && cw >= 1 && top + ch <= H && left + cw <= W, "augment_ragged: image ",
                i, " has a crop box (", top, ", ", left, ", ", ch, ", ", cw, ") outside its ", H, " x ", W, " pixels");
    most = std::max(most, H * RW);
  }
  const int64_t need = ragged_inter_bytes(geom_host);
  TORCH_CHECK(inter.numel() >= need, "augment_ragged: inter must hold ", need, " bytes, got ", inter.numel());
  // blocks per image: enough for the largest image, at most 16 blocks per SM over the batch
  const int64_t cap = std::max<int64_t>(1, 16 * b200::sm_count() / N);
  const int grid_x = (int)std::min(cap, std::max((most + 255) / 256, (OH * OW + 255) / 256));
  float m[3] = {(float)mean[0], (float)mean[1], (float)mean[2]}, s[3] = {(float)stdv[0], (float)stdv[1], (float)stdv[2]};
  b200::augment_ragged(src.data_ptr<uint8_t>(), reinterpret_cast<const long long*>(geom.data_ptr<int64_t>()),
                       f32p(params), inter.data_ptr<uint8_t>(), bfp_mut(out), (int)N, (int)OH, (int)OW, grid_x, m, s,
                       cur_stream(), mix);
}

static void augment_ragged(const at::Tensor& src, const at::Tensor& geom, const at::Tensor& params, at::Tensor inter,
                           at::Tensor out, const at::Tensor& geom_host, const at::Tensor& params_host, int64_t OH,
                           int64_t OW, std::vector<double> mean, std::vector<double> stdv) {
  augment_ragged_impl(src, geom, params, inter, out, geom_host, params_host, OH, OW, mean, stdv, nullptr);
}

static void augment_ragged_mixed(const at::Tensor& src, const at::Tensor& geom, const at::Tensor& params,
                                 at::Tensor inter, at::Tensor out, const at::Tensor& geom_host,
                                 const at::Tensor& params_host, int64_t OH, int64_t OW, std::vector<double> mean,
                                 std::vector<double> stdv, int64_t kind, double lam, std::vector<int64_t> box) {
  const b200::MixParams mix = mix_params("augment_ragged_mixed", kind, lam, box, OH, OW);
  augment_ragged_impl(src, geom, params, inter, out, geom_host, params_host, OH, OW, mean, stdv, &mix);
}
// A test-time augmentation view code (TtaPosition, or'ed with TtaFlip) whose OH x OW crop fits an RH x RW image.
static void check_view(const char* what, int64_t view, int64_t RH, int64_t RW, int64_t OH, int64_t OW) {
  TORCH_CHECK(view >= 0 && (view & ~(int64_t)b200::TtaFlip) <= b200::TtaCentreMirror, what, ": bad view code ", view);
  TORCH_CHECK(OH <= RH && OW <= RW, what, ": a ", OH, " x ", OW, " view does not fit a ", RH, " x ", RW, " image");
}

static void augment_view(const at::Tensor& src, const at::Tensor& params, at::Tensor out, int64_t RH, int64_t RW,
                         int64_t OH, int64_t OW, int64_t view, std::vector<double> mean, std::vector<double> stdv) {
  c10::cuda::CUDAGuard g(src.device());
  check_augment(src, params, out, OH, OW, 0, 4, mean, stdv);
  check_view("augment_view", view, RH, RW, OH, OW);
  float m[3] = {(float)mean[0], (float)mean[1], (float)mean[2]}, s[3] = {(float)stdv[0], (float)stdv[1], (float)stdv[2]};
  b200::augment_view(src.data_ptr<uint8_t>(), f32p(params), bfp_mut(out), src.size(0), src.size(1), src.size(2),
                     (int)RH, (int)RW, (int)OH, (int)OW, (int)view, m, s, cur_stream());
}

// augment_ragged for one view; `pass1`: the codes of every view of the batch, to run pass 1 for them first (empty:
// inter already holds it).  Every operand is checked as augment_ragged checks it, and every view against every image.
static void augment_ragged_view(const at::Tensor& src, const at::Tensor& geom, const at::Tensor& params,
                                at::Tensor inter, at::Tensor out, const at::Tensor& geom_host,
                                const at::Tensor& params_host, int64_t OH, int64_t OW, std::vector<double> mean,
                                std::vector<double> stdv, int64_t view, std::vector<int64_t> pass1) {
  c10::cuda::CUDAGuard g(src.device());
  TORCH_CHECK(src.is_cuda() && src.scalar_type() == at::kByte && src.is_contiguous(),
              "augment_ragged_view: src must be a contiguous CUDA uint8 tensor");
  TORCH_CHECK(inter.is_cuda() && inter.scalar_type() == at::kByte && inter.is_contiguous(),
              "augment_ragged_view: inter must be a contiguous CUDA uint8 tensor");
  TORCH_CHECK(geom.is_cuda() && geom.scalar_type() == at::kLong && geom.is_contiguous() && geom.dim() == 2 &&
                  geom.size(1) == 5, "augment_ragged_view: geom must be a contiguous CUDA int64 [N, 5] tensor");
  const int64_t N = geom.size(0);
  TORCH_CHECK(N > 0 && N <= 65535, "augment_ragged_view: 1 to 65535 images");
  TORCH_CHECK(params.is_cuda() && params.scalar_type() == at::kFloat && params.is_contiguous() && params.dim() == 2 &&
                  params.size(0) == N && params.size(1) == 8,
              "augment_ragged_view: params must be a contiguous CUDA fp32 [N, 8] tensor");
  TORCH_CHECK(!geom_host.is_cuda() && geom_host.scalar_type() == at::kLong && geom_host.is_contiguous() &&
                  geom_host.sizes() == geom.sizes(), "augment_ragged_view: geom_host must be the CPU int64 copy of geom");
  TORCH_CHECK(!params_host.is_cuda() && params_host.scalar_type() == at::kFloat && params_host.is_contiguous() &&
                  params_host.sizes() == params.sizes(),
              "augment_ragged_view: params_host must be the CPU fp32 copy of params");
  TORCH_CHECK(OH > 0 && OW > 0 && mean.size() == 3 && stdv.size() == 3,
              "augment_ragged_view: OH, OW > 0, 3 means and deviations");
  TORCH_CHECK((int64_t)pass1.size() <= b200::kTtaMaxViews, "augment_ragged_view: at most ", b200::kTtaMaxViews,
              " views");
  check_vec(out, at::kBFloat16, 8, "augment_ragged_view", "out");
  TORCH_CHECK(out.numel() >= N * OH * OW * 4, "augment_ragged_view: out must hold N x OH x OW x 4 elements");
  const int64_t* gh = geom_host.data_ptr<int64_t>();
  const float* ph = params_host.data_ptr<float>();
  int64_t most = 1;
  for (int64_t i = 0; i < N; ++i) {
    const int64_t off = gh[i * 5], H = gh[i * 5 + 1], W = gh[i * 5 + 2], RH = gh[i * 5 + 3], RW = gh[i * 5 + 4];
    TORCH_CHECK(H >= 1 && W >= 1 && H <= 65535 && W <= 65535 && off >= 0 && off + H * W * 3 <= src.numel(),
                "augment_ragged_view: image ", i, " (offset ", off, ", ", H, " x ", W, ") lies outside src of ",
                src.numel(), " bytes");
    TORCH_CHECK(RH >= 1 && RW >= 1 && RH <= (1 << 24) && RW <= (1 << 24), "augment_ragged_view: image ", i,
                " has a resized size of ", RH, " x ", RW);
    const int64_t top = (int64_t)ph[i * 8], left = (int64_t)ph[i * 8 + 1];
    const int64_t ch = (int64_t)ph[i * 8 + 2], cw = (int64_t)ph[i * 8 + 3];
    TORCH_CHECK(top >= 0 && left >= 0 && ch >= 1 && cw >= 1 && top + ch <= H && left + cw <= W,
                "augment_ragged_view: image ", i, " has a crop box (", top, ", ", left, ", ", ch, ", ", cw,
                ") outside its ", H, " x ", W, " pixels");
    check_view("augment_ragged_view", view, RH, RW, OH, OW);
    for (int64_t v : pass1) check_view("augment_ragged_view", v, RH, RW, OH, OW);
    most = std::max(most, H * RW);
  }
  const int64_t need = ragged_inter_bytes(geom_host);
  TORCH_CHECK(inter.numel() >= need, "augment_ragged_view: inter must hold ", need, " bytes, got ", inter.numel());
  const int64_t cap = std::max<int64_t>(1, 16 * b200::sm_count() / N);
  const int grid_x = (int)std::min(cap, std::max((most + 255) / 256, (OH * OW + 255) / 256));
  b200::TtaViews views{0ull, (int)pass1.size()};
  for (size_t v = 0; v < pass1.size(); ++v) views.codes |= (unsigned long long)pass1[v] << (4 * v);
  float m[3] = {(float)mean[0], (float)mean[1], (float)mean[2]}, s[3] = {(float)stdv[0], (float)stdv[1], (float)stdv[2]};
  b200::augment_ragged_view(src.data_ptr<uint8_t>(), reinterpret_cast<const long long*>(geom.data_ptr<int64_t>()),
                            f32p(params), inter.data_ptr<uint8_t>(), bfp_mut(out), (int)N, (int)OH, (int)OW, grid_x, m,
                            s, (int)view, pass1.empty() ? nullptr : &views, cur_stream());
}

// One view's step of the view-mean reduction (tta_accumulate in api.h).
static void tta_accumulate(const at::Tensor& logits, const at::Tensor& target, at::Tensor acc,
                           c10::optional<at::Tensor> meter, c10::optional<at::Tensor> loss_out, int64_t view,
                           int64_t views) {
  c10::cuda::CUDAGuard g(logits.device());
  TORCH_CHECK(logits.is_cuda() && logits.scalar_type() == at::kFloat && logits.is_contiguous() && logits.dim() == 2,
              "tta_accumulate: logits must be a contiguous CUDA fp32 [B, C] tensor");
  const int64_t B = logits.size(0), C = logits.size(1);
  TORCH_CHECK(B >= 1 && C >= 1, "tta_accumulate: empty logits");
  TORCH_CHECK(views >= 1 && views <= b200::kTtaMaxViews, "tta_accumulate: views must lie in [1, ",
              b200::kTtaMaxViews, "], got ", views);
  TORCH_CHECK(view >= 0 && view < views, "tta_accumulate: view ", view, " outside [0, ", views, ")");
  TORCH_CHECK(target.is_cuda() && target.scalar_type() == at::kLong && target.is_contiguous() && target.numel() >= B,
              "tta_accumulate: contiguous CUDA int64 targets of B = ", B);
  TORCH_CHECK(acc.is_cuda() && acc.scalar_type() == at::kFloat && acc.is_contiguous() && acc.numel() >= B * C,
              "tta_accumulate: acc must be a contiguous CUDA fp32 tensor of at least B x C elements");
  TORCH_CHECK(!meter.has_value() || (meter->scalar_type() == at::kFloat && meter->numel() >= 3),
              "tta_accumulate: meter must have 3 fp32 elements");
  TORCH_CHECK(!loss_out.has_value() || (loss_out->scalar_type() == at::kFloat && loss_out->numel() >= 1),
              "tta_accumulate: loss_out must have 1 fp32 element");
  b200::tta_accumulate(f32p(logits), reinterpret_cast<const long long*>(target.data_ptr()), f32p(acc),
                       f32p_opt(meter), f32p_opt(loss_out), (int)B, (int)C, (int)view, (int)views, cur_stream());
}

// Per-class evaluation counts of one batch (class_metrics in api.h).
static void class_metrics(const at::Tensor& scores, const at::Tensor& target, at::Tensor confusion, at::Tensor top5,
                          int64_t views) {
  c10::cuda::CUDAGuard g(scores.device());
  TORCH_CHECK(scores.is_cuda() && scores.scalar_type() == at::kFloat && scores.is_contiguous() && scores.dim() == 2,
              "class_metrics: scores must be a contiguous CUDA fp32 [B, C] tensor");
  const int64_t B = scores.size(0), C = scores.size(1);
  TORCH_CHECK(B >= 1 && C >= 1, "class_metrics: empty scores");
  TORCH_CHECK(views >= 1 && views <= b200::kTtaMaxViews, "class_metrics: views must lie in [1, ", b200::kTtaMaxViews,
              "], got ", views);
  TORCH_CHECK(target.device() == scores.device() && target.scalar_type() == at::kLong && target.is_contiguous() &&
                  target.numel() >= B,
              "class_metrics: contiguous int64 targets of B = ", B, " on the scores' device");
  TORCH_CHECK(confusion.device() == scores.device() && confusion.scalar_type() == at::kLong &&
                  confusion.is_contiguous(),
              "class_metrics: confusion must be a contiguous int64 tensor on the scores' device");
  TORCH_CHECK(confusion.dim() == 2 && confusion.size(0) == C && confusion.size(1) == C,
              "class_metrics: confusion must be [", C, ", ", C, "] for scores of ", C, " classes, got ",
              confusion.sizes());
  TORCH_CHECK(top5.device() == scores.device() && top5.scalar_type() == at::kLong && top5.numel() >= 1,
              "class_metrics: top5 must hold one int64 on the scores' device");
  b200::class_metrics(f32p(scores), reinterpret_cast<const long long*>(target.data_ptr()),
                      reinterpret_cast<long long*>(confusion.data_ptr()), reinterpret_cast<long long*>(top5.data_ptr()),
                      (int)B, (int)C, (int)views, cur_stream());
}

static void im2col_c3(const at::Tensor& x, at::Tensor out, int64_t kpad) {
  c10::cuda::CUDAGuard g(x.device());
  check_vec(x, at::kBFloat16, 8, "im2col_c3", "x");
  check_vec(out, at::kBFloat16, 16, "im2col_c3", "out");
  TORCH_CHECK(x.dim() == 4 && x.size(3) == 4, "im2col_c3: x must be [N, H, W, 4]");
  TORCH_CHECK(kpad >= 32 && kpad % 8 == 0 && out.numel() >= x.size(0) * x.size(1) * x.size(2) * kpad,
              "im2col_c3: kpad a multiple of 8 >= 32, out of N x H x W x kpad elements");
  b200::im2col3x3_c3(bfp(x), bfp_mut(out), x.size(0), x.size(1), x.size(2), x.size(3), (int)kpad, cur_stream());
}
static void nchw_to_nhwc(const at::Tensor& x, at::Tensor y) {
  c10::cuda::CUDAGuard g(x.device());
  TORCH_CHECK(x.is_contiguous() && x.dim() == 4, "nchw_to_nhwc: contiguous NCHW fp32");
  TORCH_CHECK(y.is_contiguous() && y.dim() == 4 && y.size(3) >= x.size(1), "nchw_to_nhwc: contiguous NHWC y, cpad >= C");
  check_nhwc(y, x.size(0), x.size(2), x.size(3), y.size(3), "nchw_to_nhwc", "y");
  b200::nchw_f32_to_nhwc_bf16(f32p(x), bfp_mut(y), x.size(0), x.size(1), x.size(2), x.size(3), y.size(3), cur_stream());
}

// ------------------------------------------------------------------------------------ PNG decode
namespace b200 {
struct PngImage {
  int w = 0, h = 0;
  std::vector<uint8_t> rgb;
  bool ok = false;
};
void decode_png_files(const std::vector<std::string>& paths, int threads, std::vector<PngImage>& out);
void decode_png_files_into(const std::vector<std::string>& paths, int threads, uint8_t* dst, const int64_t* offsets,
                           const int64_t* hw, uint8_t* ok);
void check_png_files(const std::vector<std::string>& paths, int threads, const int64_t* hw, uint8_t* ok);
}  // namespace b200

// bool [N]: which files the native PNG decoder takes at their size hw[i] = (H, W) (the stream pipeline's start-up
// check; the rest go to PIL).
static at::Tensor png_decodable(const std::vector<std::string>& paths, const at::Tensor& hw, int64_t threads) {
  const int64_t N = (int64_t)paths.size();
  TORCH_CHECK(!hw.is_cuda() && hw.scalar_type() == at::kLong && hw.is_contiguous() && hw.numel() == 2 * N,
              "png_decodable: hw must be a CPU int64 [N, 2] tensor");
  at::Tensor ok = at::zeros({N}, at::kBool);
  {
    py::gil_scoped_release nogil;
    b200::check_png_files(paths, (int)threads, hw.data_ptr<int64_t>(), reinterpret_cast<uint8_t*>(ok.data_ptr<bool>()));
  }
  return ok;
}

// Ragged splits: decode each file into flat[offsets[i] :] when it is a plain 8-bit PNG of size hw[i].
// Returns a bool [N] tensor of the files written; the caller decodes the rest with PIL.
static at::Tensor decode_pngs_into(const std::vector<std::string>& paths, at::Tensor flat, const at::Tensor& offsets,
                                   const at::Tensor& hw, int64_t threads) {
  const int64_t N = (int64_t)paths.size();
  TORCH_CHECK(!flat.is_cuda() && flat.scalar_type() == at::kByte && flat.is_contiguous(),
              "decode_pngs_into: flat must be a contiguous CPU uint8 tensor");
  TORCH_CHECK(!offsets.is_cuda() && offsets.scalar_type() == at::kLong && offsets.is_contiguous() && offsets.numel() == N,
              "decode_pngs_into: offsets must be a CPU int64 [N] tensor");
  TORCH_CHECK(!hw.is_cuda() && hw.scalar_type() == at::kLong && hw.is_contiguous() && hw.numel() == 2 * N,
              "decode_pngs_into: hw must be a CPU int64 [N, 2] tensor");
  const int64_t* o = offsets.data_ptr<int64_t>();
  const int64_t* s = hw.data_ptr<int64_t>();
  for (int64_t i = 0; i < N; ++i)
    TORCH_CHECK(o[i] >= 0 && s[2 * i] >= 0 && s[2 * i + 1] >= 0 && o[i] + s[2 * i] * s[2 * i + 1] * 3 <= flat.numel(),
                "decode_pngs_into: image ", i, " lies outside flat");
  at::Tensor ok = at::zeros({N}, at::kBool);
  {
    py::gil_scoped_release nogil;
    b200::decode_png_files_into(paths, (int)threads, flat.data_ptr<uint8_t>(), o, s,
                                reinterpret_cast<uint8_t*>(ok.data_ptr<bool>()));
  }
  return ok;
}

// All files decoded natively into one uint8 [N,H,W,3] tensor; throws if a file is not a plain 8-bit
// PNG or the sizes differ (the caller then falls back to PIL).
static at::Tensor decode_pngs(const std::vector<std::string>& paths, int64_t threads) {
  std::vector<b200::PngImage> imgs;
  {
    py::gil_scoped_release nogil;
    b200::decode_png_files(paths, (int)threads, imgs);
  }
  TORCH_CHECK(!imgs.empty(), "decode_pngs: no files");
  const int w = imgs[0].w, h = imgs[0].h;
  for (size_t i = 0; i < imgs.size(); ++i)
    TORCH_CHECK(imgs[i].ok && imgs[i].w == w && imgs[i].h == h, "decode_pngs: unsupported or non-uniform file ", paths[i]);
  at::Tensor out = at::empty({(int64_t)imgs.size(), h, w, 3}, at::kByte);
  uint8_t* dst = out.data_ptr<uint8_t>();
  const size_t per = (size_t)w * h * 3;
  for (size_t i = 0; i < imgs.size(); ++i) memcpy(dst + i * per, imgs[i].rgb.data(), per);
  return out;
}

// ------------------------------------------------------------------------------- batch prefetcher
namespace b200 {
struct StreamConfig;
struct PrefetchConfig {
  const uint8_t* cache;
  const int64_t* labels;
  int H, W, mb, slots;
  uint8_t* ring_img;
  float* ring_par;
  int64_t* ring_lab;
  bool train;
  float scale_lo, scale_hi, ratio_lo, ratio_hi, degrees;
  const int64_t* offsets = nullptr;
  const int64_t* hw = nullptr;
  int64_t* ring_geom = nullptr;
  int64_t slot_bytes = 0;
  int resize = 256;
  const StreamConfig* stream = nullptr;
};
class BatchPrefetcher;
BatchPrefetcher* prefetcher_create(const PrefetchConfig& c);
void prefetcher_destroy(BatchPrefetcher* p);
void prefetcher_start(BatchPrefetcher* p, std::vector<int64_t> idx, uint64_t seed);
bool prefetcher_next(BatchPrefetcher* p, int& slot, int& count);
void prefetcher_release(BatchPrefetcher* p, int slot, uint64_t cuda_event);
void prefetcher_stop(BatchPrefetcher* p);
}  // namespace b200

struct PyPrefetcher {
  b200::BatchPrefetcher* p = nullptr;
  at::Tensor cache, labels, ring_img, ring_par, ring_lab, offsets, hw, ring_geom;     // keep the storage alive
  // Uniform splits: cache [N,H,W,3], ring_img [slots][mb][H][W][3].  Ragged splits also pass offsets [N]
  // and hw [N,2] into a flat cache, ring_img [slots][slot bytes] and ring_geom [slots][mb][5].
  PyPrefetcher(at::Tensor cache_, at::Tensor labels_, at::Tensor ring_img_, at::Tensor ring_par_, at::Tensor ring_lab_,
               bool train, double scale_lo, double scale_hi, double ratio_lo, double ratio_hi, double degrees,
               c10::optional<at::Tensor> offsets_, c10::optional<at::Tensor> hw_, c10::optional<at::Tensor> ring_geom_,
               int64_t resize)
      : cache(cache_), labels(labels_), ring_img(ring_img_), ring_par(ring_par_), ring_lab(ring_lab_) {
    const bool ragged = offsets_.has_value();
    TORCH_CHECK(ragged == hw_.has_value() && ragged == ring_geom_.has_value(),
                "Prefetcher: offsets, hw and ring_geom come together");
    TORCH_CHECK(cache.scalar_type() == at::kByte && cache.is_contiguous() && !cache.is_cuda() &&
                    (ragged ? cache.dim() == 1 : cache.dim() == 4 && cache.size(3) == 3),
                "Prefetcher: cache must be a CPU uint8 [N,H,W,3] tensor, or flat for a ragged split");
    TORCH_CHECK(ring_img.dim() == (ragged ? 2 : 5) && ring_img.is_contiguous() && ring_par.is_contiguous() &&
                    ring_lab.is_contiguous() && labels.scalar_type() == at::kLong &&
                    ring_lab.scalar_type() == at::kLong && ring_par.scalar_type() == at::kFloat,
                "Prefetcher: bad ring tensors");
    const int64_t N = labels.numel();
    TORCH_CHECK(ring_par.dim() == 3 && ring_par.size(2) == 8 && ring_lab.dim() == 2 &&
                    ring_par.size(0) == ring_img.size(0) && ring_lab.size(0) == ring_img.size(0) &&
                    ring_par.size(1) == ring_lab.size(1),
                "Prefetcher: ring_par [slots][mb][8] and ring_lab [slots][mb]");
    b200::PrefetchConfig c;
    c.cache = cache.data_ptr<uint8_t>(); c.labels = labels.data_ptr<int64_t>();
    c.slots = (int)ring_img.size(0); c.mb = (int)ring_par.size(1);
    if (ragged) {
      offsets = *offsets_; hw = *hw_; ring_geom = *ring_geom_;
      TORCH_CHECK(offsets.scalar_type() == at::kLong && offsets.is_contiguous() && offsets.numel() == N &&
                      hw.scalar_type() == at::kLong && hw.is_contiguous() && hw.numel() == 2 * N,
                  "Prefetcher: offsets int64 [N] and hw int64 [N, 2]");
      TORCH_CHECK(ring_geom.scalar_type() == at::kLong && ring_geom.is_contiguous() && ring_geom.dim() == 3 &&
                      ring_geom.size(0) == c.slots && ring_geom.size(1) == c.mb && ring_geom.size(2) == 5,
                  "Prefetcher: ring_geom must be int64 [slots][mb][5]");
      // a slot must hold the mb largest images, the cache every image
      const int64_t* o = offsets.data_ptr<int64_t>();
      const int64_t* s = hw.data_ptr<int64_t>();
      std::vector<int64_t> sizes(N);
      for (int64_t i = 0; i < N; ++i) {
        sizes[i] = s[2 * i] * s[2 * i + 1] * 3;
        TORCH_CHECK(s[2 * i] >= 1 && s[2 * i + 1] >= 1 && o[i] >= 0 && o[i] + sizes[i] <= cache.numel(),
                    "Prefetcher: image ", i, " lies outside the cache");
      }
      std::sort(sizes.begin(), sizes.end(), std::greater<int64_t>());
      int64_t need = 0;
      for (int64_t i = 0; i < std::min<int64_t>(N, c.mb); ++i) need += sizes[i];
      TORCH_CHECK(ring_img.size(1) >= need, "Prefetcher: a slot of ", ring_img.size(1), " bytes cannot hold ", c.mb,
                  " images of up to ", need, " bytes");
      c.offsets = o; c.hw = s; c.ring_geom = ring_geom.data_ptr<int64_t>();
      c.slot_bytes = ring_img.size(1); c.resize = (int)resize;
      c.H = 0; c.W = 0;
    } else {
      c.H = (int)cache.size(1); c.W = (int)cache.size(2);
      TORCH_CHECK(ring_img.size(1) == c.mb && ring_img.size(2) == c.H && ring_img.size(3) == c.W,
                  "Prefetcher: ring_img must be [slots][mb][H][W][3]");
    }
    c.ring_img = ring_img.data_ptr<uint8_t>(); c.ring_par = ring_par.data_ptr<float>(); c.ring_lab = ring_lab.data_ptr<int64_t>();
    c.train = train; c.scale_lo = (float)scale_lo; c.scale_hi = (float)scale_hi;
    c.ratio_lo = (float)ratio_lo; c.ratio_hi = (float)ratio_hi; c.degrees = (float)degrees;
    p = b200::prefetcher_create(c);
  }
  ~PyPrefetcher() { if (p) b200::prefetcher_destroy(p); }
  void start(std::vector<int64_t> idx, uint64_t seed) {
    py::gil_scoped_release nogil;
    b200::prefetcher_start(p, std::move(idx), seed);
  }
  py::object next() {
    int slot = -1, count = 0;
    bool ok;
    {
      py::gil_scoped_release nogil;
      ok = b200::prefetcher_next(p, slot, count);
    }
    if (!ok) return py::none();
    return py::make_tuple(slot, count);
  }
  void release(int64_t slot, uint64_t ev) { b200::prefetcher_release(p, (int)slot, ev); }
  void stop() {
    py::gil_scoped_release nogil;
    b200::prefetcher_stop(p);
  }
};

// ---------------------------------------------------------------------------------- streaming JPEG input
namespace b200 {
struct StreamConfig {
  std::vector<std::string> paths;
  std::vector<ImageHeader> headers;
  const uint8_t* other = nullptr;
  const int64_t* other_off = nullptr;
  int16_t* ring_coef = nullptr;
  int64_t coef_cap = 0;
  int32_t* ring_quant = nullptr;
  uint8_t* ring_raw = nullptr;
  int64_t raw_cap = 0;
  int32_t* ring_desc = nullptr;
  int threads = 8;
};
}  // namespace b200

// Header rows as jpeg_scan returns them: kind, H, W, sof, ncomp, h0, v0, h1, v1, h2, v2, blocks.
constexpr int kHeaderCols = 12;
static void header_row(const b200::ImageHeader& h, int64_t* r) {
  const int64_t v[kHeaderCols] = {h.kind, h.H, h.W, h.sof, h.ncomp, h.h[0], h.v[0], h.h[1], h.v[1], h.h[2], h.v[2],
                                  h.blocks};
  std::copy(v, v + kHeaderCols, r);
}
static b200::ImageHeader header_from_row(const int64_t* r) {
  b200::ImageHeader h;
  h.kind = (int)r[0]; h.H = (int)r[1]; h.W = (int)r[2]; h.sof = (int)r[3]; h.ncomp = (int)r[4];
  for (int c = 0; c < 3; ++c) { h.h[c] = (int)r[5 + 2 * c]; h.v[c] = (int)r[6 + 2 * c]; }
  h.blocks = r[11];
  return h;
}

static at::Tensor jpeg_scan(const std::vector<std::string>& paths, int64_t threads) {
  std::vector<b200::ImageHeader> hs;
  {
    py::gil_scoped_release nogil;
    b200::scan_image_headers(paths, (int)threads, hs);
  }
  at::Tensor out = at::empty({(int64_t)paths.size(), kHeaderCols}, at::kLong);
  for (size_t i = 0; i < hs.size(); ++i) header_row(hs[i], out.data_ptr<int64_t>() + i * kHeaderCols);
  return out;
}

static void check_header_rows(const at::Tensor& headers, int64_t N, const char* op) {
  TORCH_CHECK(!headers.is_cuda() && headers.scalar_type() == at::kLong && headers.is_contiguous() &&
                  headers.dim() == 2 && headers.size(0) == N && headers.size(1) == kHeaderCols,
              op, ": headers must be jpeg_scan's CPU int64 [N, ", kHeaderCols, "] rows");
}

// One stream-JPEG file's quantised coefficients int16 [blocks, 64] and its components' tables int32 [ncomp, 64].
static std::tuple<at::Tensor, at::Tensor> jpeg_entropy_decode(const std::string& path, const at::Tensor& header) {
  check_header_rows(header.view({1, -1}), 1, "jpeg_entropy_decode");
  const b200::ImageHeader h = header_from_row(header.data_ptr<int64_t>());
  TORCH_CHECK(h.kind == b200::kFileJpeg, "jpeg_entropy_decode: ", path, " is not a file the stream decoder takes");
  at::Tensor coef = at::empty({h.blocks, 64}, at::kShort);
  at::Tensor quant = at::zeros({h.ncomp, 64}, at::kInt);
  {
    py::gil_scoped_release nogil;
    b200::jpeg_entropy_decode(path, h, coef.data_ptr<int16_t>(), quant.data_ptr<int32_t>());
  }
  return {coef, quant};
}

// The stream pipeline's prefetcher: BatchPrefetcher over a split that is never cached.  Its ring: ring_geom,
// ring_par, ring_lab as for a ragged split, and per slot ring_coef int16 [coef_cap], ring_quant int32
// [mb * 3][64], ring_raw uint8 [raw_cap] and ring_desc int32 [mb][kJpegDesc].  `other` holds the RGB of the
// files PIL decoded at start-up, file i at other_off[i] (-1 for the files decoded per batch).
struct PyStreamPrefetcher {
  b200::BatchPrefetcher* p = nullptr;
  b200::StreamConfig sc;
  at::Tensor labels, hw, other, other_off, ring_coef, ring_quant, ring_raw, ring_desc, ring_geom, ring_par, ring_lab;
  PyStreamPrefetcher(std::vector<std::string> paths, const at::Tensor& headers, at::Tensor labels_, at::Tensor hw_,
                     at::Tensor other_, at::Tensor other_off_, at::Tensor ring_coef_, at::Tensor ring_quant_,
                     at::Tensor ring_raw_, at::Tensor ring_desc_, at::Tensor ring_geom_, at::Tensor ring_par_,
                     at::Tensor ring_lab_, bool train, double scale_lo, double scale_hi, double ratio_lo,
                     double ratio_hi, double degrees, int64_t resize, int64_t threads)
      : labels(labels_), hw(hw_), other(other_), other_off(other_off_), ring_coef(ring_coef_), ring_quant(ring_quant_),
        ring_raw(ring_raw_), ring_desc(ring_desc_), ring_geom(ring_geom_), ring_par(ring_par_), ring_lab(ring_lab_) {
    const int64_t N = (int64_t)paths.size();
    check_header_rows(headers, N, "StreamPrefetcher");
    auto cpu = [](const at::Tensor& t, at::ScalarType dt) { return !t.is_cuda() && t.scalar_type() == dt && t.is_contiguous(); };
    TORCH_CHECK(cpu(labels, at::kLong) && labels.numel() == N && cpu(hw, at::kLong) && hw.numel() == 2 * N &&
                    cpu(other, at::kByte) && cpu(other_off, at::kLong) && other_off.numel() == N,
                "StreamPrefetcher: labels int64 [N], hw int64 [N, 2], other uint8, other_off int64 [N]");
    TORCH_CHECK(cpu(ring_par, at::kFloat) && ring_par.dim() == 3 && ring_par.size(2) == 8 && cpu(ring_lab, at::kLong) &&
                    ring_lab.dim() == 2 && ring_lab.sizes() == ring_par.sizes().slice(0, 2),
                "StreamPrefetcher: ring_par [slots][mb][8] and ring_lab [slots][mb]");
    const int64_t slots = ring_par.size(0), mb = ring_par.size(1);
    TORCH_CHECK(cpu(ring_geom, at::kLong) && ring_geom.dim() == 3 && ring_geom.size(0) == slots &&
                    ring_geom.size(1) == mb && ring_geom.size(2) == 5, "StreamPrefetcher: ring_geom int64 [slots][mb][5]");
    TORCH_CHECK(cpu(ring_coef, at::kShort) && ring_coef.dim() == 2 && ring_coef.size(0) == slots &&
                    cpu(ring_raw, at::kByte) && ring_raw.dim() == 2 && ring_raw.size(0) == slots &&
                    cpu(ring_quant, at::kInt) && ring_quant.dim() == 3 && ring_quant.size(0) == slots &&
                    ring_quant.size(1) == mb * 3 && ring_quant.size(2) == 64 && cpu(ring_desc, at::kInt) &&
                    ring_desc.dim() == 3 && ring_desc.size(0) == slots && ring_desc.size(1) == mb &&
                    ring_desc.size(2) == b200::kJpegDesc,
                "StreamPrefetcher: ring_coef int16 [slots][cap], ring_raw uint8 [slots][cap], ring_quant int32 "
                "[slots][mb*3][64], ring_desc int32 [slots][mb][", b200::kJpegDesc, "]");
    const int64_t* hr = headers.data_ptr<int64_t>();
    const int64_t* s = hw.data_ptr<int64_t>();
    const int64_t* oo = other_off.data_ptr<int64_t>();
    std::vector<int64_t> coef_sizes, raw_sizes;
    sc.paths = std::move(paths);
    sc.headers.resize(N);
    for (int64_t i = 0; i < N; ++i) {
      const b200::ImageHeader h = header_from_row(hr + i * kHeaderCols);
      sc.headers[i] = h;
      const int64_t H = s[2 * i], W = s[2 * i + 1];
      TORCH_CHECK(H >= 1 && W >= 1 && H <= 65535 && W <= 65535, "StreamPrefetcher: image ", i, " has size ", H, " x ", W);
      if (h.kind == b200::kFileOther) {
        TORCH_CHECK(oo[i] >= 0 && oo[i] + H * W * 3 <= other.numel(), "StreamPrefetcher: image ", i,
                    " lies outside the start-up cache");
      } else {
        TORCH_CHECK(h.H == H && h.W == W, "StreamPrefetcher: image ", i, "'s size differs from its header");
      }
      if (h.kind == b200::kFileJpeg) {
        int64_t want = 0;
        for (int c = 0; c < h.ncomp; ++c) {
          int bw, bh;
          b200::jpeg_block_grid(h, c, bw, bh);
          want += (int64_t)bw * bh;
        }
        TORCH_CHECK(h.blocks == want && (h.ncomp == 1 || h.ncomp == 3), "StreamPrefetcher: image ", i,
                    " has an inconsistent header row");
        coef_sizes.push_back(h.blocks * 64);
      } else {
        raw_sizes.push_back(H * W * 3);
      }
    }
    // a slot must hold any batch: the coefficients of the mb largest JPEGs and the RGB of the mb largest others
    for (auto* v : {&coef_sizes, &raw_sizes}) std::sort(v->begin(), v->end(), std::greater<int64_t>());
    int64_t coef_need = 0, raw_need = 0, blocks_need = 0;
    for (int64_t i = 0; i < std::min<int64_t>(mb, coef_sizes.size()); ++i) coef_need += coef_sizes[i];
    for (int64_t i = 0; i < std::min<int64_t>(mb, raw_sizes.size()); ++i) raw_need += raw_sizes[i];
    blocks_need = coef_need / 64;
    TORCH_CHECK(ring_coef.size(1) >= coef_need && ring_raw.size(1) >= raw_need && blocks_need < (1ll << 31) &&
                    raw_need < (1ll << 31), "StreamPrefetcher: a slot of ", ring_coef.size(1), " coefficients and ",
                ring_raw.size(1), " raw bytes cannot hold ", coef_need, " and ", raw_need);
    sc.other = other.data_ptr<uint8_t>(); sc.other_off = oo;
    sc.ring_coef = ring_coef.data_ptr<int16_t>(); sc.coef_cap = ring_coef.size(1);
    sc.ring_quant = ring_quant.data_ptr<int32_t>();
    sc.ring_raw = ring_raw.data_ptr<uint8_t>(); sc.raw_cap = ring_raw.size(1);
    sc.ring_desc = ring_desc.data_ptr<int32_t>();
    sc.threads = (int)std::max<int64_t>(1, threads);
    b200::PrefetchConfig c;
    c.cache = nullptr; c.labels = labels.data_ptr<int64_t>();
    c.H = 0; c.W = 0; c.mb = (int)mb; c.slots = (int)slots;
    c.ring_img = nullptr; c.ring_par = ring_par.data_ptr<float>(); c.ring_lab = ring_lab.data_ptr<int64_t>();
    c.train = train; c.scale_lo = (float)scale_lo; c.scale_hi = (float)scale_hi;
    c.ratio_lo = (float)ratio_lo; c.ratio_hi = (float)ratio_hi; c.degrees = (float)degrees;
    c.hw = s; c.ring_geom = ring_geom.data_ptr<int64_t>(); c.resize = (int)resize;
    c.stream = &sc;
    p = b200::prefetcher_create(c);
  }
  ~PyStreamPrefetcher() { if (p) b200::prefetcher_destroy(p); }
  void start(std::vector<int64_t> idx, uint64_t seed) {
    for (int64_t i : idx) TORCH_CHECK(i >= 0 && i < (int64_t)sc.paths.size(), "StreamPrefetcher: index ", i, " out of range");
    py::gil_scoped_release nogil;
    b200::prefetcher_start(p, std::move(idx), seed);
  }
  py::object next() {
    int slot = -1, count = 0;
    bool ok;
    {
      py::gil_scoped_release nogil;
      ok = b200::prefetcher_next(p, slot, count);
    }
    if (!ok) return py::none();
    return py::make_tuple(slot, count);
  }
  void release(int64_t slot, uint64_t ev) { b200::prefetcher_release(p, (int)slot, ev); }
  void stop() {
    py::gil_scoped_release nogil;
    b200::prefetcher_stop(p);
  }
};

// The device decode of a stream batch.  The kernels read desc and geom on the device; the host copies they were
// made from are checked here, so that no row can send a launch outside coef, quant, raw, planes or out.
static void jpeg_decode(const at::Tensor& coef, const at::Tensor& quant, const at::Tensor& desc, const at::Tensor& geom,
                        const at::Tensor& raw, at::Tensor planes, at::Tensor out, const at::Tensor& desc_host,
                        const at::Tensor& geom_host) {
  c10::cuda::CUDAGuard g(out.device());
  auto dev = [](const at::Tensor& t, at::ScalarType dt) { return t.is_cuda() && t.scalar_type() == dt && t.is_contiguous(); };
  TORCH_CHECK(dev(desc, at::kInt) && desc.dim() == 2 && desc.size(1) == b200::kJpegDesc,
              "jpeg_decode: desc must be a contiguous CUDA int32 [k, ", b200::kJpegDesc, "] tensor");
  const int64_t k = desc.size(0);
  TORCH_CHECK(k >= 1 && k <= 65535, "jpeg_decode: 1 to 65535 images");
  TORCH_CHECK(dev(geom, at::kLong) && geom.dim() == 2 && geom.size(0) == k && geom.size(1) == 5,
              "jpeg_decode: geom must be a contiguous CUDA int64 [k, 5] tensor");
  TORCH_CHECK(!desc_host.is_cuda() && desc_host.scalar_type() == at::kInt && desc_host.is_contiguous() &&
                  desc_host.sizes() == desc.sizes(), "jpeg_decode: desc_host must be the CPU int32 copy of desc");
  TORCH_CHECK(!geom_host.is_cuda() && geom_host.scalar_type() == at::kLong && geom_host.is_contiguous() &&
                  geom_host.sizes() == geom.sizes(), "jpeg_decode: geom_host must be the CPU int64 copy of geom");
  TORCH_CHECK(dev(coef, at::kShort) && dev(quant, at::kInt) && quant.dim() == 2 && quant.size(1) == 64 &&
                  dev(raw, at::kByte) && dev(planes, at::kByte) && dev(out, at::kByte),
              "jpeg_decode: coef int16, quant int32 [rows, 64], raw, planes and out uint8, all contiguous CUDA tensors");
  TORCH_CHECK(reinterpret_cast<uintptr_t>(planes.data_ptr()) % 8 == 0, "jpeg_decode: planes must be 8-byte aligned");
  for (const at::Tensor* t : std::initializer_list<const at::Tensor*>{&coef, &quant, &desc, &geom, &raw, &planes})
    TORCH_CHECK(t->device() == out.device(), "jpeg_decode: every operand on out's device");
  const int32_t* d = desc_host.data_ptr<int32_t>();
  const int64_t* gh = geom_host.data_ptr<int64_t>();
  int64_t blocks = 0, most = 1;
  for (int64_t i = 0; i < k; ++i) {
    const int32_t* r = d + i * b200::kJpegDesc;
    const int64_t off = gh[i * 5], H = gh[i * 5 + 1], W = gh[i * 5 + 2];
    TORCH_CHECK(H >= 1 && W >= 1 && H <= 65535 && W <= 65535 && off >= 0 && off + H * W * 3 <= out.numel(),
                "jpeg_decode: image ", i, " (offset ", off, ", ", H, " x ", W, ") lies outside out of ", out.numel(),
                " bytes");
    TORCH_CHECK(r[3] == blocks, "jpeg_decode: image ", i, " starts at block ", r[3], ", the batch is at ", blocks);
    most = std::max(most, H * W);
    const int n = r[0];
    if (n == 0) {
      TORCH_CHECK(r[4] >= 0 && r[4] + H * W * 3 <= raw.numel(), "jpeg_decode: image ", i, " lies outside raw");
      continue;
    }
    b200::ImageHeader h;
    h.H = (int)H; h.W = (int)W; h.ncomp = n;
    h.h[0] = r[1]; h.v[0] = r[2]; h.h[1] = h.v[1] = h.h[2] = h.v[2] = 1;
    const bool sampling = n == 1 ? r[1] == 1 && r[2] == 1
                                 : (r[1] == 1 && r[2] == 1) || (r[1] == 2 && r[2] == 1) || (r[1] == 2 && r[2] == 2);
    TORCH_CHECK((n == 1 || n == 3) && sampling, "jpeg_decode: image ", i, " has ", n, " components sampled ", r[1],
                "x", r[2]);
    for (int c = 0; c < n; ++c) {
      int bw, bh;
      b200::jpeg_block_grid(h, c, bw, bh);
      TORCH_CHECK(r[5 + c] == bw && r[8 + c] == bh, "jpeg_decode: image ", i, " component ", c, " has a ", r[5 + c],
                  " x ", r[8 + c], " block grid, its geometry needs ", bw, " x ", bh);
      TORCH_CHECK(r[11 + c] >= 0 && r[11 + c] < quant.size(0), "jpeg_decode: image ", i, " component ", c,
                  " reads quantisation row ", r[11 + c], " of ", quant.size(0));
      blocks += (int64_t)bw * bh;
    }
  }
  TORCH_CHECK(blocks * 64 <= coef.numel() && blocks * 64 <= planes.numel(), "jpeg_decode: ", blocks,
              " blocks do not fit coef (", coef.numel(), ") or planes (", planes.numel(), ")");
  const int64_t cap = std::max<int64_t>(1, 16 * b200::sm_count() / k);
  const int grid_x = (int)std::min(cap, (most + 255) / 256);
  b200::jpeg_decode(coef.data_ptr<int16_t>(), quant.data_ptr<int32_t>(), desc.data_ptr<int32_t>(),
                    reinterpret_cast<const long long*>(geom.data_ptr<int64_t>()), raw.data_ptr<uint8_t>(),
                    planes.data_ptr<uint8_t>(), out.data_ptr<uint8_t>(), (int)k, blocks, grid_x, cur_stream());
}

// ------------------------------------------------------------------------------------------- comm
// The collectives write into every peer's wire buffer and signal pad: a range past the wire or a slot
// past the pad lands in another GPU's memory.  Every binding below refuses such operands before it
// launches anything.
struct PyComm {
  b200::CommCtx c;
  int64_t wire_bytes;   // size of each rank's wire buffer
  int64_t slots;        // barrier groups of each rank's signal pad (allreduce_signal_words(slots) words)
};
static PyComm make_comm(int64_t rank, int64_t world, int64_t wire_ptrs_dev, int64_t signal_ptrs_dev,
                        int64_t wire_mc, int64_t signal_mc, int64_t wire_bytes, int64_t slots) {
  TORCH_CHECK(world >= 1 && world <= b200::AR_MAX_WORLD, "make_comm: world must be in [1, ", b200::AR_MAX_WORLD,
              "], got ", world);
  TORCH_CHECK(rank >= 0 && rank < world, "make_comm: rank ", rank, " is not in [0, ", world, ")");
  TORCH_CHECK(wire_bytes >= 0 && slots >= 1, "make_comm: a wire of >= 0 bytes and at least one slot");
  PyComm p;
  p.wire_bytes = wire_bytes; p.slots = slots;
  p.c.rank = (int)rank; p.c.world = (int)world;
  p.c.wire_ptrs = reinterpret_cast<void* const*>(wire_ptrs_dev);
  p.c.signal_ptrs = reinterpret_cast<uint32_t* const*>(signal_ptrs_dev);
  p.c.wire_mc = reinterpret_cast<void*>(wire_mc);
  p.c.signal_mc = reinterpret_cast<uint32_t*>(signal_mc);
  // cross-GPU waits are bounded by wall clock; minutes by default so that host-side skew (rank 0
  // writing a checkpoint, a slow loader) never trips it -- only a dead peer does
  double secs = 600.0;
  if (const char* e = std::getenv("B200_BARRIER_TIMEOUT_S")) secs = std::atof(e) > 0 ? std::atof(e) : secs;
  p.c.timeout_ns = static_cast<unsigned long long>(secs * 1e9);
  return p;
}
// [start, start+n) of elements of `elem_bytes` inside the wire, and a slot inside the signal pad
static void check_comm_range(const PyComm& comm, int64_t start, int64_t n, int64_t elem_bytes, int64_t slot,
                             const char* op) {
  TORCH_CHECK(start >= 0 && n >= 0, op, ": start and n must be >= 0");
  TORCH_CHECK((start + n) * elem_bytes <= comm.wire_bytes, op, ": [", start, ", ", start + n, ") of ", elem_bytes,
              "-byte elements runs past the ", comm.wire_bytes, "-byte wire");
  TORCH_CHECK(slot >= 0 && slot < comm.slots, op, ": slot ", slot, " is not in [0, ", comm.slots, ")");
}
// an arena (gradient, optimizer state or shadow) the kernels address at [start, start+n) with 16-byte vectors
static void check_arena(const at::Tensor& t, at::ScalarType dt, int64_t start, int64_t n, const char* op,
                        const char* name) {
  check_vec(t, dt, 16, op, name);
  TORCH_CHECK(t.numel() >= start + n, op, ": ", name, " must hold start + n = ", start + n, " elements, got ",
              t.numel());
}
static void allreduce(const PyComm& comm, c10::optional<at::Tensor> grad, c10::optional<at::Tensor> grad_out,
                      int64_t start, int64_t n, double inv_world, int64_t algo, bool wire_fp32, int64_t slot,
                      int64_t epoch, int64_t max_ctas) {
  check_comm_range(comm, start, n, wire_fp32 ? 4 : 2, slot, "allreduce");
  if (grad.has_value()) check_arena(*grad, at::kFloat, start, n, "allreduce", "grad");
  if (grad_out.has_value()) check_arena(*grad_out, at::kFloat, start, n, "allreduce", "grad_out");
  b200::allreduce_fused(comm.c, f32p_opt(grad), f32p_opt(grad_out), start, n, (float)inv_world, (int)algo,
                        wire_fp32, (int)slot, (uint32_t)epoch, (int)max_ctas, cur_stream());
}
// EXPERIMENTAL (--zero1): fused reduce-scatter + Adam on the owned cells + all-gather of bf16 weights
static void zero1_step(const PyComm& comm, c10::optional<at::Tensor> grad, at::Tensor p, at::Tensor m, at::Tensor v,
                       at::Tensor shadow, int64_t start, int64_t n, double inv_world, int64_t algo, int64_t slot,
                       int64_t epoch, int64_t max_ctas, double lr, double beta1, double beta2, double eps,
                       double weight_decay, int64_t step, c10::optional<at::Tensor> ema, double ema_decay,
                       bool ema_first, bool decoupled) {
  TORCH_CHECK(p.scalar_type() == at::kFloat && m.scalar_type() == at::kFloat && v.scalar_type() == at::kFloat &&
                  shadow.scalar_type() == at::kBFloat16 && p.numel() == m.numel() && p.numel() == v.numel() &&
                  p.numel() == shadow.numel() && start + n <= p.numel(),
              "zero1_step: full fp32 arenas (p, m, v) and the bf16 shadow of the same length");
  check_comm_range(comm, start, n, 2, slot, "zero1_step");
  if (grad.has_value()) check_arena(*grad, at::kFloat, start, n, "zero1_step", "grad");
  for (auto* t : {&p, &m, &v}) check_arena(*t, at::kFloat, start, n, "zero1_step", "p, m and v");
  check_arena(shadow, at::kBFloat16, start, n, "zero1_step", "shadow");
  if (ema.has_value()) {
    check_arena(*ema, at::kFloat, start, n, "zero1_step", "ema");
    TORCH_CHECK(ema->numel() == p.numel(), "zero1_step: ema must have p's size");
    TORCH_CHECK(ema_decay >= 0.0 && ema_decay <= 1.0, "zero1_step: ema_decay must lie in [0, 1], got ", ema_decay);
  }
  TORCH_CHECK(!decoupled || (std::isfinite(weight_decay) && weight_decay >= 0.0),
              "zero1_step: the AdamW weight decay must be finite and >= 0, got ", weight_decay);
  const b200::OptStep o =
      b200::make_opt_step("zero1_step", decoupled ? b200::OPT_ADAMW : b200::OPT_ADAM, n, lr, beta1, beta2, eps, 0.0,
                          (int)step, false, 1.0, weight_decay, {}, {}, ema_decay, ema_first);
  b200::zero1_step(comm.c, o, grad.has_value() ? grad->data_ptr<float>() : nullptr, p.data_ptr<float>(),
                   m.data_ptr<float>(), v.data_ptr<float>(), bfp_mut(shadow), f32p_opt(ema), start, n,
                   (float)inv_world, (int)algo, (int)slot, (uint32_t)epoch, (int)max_ctas, cur_stream());
}
static int64_t allreduce_grid(int64_t n, int64_t world, int64_t max_ctas, bool wire_fp32) {
  return b200::allreduce_grid(n, (int)world, (int)max_ctas, wire_fp32);
}
static void broadcast(const PyComm& comm, at::Tensor data, int64_t root, int64_t slot, int64_t epoch) {
  check_vec(data, at::kFloat, 16, "broadcast", "data");
  check_comm_range(comm, 0, data.numel(), 4, slot, "broadcast");
  TORCH_CHECK(root >= 0 && root < comm.c.world, "broadcast: root ", root, " is not in [0, ", comm.c.world, ")");
  b200::broadcast_fused(comm.c, f32p(data), data.numel(), (int)root, (int)slot, (uint32_t)epoch, cur_stream());
}
static void barrier(const PyComm& comm, int64_t slot, int64_t epoch) {
  check_comm_range(comm, 0, 0, 1, slot, "barrier");
  b200::device_barrier(comm.c, (int)slot, (uint32_t)epoch, cur_stream());
}

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.doc() = "distributed-vgg-f_b200 native sm_90a kernels";
  m.def("launch_count", &b200::launch_count);
  m.def("decode_pngs", &decode_pngs);
  m.def("decode_pngs_into", &decode_pngs_into);
  m.def("gemm", &gemm);
  m.def("conv0_fprop", &conv0_fprop);
  m.def("conv0_wgrad", &conv0_wgrad);
  m.def("conv_fprop", &conv_fprop);
  m.def("conv_fprop_pool", &conv_fprop_pool);
  m.def("conv_pool_fusable", &conv_pool_fusable);
  m.def("conv_pixel_box", &conv_pixel_box);
  m.def("conv_plan", &conv_plan, py::arg("kind"), py::arg("N"), py::arg("H"), py::arg("W"), py::arg("Cin"),
        py::arg("Cout"), py::arg("sms"), py::arg("bn") = 0);
  m.def("conv_bn_choice", &conv_bn_choice);
  m.def("unpool2x2", &unpool);
  m.def("conv_dgrad", &conv_dgrad);
  m.def("conv_wgrad", &conv_wgrad);
  m.def("gemm_partial", &gemm_partial);
  m.def("conv_wgrad_partial", &conv_wgrad_partial);
  m.def("conv0_wgrad_partial", &conv0_wgrad_partial);
  m.def("colsum_partial", &colsum_partial);
  m.def("splitk_reduce", &splitk_reduce);
  m.def("conv_wgrad_splits", [](int64_t N, int64_t H, int64_t W, int64_t Cin, int64_t Cout, int64_t sms) {
    return b200::conv_wgrad_splits((int)N, (int)H, (int)W, (int)Cin, (int)Cout, (int)sms); });
  m.def("conv0_wgrad_splits", [](int64_t N, int64_t H, int64_t W, int64_t sms) {
    return b200::conv0_wgrad_splits((int)N, (int)H, (int)W, (int)sms); });
  m.def("gemm_splits", [](int64_t K, int64_t ksplit) { return b200::gemm_splits((int)K, (int)ksplit); });
  m.def("colsum_partial_blocks", [](int64_t rows, int64_t C, int64_t sms) {
    return b200::colsum_partial_blocks(rows, (int)C, (int)sms); });
  m.def("workspace_slice", [](int64_t elems) { return (int64_t)b200::workspace_slice(elems); });
  m.def("sm_count", [] { return b200::sm_count(); });
  m.def("maxpool_fwd", &maxpool_fwd);
  m.def("maxpool_relu_bwd", &maxpool_relu_bwd);
  m.def("avgpool_fwd", &avgpool_fwd);
  m.def("avgpool_bwd", &avgpool_bwd);
  m.def("bias_grad", &bias_grad);
  m.def("fc_bias_act", &fc_bias_act);
  m.def("fc_grad_act", &fc_grad_act);
  m.def("cast_to_bf16", &cast_to_bf16);
  m.def("cast_to_f32", &cast_to_f32);
  m.def("cross_entropy", &cross_entropy);
  m.def("cross_entropy_soft", &cross_entropy_soft);
  m.def("cross_entropy_kd", &cross_entropy_kd, py::arg("logits"), py::arg("target"), py::arg("dlogits"), py::arg("ldd"),
        py::arg("meter"), py::arg("loss_out"), py::arg("grad_scale"), py::arg("class_weights"), py::arg("teacher"),
        py::arg("alpha"), py::arg("temperature"), py::arg("soft") = py::none());
  m.def("head_ce_supported", [](int64_t B, int64_t C, int64_t K) { return b200::head_ce_supported((int)B, (int)C, (int)K); });
  m.def("head_ce", [](const at::Tensor& h, const at::Tensor& W, const at::Tensor& bias, const at::Tensor& target,
                      at::Tensor logits, c10::optional<at::Tensor> dlogits, int64_t ldd, c10::optional<at::Tensor> dW,
                      c10::optional<at::Tensor> db, c10::optional<at::Tensor> dh, double drop_scale, bool relu,
                      c10::optional<at::Tensor> meter, c10::optional<at::Tensor> loss_out,
                      c10::optional<at::Tensor> class_weights, bool accumulate,
                      c10::optional<std::vector<double>> soft) {
    c10::cuda::CUDAGuard g(h.device());
    check_head_ce("head_ce", h, W, bias, target, logits, dlogits, ldd, dW, db, dh, drop_scale, relu, meter, loss_out,
                  class_weights);
    TORCH_CHECK(!soft.has_value() || soft->size() == 3, "head_ce: soft is (eps, lam, mix)");
    b200::SoftTargets st{};
    if (soft.has_value()) st = soft_targets("head_ce", (*soft)[0], (*soft)[1], (*soft)[2] != 0.0);
    b200::head_ce_fused(bfp(h), bfp(W), f32p(bias), reinterpret_cast<const long long*>(target.data_ptr()), f32p(logits),
                        dlogits.has_value() ? bfp_mut(*dlogits) : nullptr, (int)ldd, f32p_opt(dW), f32p_opt(db),
                        dh.has_value() ? bfp_mut(*dh) : nullptr, (float)drop_scale, relu, f32p_opt(meter),
                        f32p_opt(loss_out), (int)h.size(0), (int)W.size(0), (int)h.size(1), f32p_opt(class_weights),
                        accumulate, cur_stream(), soft.has_value() ? &st : nullptr);
  },
  // accumulate: dW += the batch's gradient instead of dW = (later micro-batches of an accumulation group)
  py::arg("h"), py::arg("W"), py::arg("bias"), py::arg("target"), py::arg("logits"), py::arg("dlogits"), py::arg("ldd"),
  py::arg("dW"), py::arg("db"), py::arg("dh"), py::arg("drop_scale"), py::arg("relu"), py::arg("meter"),
  py::arg("loss_out"), py::arg("class_weights"), py::arg("accumulate") = false,
  // soft = (eps, lam, mix): label smoothing and MixUp / CutMix targets (cross_entropy_soft); None: integer labels
  py::arg("soft") = py::none());
  // head_ce with the distillation loss against teacher logits [B][C] fp32 (see cross_entropy_kd)
  m.def("head_ce_kd", [](const at::Tensor& h, const at::Tensor& W, const at::Tensor& bias, const at::Tensor& target,
                         at::Tensor logits, c10::optional<at::Tensor> dlogits, int64_t ldd, c10::optional<at::Tensor> dW,
                         c10::optional<at::Tensor> db, c10::optional<at::Tensor> dh, double drop_scale, bool relu,
                         c10::optional<at::Tensor> meter, c10::optional<at::Tensor> loss_out,
                         c10::optional<at::Tensor> class_weights, bool accumulate,
                         c10::optional<std::vector<double>> soft, const at::Tensor& teacher, double alpha,
                         double temperature) {
    c10::cuda::CUDAGuard g(h.device());
    check_head_ce("head_ce_kd", h, W, bias, target, logits, dlogits, ldd, dW, db, dh, drop_scale, relu, meter, loss_out,
                  class_weights);
    const b200::KdParams kd = check_kd("head_ce_kd", teacher, h.device(), h.size(0), W.size(0), alpha, temperature);
    const b200::SoftTargets st = soft_list("head_ce_kd", soft);
    b200::head_ce_kd_fused(bfp(h), bfp(W), f32p(bias), reinterpret_cast<const long long*>(target.data_ptr()),
                           f32p(logits), dlogits.has_value() ? bfp_mut(*dlogits) : nullptr, (int)ldd, f32p_opt(dW),
                           f32p_opt(db), dh.has_value() ? bfp_mut(*dh) : nullptr, (float)drop_scale, relu,
                           f32p_opt(meter), f32p_opt(loss_out), (int)h.size(0), (int)W.size(0), (int)h.size(1),
                           f32p_opt(class_weights), accumulate, soft.has_value() ? &st : nullptr, f32p(teacher), kd,
                           cur_stream());
  },
  py::arg("h"), py::arg("W"), py::arg("bias"), py::arg("target"), py::arg("logits"), py::arg("dlogits"), py::arg("ldd"),
  py::arg("dW"), py::arg("db"), py::arg("dh"), py::arg("drop_scale"), py::arg("relu"), py::arg("meter"),
  py::arg("loss_out"), py::arg("class_weights"), py::arg("accumulate"), py::arg("soft"), py::arg("teacher"),
  py::arg("alpha"), py::arg("temperature"));
  m.def("adam", &adam, py::arg("p"), py::arg("m"), py::arg("v"), py::arg("g32"), py::arg("g16"), py::arg("shadow"),
        py::arg("lr"), py::arg("b1"), py::arg("b2"), py::arg("eps"), py::arg("wd"), py::arg("step"),
        py::arg("grad_scale"), py::arg("gzero"), py::arg("ema") = py::none(), py::arg("ema_decay") = 0.0,
        py::arg("ema_first") = false, py::arg("decoupled") = false, py::arg("wd_starts") = std::vector<int64_t>(),
        py::arg("wd_values") = std::vector<double>());
  m.def("sgd", &sgd, py::arg("p"), py::arg("mom"), py::arg("g32"), py::arg("g16"), py::arg("shadow"), py::arg("lr"),
        py::arg("momentum"), py::arg("wd"), py::arg("first"), py::arg("grad_scale"), py::arg("gzero"),
        py::arg("ema") = py::none(), py::arg("ema_decay") = 0.0, py::arg("ema_first") = false,
        py::arg("wd_starts") = std::vector<int64_t>(), py::arg("wd_values") = std::vector<double>());
  m.def("ema_update", &ema_update, py::arg("p"), py::arg("ema"), py::arg("decay"), py::arg("first"));
  m.def("layerwise", &layerwise, py::arg("phase"), py::arg("kind"), py::arg("p"), py::arg("m"), py::arg("v"),
        py::arg("g32"), py::arg("g16"), py::arg("shadow"), py::arg("gzero"), py::arg("ema"), py::arg("ws"),
        py::arg("ratio"), py::arg("lr"), py::arg("b1"), py::arg("b2"), py::arg("eps"), py::arg("momentum"),
        py::arg("step"), py::arg("first"), py::arg("grad_scale"), py::arg("ema_decay"), py::arg("ema_first"),
        py::arg("starts"), py::arg("ctas"), py::arg("slots"), py::arg("nslots"), py::arg("tensors"), py::arg("wds"),
        py::arg("trust_coeff"), py::arg("trust_eps"));
  m.def("layerwise_max_segments", [] { return b200::LW_MAX_SEGMENTS; });
  m.def("psgd_project", &psgd_project, py::arg("g"), py::arg("e"), py::arg("q"), py::arg("p"), py::arg("n"),
        py::arg("m"), py::arg("rank"), py::arg("scale"));
  m.def("psgd_backproject", &psgd_backproject, py::arg("M"), py::arg("p"), py::arg("q"), py::arg("ws"), py::arg("n"),
        py::arg("m"), py::arg("rank"));
  m.def("psgd_orthogonalize", &psgd_orthogonalize, py::arg("x"), py::arg("rows"), py::arg("rank"),
        py::arg("count") = 1);
  m.def("psgd_decompress", &psgd_decompress, py::arg("p"), py::arg("q"), py::arg("g"), py::arg("e"), py::arg("n"),
        py::arg("m"), py::arg("rank"), py::arg("alpha"));
  // host arithmetic of the back-projection's row splits (no GPU needed): the workspace a launch needs
  m.def("psgd_workspace_elems", [](int64_t n, int64_t m, int64_t rank, int64_t sms) {
    return (int64_t)b200::psgd_workspace_elems((int)n, (int)m, (int)rank, (int)sms);
  });
  m.attr("PSGD_MAX_RANK") = b200::PSGD_MAX_RANK;
  m.def("augment", &augment);
  m.def("augment_mixed", &augment_mixed);
  m.def("augment_ragged", &augment_ragged);
  m.def("augment_ragged_mixed", &augment_ragged_mixed);
  m.def("ragged_inter_bytes", &ragged_inter_bytes);
  m.def("augment_view", &augment_view);
  m.def("augment_ragged_view", &augment_ragged_view);
  m.def("tta_accumulate", &tta_accumulate);
  m.def("class_metrics", &class_metrics);
  m.attr("TTA_FLIP") = (int)b200::TtaFlip;
  m.def("im2col_c3", &im2col_c3);
  m.def("nchw_to_nhwc", &nchw_to_nhwc);
  py::class_<PyPrefetcher>(m, "Prefetcher")
      .def(py::init<at::Tensor, at::Tensor, at::Tensor, at::Tensor, at::Tensor, bool, double, double, double, double, double,
                    c10::optional<at::Tensor>, c10::optional<at::Tensor>, c10::optional<at::Tensor>, int64_t>(),
           py::arg("cache"), py::arg("labels"), py::arg("ring_img"), py::arg("ring_par"), py::arg("ring_lab"),
           py::arg("train"), py::arg("scale_lo"), py::arg("scale_hi"), py::arg("ratio_lo"), py::arg("ratio_hi"),
           py::arg("degrees"), py::arg("offsets") = py::none(), py::arg("hw") = py::none(),
           py::arg("ring_geom") = py::none(), py::arg("resize") = 256)
      .def("start", &PyPrefetcher::start)
      .def("next", &PyPrefetcher::next)
      .def("release", &PyPrefetcher::release)
      .def("stop", &PyPrefetcher::stop);
  m.def("jpeg_scan", &jpeg_scan, py::arg("paths"), py::arg("threads"));
  m.def("png_decodable", &png_decodable, py::arg("paths"), py::arg("hw"), py::arg("threads"));
  m.def("jpeg_entropy_decode", &jpeg_entropy_decode, py::arg("path"), py::arg("header"));
  m.def("jpeg_decode", &jpeg_decode, py::arg("coef"), py::arg("quant"), py::arg("desc"), py::arg("geom"), py::arg("raw"),
        py::arg("planes"), py::arg("out"), py::arg("desc_host"), py::arg("geom_host"));
  m.attr("JPEG_DESC") = b200::kJpegDesc;
  py::class_<PyStreamPrefetcher>(m, "StreamPrefetcher")
      .def(py::init<std::vector<std::string>, const at::Tensor&, at::Tensor, at::Tensor, at::Tensor, at::Tensor,
                    at::Tensor, at::Tensor, at::Tensor, at::Tensor, at::Tensor, at::Tensor, at::Tensor, bool, double,
                    double, double, double, double, int64_t, int64_t>(),
           py::arg("paths"), py::arg("headers"), py::arg("labels"), py::arg("hw"), py::arg("other"),
           py::arg("other_off"), py::arg("ring_coef"), py::arg("ring_quant"), py::arg("ring_raw"),
           py::arg("ring_desc"), py::arg("ring_geom"), py::arg("ring_par"), py::arg("ring_lab"), py::arg("train"),
           py::arg("scale_lo"), py::arg("scale_hi"), py::arg("ratio_lo"), py::arg("ratio_hi"), py::arg("degrees"),
           py::arg("resize"), py::arg("threads"))
      .def("start", &PyStreamPrefetcher::start)
      .def("next", &PyStreamPrefetcher::next)
      .def("release", &PyStreamPrefetcher::release)
      .def("stop", &PyStreamPrefetcher::stop);
  py::class_<PyComm>(m, "Comm");
  m.def("probe_background", [](at::Tensor buf, int64_t mode, int64_t ctas, int64_t reps, at::Tensor sink) {
    b200::probe_background(f32p(buf), buf.numel(), (int)mode, (int)ctas, (int)reps, f32p(sink), cur_stream());
  });
  m.def("make_comm", &make_comm);
  m.def("allreduce", &allreduce);
  m.def("zero1_step", &zero1_step, py::arg("comm"), py::arg("grad"), py::arg("p"), py::arg("m"), py::arg("v"),
        py::arg("shadow"), py::arg("start"), py::arg("n"), py::arg("inv_world"), py::arg("algo"), py::arg("slot"),
        py::arg("epoch"), py::arg("max_ctas"), py::arg("lr"), py::arg("beta1"), py::arg("beta2"), py::arg("eps"),
        py::arg("weight_decay"), py::arg("step"), py::arg("ema") = py::none(), py::arg("ema_decay") = 0.0,
        py::arg("ema_first") = false, py::arg("decoupled") = false);
  m.def("wd_max_segments", [] { return b200::WD_MAX_SEGMENTS; });
  m.def("allreduce_grid", &allreduce_grid);
  m.def("broadcast", &broadcast);
  m.def("barrier", &barrier);
  m.def("allreduce_signal_words", &b200::allreduce_signal_words);
  m.attr("EPI_F32_STORE") = 0;
  m.attr("EPI_F32_ATOMIC") = 1;
  m.attr("EPI_F32_ATOMIC_T") = 2;
  m.attr("EPI_BF16_BIAS_RELU") = 3;
  m.attr("EPI_F32_STORE_T") = 4;
  m.attr("EPI_BF16_STORE") = 5;
  m.attr("AR_ONESHOT") = 0;
  m.attr("AR_TWOSHOT") = 1;
  m.attr("AR_NVLS") = 2;
}
