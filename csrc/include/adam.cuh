// The per-element updates of the optimizers (Adam, AdamW, SGD) and of the weights' moving average,
// shared by the optimizer kernels (loss_optim.cu) and zero1_kernel (allreduce.cu) so that the fused
// ZeRO-1 step and the replicated optimizer give the same update bit for bit.  Every rounding is spelled
// out: left to itself, nvcc contracted `g * gscale + wd * p` to fma(g, gscale, wd * p) in one kernel and
// `g + wd * p` to fma(wd, p, g) in the other, and the two differ in the last bit of the moments
// (tests/test_collectives_gpu.py).
#pragma once
#include <cuda_runtime.h>
#include "api.h"

namespace b200 {

// The moments and the step of one Adam update from the (already decayed, scaled) gradient gk.
__device__ __forceinline__ void adam_moments_step(float gk, float& p, float& m, float& v, float lr_bc1, float b1,
                                                  float b2, float eps, float bc2_inv_sqrt) {
  m = __fmaf_rn(b1, m, __fmul_rn(1.f - b1, gk));
  v = __fmaf_rn(b2, v, __fmul_rn(__fmul_rn(1.f - b2, gk), gk));
  const float denom = __fmaf_rn(__fsqrt_rn(v), bc2_inv_sqrt, eps);
  p = __fsub_rn(p, __fdiv_rn(__fmul_rn(lr_bc1, m), denom));
}

// lr_bc1 = lr / (1 - beta1^step), bc2_inv_sqrt = 1 / sqrt(1 - beta2^step), both rounded to fp32 once
__device__ __forceinline__ void adam_update(float g, float gscale, float& p, float& m, float& v, float lr_bc1,
                                            float b1, float b2, float eps, float wd, float bc2_inv_sqrt) {
  adam_moments_step(__fmaf_rn(g, gscale, __fmul_rn(wd, p)), p, m, v, lr_bc1, b1, b2, eps, bc2_inv_sqrt);
}

// One AdamW step (torch.optim.AdamW: decoupled weight decay).  keep = fp32(1 - lr * wd), taken in double
// on the host as torch takes the Python scalar of `p.mul_(1 - lr * weight_decay)`; then Adam on the
// scaled gradient alone, with no L2 term.
__device__ __forceinline__ void adamw_update(float g, float gscale, float& p, float& m, float& v, float lr_bc1,
                                             float b1, float b2, float eps, float keep, float bc2_inv_sqrt) {
  p = __fmul_rn(p, keep);
  adam_moments_step(__fmul_rn(g, gscale), p, m, v, lr_bc1, b1, b2, eps, bc2_inv_sqrt);
}

// One update of the exponential moving average of a weight (torch.optim.swa_utils.AveragedModel with
// torchvision's ema_avg): e' = d * e + a * p, d = fp32(decay), a = fp32(1 - decay) with 1 - decay
// taken in double on the host.  Two multiplies and one add, each rounded, no FMA: what torch's eager
// `decay * e + (1 - decay) * p` computes in fp32.  `first`: AveragedModel's first update copies p.
__device__ __forceinline__ float ema_update(float e, float p, float d, float a, bool first) {
  return first ? p : __fadd_rn(__fmul_rn(d, e), __fmul_rn(a, p));
}

// ema_update of 4 consecutive weights; ema is 16-byte aligned and streamed like every optimizer operand.
__device__ __forceinline__ void ema_update4(float* __restrict__ ema, const float* pp, const EmaCoef& c) {
  float4 e = __ldcs(reinterpret_cast<const float4*>(ema));
  e.x = ema_update(e.x, pp[0], c.d, c.a, c.first);
  e.y = ema_update(e.y, pp[1], c.d, c.a, c.first);
  e.z = ema_update(e.z, pp[2], c.d, c.a, c.first);
  e.w = ema_update(e.w, pp[3], c.d, c.a, c.first);
  __stcs(reinterpret_cast<float4*>(ema), e);
}

// One step of torch.optim.SGD with momentum and L2 weight decay: buf = g (first step) or
// momentum * buf + g, then p -= lr * buf.  The roundings are the ones nvcc's contraction chose when this
// was written as plain expressions: the decay product alone, everything else fused.
__device__ __forceinline__ void sgd_update(float g, float gscale, float& p, float& buf, float lr, float momentum,
                                           float wd, bool first) {
  const float gk = __fmaf_rn(g, gscale, __fmul_rn(wd, p));
  const float acc = __fmaf_rn(momentum, buf, gk);   // unconditional: keeps sgd_kernel at 32 registers
  buf = first ? gk : acc;
  p = __fmaf_rn(-lr, buf, p);
}

// LAMB's moments from the scaled gradient gk = g * gscale (no decay term: LAMB adds it to the update),
// rounded as adam_moments_step rounds them.
__device__ __forceinline__ void lamb_moments(float gk, float& m, float& v, float b1, float b2) {
  m = __fmaf_rn(b1, m, __fmul_rn(1.f - b1, gk));
  v = __fmaf_rn(b2, v, __fmul_rn(__fmul_rn(1.f - b2, gk), gk));
}

// LAMB's update direction u = (m bc1_inv) / (sqrt(v) bc2_inv_sqrt + eps) + wd p.  Phase 1 takes the norm of
// this u and phase 2 applies it, both through this function, so the norm is the norm of what is applied.
__device__ __forceinline__ float lamb_direction(float m, float v, float p, float bc1_inv, float bc2_inv_sqrt,
                                                float eps, float wd) {
  const float denom = __fmaf_rn(__fsqrt_rn(v), bc2_inv_sqrt, eps);
  return __fmaf_rn(wd, p, __fdiv_rn(__fmul_rn(m, bc1_inv), denom));
}

// Trust ratios from the whole tensor's sums of squares (timm's Lamb / Lars with trust_clip and always_adapt
// off): a tensor without decay, or with a zero norm, is not adapted.
__device__ __forceinline__ float lamb_ratio(float sum_p2, float sum_u2, float wd) {
  const float pn = __fsqrt_rn(sum_p2), un = __fsqrt_rn(sum_u2);
  return (wd != 0.f && pn > 0.f && un > 0.f) ? __fdiv_rn(pn, un) : 1.f;
}
__device__ __forceinline__ float lars_ratio(float sum_p2, float sum_g2, float wd, float coeff, float eps) {
  const float pn = __fsqrt_rn(sum_p2), gn = __fsqrt_rn(sum_g2);
  return (wd != 0.f && pn > 0.f && gn > 0.f)
             ? __fdiv_rn(__fmul_rn(coeff, pn), __fadd_rn(__fadd_rn(gn, __fmul_rn(wd, pn)), eps))
             : 1.f;
}

// One LARS step of an element: d = r (g gscale + wd p), buf = d (first step) or momentum buf + d,
// p -= lr buf.
__device__ __forceinline__ void lars_update(float g, float gscale, float& p, float& buf, float lr, float momentum,
                                            float wd, float r, bool first) {
  const float d = __fmul_rn(r, __fmaf_rn(wd, p, __fmul_rn(g, gscale)));
  buf = first ? d : __fmaf_rn(momentum, buf, d);
  p = __fmaf_rn(-lr, buf, p);
}

// The update of one element for the optimizer KIND (OptKind) of the step `o`, with decay value w (an L2
// decay, or AdamW's keep factor).  m is SGD's momentum buffer; SGD leaves v alone.
template <int KIND>
__device__ __forceinline__ void optimizer_update(const OptStep& o, float g, float gscale, float w, float& p, float& m,
                                                 float& v) {
  if constexpr (KIND == OPT_SGD)
    sgd_update(g, gscale, p, m, o.lr, o.momentum, w, o.first);
  else if constexpr (KIND == OPT_ADAMW)
    adamw_update(g, gscale, p, m, v, o.lr * o.bc1_inv, o.beta1, o.beta2, o.eps, w, o.bc2_inv_sqrt);
  else
    adam_update(g, gscale, p, m, v, o.lr * o.bc1_inv, o.beta1, o.beta2, o.eps, w, o.bc2_inv_sqrt);
}

}  // namespace b200
