// Fused cross-entropy (forward + backward + metrics) and the fused flat-arena optimizers.
//
// Reference semantics: F.cross_entropy(outputs, targets) with mean reduction
// (distributedVggf.py:168), Accuracy2 = argmax == target count (distributedUtil.py:92-99),
// Average = sample-weighted loss mean (distributedUtil.py:55-58), torch.optim.Adam with default
// betas/eps (distributedVggf.py:230).  The reference pays two host syncs per step for the metrics;
// here they are three atomics into a device meter.
#include <cmath>
#include <cstdlib>
#include <sstream>
#include <stdexcept>
#include <string>

#include "adam.cuh"
#include "api.h"
#include "ptx.cuh"

namespace b200 {

// Soft-target coefficient of class c in a row (SoftTargets in api.h): loss_r = sum_c q_c (-log p_c),
// q_c = w_c ((lam_a [c == t] + lam_b [c == tb]) (1 - eps) + eps / C); for integer targets lam_a = 1,
// lam_b = 0.  Its gradient is (p_c sum_k q_k - q_c) / normaliser.
__device__ __forceinline__ float soft_q(int c, int t, int tb, float la, float lb, float keep, float eps_c,
                                        const float* __restrict__ cw) {
  const float tc = ((c == t ? la : 0.f) + (c == tb ? lb : 0.f)) * keep + eps_c;
  return cw ? cw[c] * tc : tc;
}

// Row r's partner label and the two target weights (lam_b = 0 without mixing), and argmax of the
// unsmoothed target with torch's first-maximum rule.
__device__ __forceinline__ void soft_row(const long long* __restrict__ target, int r, int B, const SoftTargets& st,
                                         int& t, int& tb, float& la, float& lb, int& tmax) {
  t = static_cast<int>(target[r]);
  tb = st.mix ? static_cast<int>(target[r == 0 ? B - 1 : r - 1]) : t;
  la = st.mix ? st.lam_a : 1.f;
  lb = st.mix ? st.lam_b : 0.f;
  tmax = (tb != t && (lb > la || (lb == la && tb < t))) ? tb : t;
}

// Knowledge distillation (KdParams in api.h): for student logits z and teacher logits u of a row,
// log ps = log_softmax(z / T), log pt = log_softmax(u / T); the row's KL term is sum_c pt_c (log pt_c - log ps_c)
// and its gradient contribution kd.g (ps_c - pt_c).  Both log-softmaxes are taken from the row maxima.
__device__ __forceinline__ void kd_logs(float z, float mz, float ls, float u, float mu, float lt, float inv_t,
                                        float& lps, float& lpt) {
  lps = (z - mz) * inv_t - ls;
  lpt = (u - mu) * inv_t - lt;
}

// dlogit of class c: kd.ce * (the cross-entropy gradient g) + kd.g * (ps_c - pt_c).
__device__ __forceinline__ float kd_grad(float g, float z, float mz, float ls, float u, float mu, float lt,
                                         const KdParams& kd) {
  float lps, lpt;
  kd_logs(z, mz, ls, u, mu, lt, kd.inv_t, lps, lpt);
  return fmaf(kd.g, __expf(lps) - __expf(lpt), kd.ce * g);
}

// The batch's loss: kd.ce * (cross-entropy mean) + kd.l * (sum of the warps' KL terms) / B.
__device__ __forceinline__ float kd_loss(float ce_mean, const float* s_kl, int nwarps, int B, const KdParams& kd) {
  float kl = 0.f;
  for (int i = 0; i < nwarps; ++i) kl += s_kl[i];
  return fmaf(kd.l, kl / static_cast<float>(B), kd.ce * ce_mean);
}

// One block, one warp per row (round-robin).  C is small (3) or moderate (1000).
// SOFT: label smoothing and / or mixed targets (cross_entropy_soft); !SOFT is the integer-label loss.
template <bool SOFT>
__global__ void cross_entropy_kernel(const float* __restrict__ logits, const long long* __restrict__ target,
                                     bf16* __restrict__ dlogits, int ldd, float* __restrict__ meter,
                                     float* __restrict__ loss_out, int B, int C, float grad_scale,
                                     const float* __restrict__ cw, SoftTargets st) {
  __shared__ float s_loss[32], s_correct[32], s_wsum[32];
  __shared__ float s_total_w;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;

  // pass 0 (only with class weights): normaliser = sum_i w[target_i]
  float wsum_local = 0.f;
  if (cw) {
    for (int r = threadIdx.x; r < B; r += blockDim.x) wsum_local += cw[target[r]];
    for (int o = 16; o; o >>= 1) wsum_local += __shfl_xor_sync(0xffffffffu, wsum_local, o);
    if (lane == 0) s_wsum[warp] = wsum_local;
    __syncthreads();
    if (threadIdx.x == 0) {
      float t = 0.f;
      for (int i = 0; i < nwarps; ++i) t += s_wsum[i];
      s_total_w = t;
    }
    __syncthreads();
  }
  // probability targets (mixed batches) are divided by B even with class weights, as torch does
  const bool by_weight = cw && !(SOFT && st.mix);
  const float norm = by_weight ? 1.f / s_total_w : grad_scale;   // grad_scale == 1/B for the mean
  const float keep = 1.f - st.eps, eps_c = st.eps / static_cast<float>(C);

  float loss_acc = 0.f, correct_acc = 0.f;
  for (int r = warp; r < B; r += nwarps) {
    const float* row = logits + static_cast<long long>(r) * C;
    int t = static_cast<int>(target[r]), tb = t, tmax = t;
    float la = 1.f, lb = 0.f;
    if constexpr (SOFT) soft_row(target, r, B, st, t, tb, la, lb, tmax);
    float mx = -INFINITY;
    int amax = 0x7fffffff;
    for (int c = lane; c < C; c += 32) {
      const float v = row[c];
      if (v > mx) { mx = v; amax = c; }
    }
    for (int o = 16; o; o >>= 1) {
      const float om = __shfl_xor_sync(0xffffffffu, mx, o);
      const int oa = __shfl_xor_sync(0xffffffffu, amax, o);
      if (om > mx || (om == mx && oa < amax)) { mx = om; amax = oa; }
    }
    float se = 0.f;
    for (int c = lane; c < C; c += 32) se += __expf(row[c] - mx);
    for (int o = 16; o; o >>= 1) se += __shfl_xor_sync(0xffffffffu, se, o);
    const float lse = mx + __logf(se);
    if constexpr (SOFT) {
      float qs = 0.f, ql = 0.f;          // sum_c q_c and the row's loss sum_c q_c (lse - z_c)
      for (int c = lane; c < C; c += 32) {
        const float q = soft_q(c, t, tb, la, lb, keep, eps_c, cw);
        qs += q;
        ql += q * (lse - row[c]);
      }
      for (int o = 16; o; o >>= 1) {
        qs += __shfl_xor_sync(0xffffffffu, qs, o);
        ql += __shfl_xor_sync(0xffffffffu, ql, o);
      }
      if (dlogits) {
        for (int c = lane; c < ldd; c += 32) {
          float g = 0.f;
          if (c < C) g = (__expf(row[c] - lse) * qs - soft_q(c, t, tb, la, lb, keep, eps_c, cw)) * norm;
          dlogits[static_cast<long long>(r) * ldd + c] = __float2bfloat16(g);
        }
      }
      if (lane == 0) {
        loss_acc += ql;
        correct_acc += (amax == tmax) ? 1.f : 0.f;
      }
    } else {
      const float w = cw ? cw[t] : 1.f;
      if (dlogits) {
        for (int c = lane; c < ldd; c += 32) {
          float g = 0.f;
          if (c < C) g = (__expf(row[c] - lse) - (c == t ? 1.f : 0.f)) * w * norm;
          dlogits[static_cast<long long>(r) * ldd + c] = __float2bfloat16(g);
        }
      }
      if (lane == 0) {
        loss_acc += w * (lse - row[t]);
        correct_acc += (amax == t) ? 1.f : 0.f;
      }
    }
  }
  if (lane == 0) { s_loss[warp] = loss_acc; s_correct[warp] = correct_acc; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float tl = 0.f, tc = 0.f;
    for (int i = 0; i < nwarps; ++i) { tl += s_loss[i]; tc += s_correct[i]; }
    // batch loss as torch reports it: mean over the batch, or sum_i w_i nll_i / sum_i w_i with
    // class weights; the meter accumulates loss * B like Average.update(loss.item(), B)
    const float mean = by_weight ? tl / s_total_w : tl / static_cast<float>(B);
    if (meter) {
      atomicAdd(meter + 0, mean * static_cast<float>(B));
      atomicAdd(meter + 1, tc);
      atomicAdd(meter + 2, static_cast<float>(B));
    }
    if (loss_out) *loss_out = mean;
  }
}

// cross_entropy_kernel with the distillation loss (cross_entropy_kd): L = kd.ce * CE + kd.l * KL / B against the
// teacher logits `tlog` [B][C], dlogits kd.ce * (the cross-entropy gradient) + kd.g * (ps - pt).  A kernel of its own
// rather than a template parameter of cross_entropy_kernel, whose instantiations keep their code.
template <bool SOFT>
__global__ void __launch_bounds__(1024)
cross_entropy_kd_kernel(const float* __restrict__ logits, const long long* __restrict__ target,
                        bf16* __restrict__ dlogits, int ldd, float* __restrict__ meter,
                        float* __restrict__ loss_out, int B, int C, float grad_scale,
                        const float* __restrict__ cw, SoftTargets st,
                        const float* __restrict__ tlog, KdParams kd) {
  __shared__ float s_loss[32], s_correct[32], s_wsum[32];
  float* s_kl = s_wsum;          // the warps' KL terms (s_wsum is free once pass 0 is over)
  __shared__ float s_total_w;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;

  // pass 0 (only with class weights): normaliser = sum_i w[target_i]
  float wsum_local = 0.f;
  if (cw) {
    for (int r = threadIdx.x; r < B; r += blockDim.x) wsum_local += cw[target[r]];
    for (int o = 16; o; o >>= 1) wsum_local += __shfl_xor_sync(0xffffffffu, wsum_local, o);
    if (lane == 0) s_wsum[warp] = wsum_local;
    __syncthreads();
    if (threadIdx.x == 0) {
      float t = 0.f;
      for (int i = 0; i < nwarps; ++i) t += s_wsum[i];
      s_total_w = t;
    }
    __syncthreads();
  }
  // probability targets (mixed batches) are divided by B even with class weights, as torch does
  const bool by_weight = cw && !(SOFT && st.mix);
  const float norm = by_weight ? 1.f / s_total_w : grad_scale;   // grad_scale == 1/B for the mean
  const float keep = 1.f - st.eps, eps_c = st.eps / static_cast<float>(C);

  float loss_acc = 0.f, correct_acc = 0.f, kl_acc = 0.f;
  for (int r = warp; r < B; r += nwarps) {
    const float* row = logits + static_cast<long long>(r) * C;
    int t = static_cast<int>(target[r]), tb = t, tmax = t;
    float la = 1.f, lb = 0.f;
    if constexpr (SOFT) soft_row(target, r, B, st, t, tb, la, lb, tmax);
    float mx = -INFINITY;
    int amax = 0x7fffffff;
    for (int c = lane; c < C; c += 32) {
      const float v = row[c];
      if (v > mx) { mx = v; amax = c; }
    }
    for (int o = 16; o; o >>= 1) {
      const float om = __shfl_xor_sync(0xffffffffu, mx, o);
      const int oa = __shfl_xor_sync(0xffffffffu, amax, o);
      if (om > mx || (om == mx && oa < amax)) { mx = om; amax = oa; }
    }
    float se = 0.f;
    for (int c = lane; c < C; c += 32) se += __expf(row[c] - mx);
    for (int o = 16; o; o >>= 1) se += __shfl_xor_sync(0xffffffffu, se, o);
    const float lse = mx + __logf(se);
    // teacher row maximum, both log-normalisers at temperature T, and the row's KL term
    float mu = -INFINITY, ls = 0.f, lt = 0.f;
    {
      const float* trow = tlog + static_cast<long long>(r) * C;
      for (int c = lane; c < C; c += 32) mu = fmaxf(mu, trow[c]);
      for (int o = 16; o; o >>= 1) mu = fmaxf(mu, __shfl_xor_sync(0xffffffffu, mu, o));
      float ss = 0.f, su = 0.f;
      for (int c = lane; c < C; c += 32) {
        ss += __expf((row[c] - mx) * kd.inv_t);
        su += __expf((trow[c] - mu) * kd.inv_t);
      }
      for (int o = 16; o; o >>= 1) {
        ss += __shfl_xor_sync(0xffffffffu, ss, o);
        su += __shfl_xor_sync(0xffffffffu, su, o);
      }
      ls = __logf(ss);
      lt = __logf(su);
      float kl = 0.f;
      for (int c = lane; c < C; c += 32) {
        float lps, lpt;
        kd_logs(row[c], mx, ls, trow[c], mu, lt, kd.inv_t, lps, lpt);
        kl += __expf(lpt) * (lpt - lps);
      }
      for (int o = 16; o; o >>= 1) kl += __shfl_xor_sync(0xffffffffu, kl, o);
      if (lane == 0) kl_acc += kl;
    }
    if constexpr (SOFT) {
      float qs = 0.f, ql = 0.f;          // sum_c q_c and the row's loss sum_c q_c (lse - z_c)
      for (int c = lane; c < C; c += 32) {
        const float q = soft_q(c, t, tb, la, lb, keep, eps_c, cw);
        qs += q;
        ql += q * (lse - row[c]);
      }
      for (int o = 16; o; o >>= 1) {
        qs += __shfl_xor_sync(0xffffffffu, qs, o);
        ql += __shfl_xor_sync(0xffffffffu, ql, o);
      }
      if (dlogits) {
        for (int c = lane; c < ldd; c += 32) {
          float g = 0.f;
          if (c < C) g = (__expf(row[c] - lse) * qs - soft_q(c, t, tb, la, lb, keep, eps_c, cw)) * norm;
          if (c < C) g = kd_grad(g, row[c], mx, ls, tlog[static_cast<long long>(r) * C + c], mu, lt, kd);
          dlogits[static_cast<long long>(r) * ldd + c] = __float2bfloat16(g);
        }
      }
      if (lane == 0) {
        loss_acc += ql;
        correct_acc += (amax == tmax) ? 1.f : 0.f;
      }
    } else {
      const float w = cw ? cw[t] : 1.f;
      if (dlogits) {
        for (int c = lane; c < ldd; c += 32) {
          float g = 0.f;
          if (c < C) g = (__expf(row[c] - lse) - (c == t ? 1.f : 0.f)) * w * norm;
          if (c < C) g = kd_grad(g, row[c], mx, ls, tlog[static_cast<long long>(r) * C + c], mu, lt, kd);
          dlogits[static_cast<long long>(r) * ldd + c] = __float2bfloat16(g);
        }
      }
      if (lane == 0) {
        loss_acc += w * (lse - row[t]);
        correct_acc += (amax == t) ? 1.f : 0.f;
      }
    }
  }
  if (lane == 0) { s_loss[warp] = loss_acc; s_correct[warp] = correct_acc; }
  if (lane == 0) s_kl[warp] = kl_acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float tl = 0.f, tc = 0.f;
    for (int i = 0; i < nwarps; ++i) { tl += s_loss[i]; tc += s_correct[i]; }
    // batch loss as torch reports it: mean over the batch, or sum_i w_i nll_i / sum_i w_i with
    // class weights; the meter accumulates loss * B like Average.update(loss.item(), B)
    const float ce = by_weight ? tl / s_total_w : tl / static_cast<float>(B);
    const float mean = kd_loss(ce, s_kl, nwarps, B, kd);
    if (meter) {
      atomicAdd(meter + 0, mean * static_cast<float>(B));
      atomicAdd(meter + 1, tc);
      atomicAdd(meter + 2, static_cast<float>(B));
    }
    if (loss_out) *loss_out = mean;
  }
}

void cross_entropy_fused(const float* logits, const long long* target, bf16* dlogits, int ldd,
                         float* meter, float* loss_out, int B, int C, float grad_scale,
                         const float* class_weights, cudaStream_t s) {
  cross_entropy_kernel<false><<<1, 1024, 0, s>>>(logits, target, dlogits, ldd, meter, loss_out, B, C,
                                                 grad_scale, class_weights, SoftTargets{0.f, 1.f, 0.f, 0});
  count_launch();
  check_last("cross_entropy_fused");
}

void cross_entropy_soft(const float* logits, const long long* target, bf16* dlogits, int ldd, float* meter,
                        float* loss_out, int B, int C, float grad_scale, const float* class_weights,
                        const SoftTargets& st, cudaStream_t s) {
  cross_entropy_kernel<true><<<1, 1024, 0, s>>>(logits, target, dlogits, ldd, meter, loss_out, B, C,
                                                grad_scale, class_weights, st);
  count_launch();
  check_last("cross_entropy_soft");
}

void cross_entropy_kd(const float* logits, const long long* target, bf16* dlogits, int ldd, float* meter,
                      float* loss_out, int B, int C, float grad_scale, const float* class_weights,
                      const SoftTargets* soft, const float* teacher, const KdParams& kd, cudaStream_t s) {
  if (soft)
    cross_entropy_kd_kernel<true><<<1, 1024, 0, s>>>(logits, target, dlogits, ldd, meter, loss_out, B, C, grad_scale,
                                                     class_weights, *soft, teacher, kd);
  else
    cross_entropy_kd_kernel<false><<<1, 1024, 0, s>>>(logits, target, dlogits, ldd, meter, loss_out, B, C,
                                                      grad_scale, class_weights, SoftTargets{0.f, 1.f, 0.f, 0},
                                                      teacher, kd);
  count_launch();
  check_last("cross_entropy_kd");
}

// Test-time augmentation (tta_accumulate): one block, one warp per row, as cross_entropy_kernel.  Each view adds its
// softmax into acc in view order with plain stores (no atomics: the same bits on every run).  The last view also
// scores the mean probability m = acc / V: loss -log m[y], argmax with the lowest index on ties.
__global__ void __launch_bounds__(1024)
tta_accumulate_kernel(const float* __restrict__ logits, const long long* __restrict__ target, float* __restrict__ acc,
                      float* __restrict__ meter, float* __restrict__ loss_out, int B, int C, int view, int views) {
  __shared__ float s_loss[32], s_correct[32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  const bool last = view == views - 1;
  const float fv = static_cast<float>(views);
  float loss_acc = 0.f, correct_acc = 0.f;
  for (int r = warp; r < B; r += nwarps) {
    const float* row = logits + static_cast<long long>(r) * C;
    float* arow = acc + static_cast<long long>(r) * C;
    float mx = -INFINITY;
    for (int c = lane; c < C; c += 32) mx = fmaxf(mx, row[c]);
    for (int o = 16; o; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float se = 0.f;
    for (int c = lane; c < C; c += 32) se += expf(row[c] - mx);
    for (int o = 16; o; o >>= 1) se += __shfl_xor_sync(0xffffffffu, se, o);
    float best = -INFINITY;
    int amax = 0x7fffffff;
    for (int c = lane; c < C; c += 32) {
      const float p = __fdiv_rn(expf(row[c] - mx), se);
      const float a = view == 0 ? p : __fadd_rn(arow[c], p);
      arow[c] = a;
      if (last) {
        const float m = __fdiv_rn(a, fv);
        if (m > best) { best = m; amax = c; }
      }
    }
    if (last) {
      for (int o = 16; o; o >>= 1) {
        const float ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int oa = __shfl_xor_sync(0xffffffffu, amax, o);
        if (ob > best || (ob == best && oa < amax)) { best = ob; amax = oa; }
      }
      __syncwarp();                  // the lane that stored acc[r][t] may be another one
      if (lane == 0) {
        const int t = static_cast<int>(target[r]);
        loss_acc += -logf(__fdiv_rn(arow[t], fv));
        correct_acc += (amax == t) ? 1.f : 0.f;
      }
    }
  }
  if (!last) return;
  if (lane == 0) { s_loss[warp] = loss_acc; s_correct[warp] = correct_acc; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float tl = 0.f, tc = 0.f;
    for (int i = 0; i < nwarps; ++i) { tl += s_loss[i]; tc += s_correct[i]; }
    const float mean = tl / static_cast<float>(B);     // the meter takes loss * B, as cross_entropy_kernel's
    if (meter) {
      atomicAdd(meter + 0, mean * static_cast<float>(B));
      atomicAdd(meter + 1, tc);
      atomicAdd(meter + 2, static_cast<float>(B));
    }
    if (loss_out) *loss_out = mean;
  }
}

void tta_accumulate(const float* logits, const long long* target, float* acc, float* meter, float* loss_out, int B,
                    int C, int view, int views, cudaStream_t s) {
  tta_accumulate_kernel<<<1, 1024, 0, s>>>(logits, target, acc, meter, loss_out, B, C, view, views);
  count_launch();
  check_last("tta_accumulate");
}

// Per-class evaluation counts (class_metrics, --val-metrics): one warp per row, as tta_accumulate_kernel, eight rows
// per block so that a batch's rows run on several SMs.  A row's scores are s_c = scores[r][c] / V with __fdiv_rn,
// tta_accumulate's view mean (V = 1: the logits as they are, x / 1 being x).  The prediction is the first maximum
// (v > max from -inf, lowest index on ties), the rule of the correct-counts of cross_entropy_kernel and
// tta_accumulate_kernel, so the diagonal of M sums to their count.  The label's rank is
// #{c : s_c > s_y} + #{c < y : s_c == s_y}; below 5 the row counts toward top-5.  A row without a maximum (every
// score NaN or -inf) or with a label outside [0, C) is counted nowhere.  Integer atomics: the same counts every run.
constexpr int CM_ROWS = 8, CM_UNROLL = 4;
__global__ void __launch_bounds__(CM_ROWS * 32)
class_metrics_kernel(const float* __restrict__ scores, const long long* __restrict__ target,
                     unsigned long long* __restrict__ M, unsigned long long* __restrict__ top5, int B, int C, int views) {
  __shared__ unsigned int s_top5[CM_ROWS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r = blockIdx.x * CM_ROWS + warp;
  unsigned int hit = 0;
  const long long t = r < B ? target[r] : -1;
  if (t >= 0 && t < C) {                               // the same for every lane of the warp
    const int y = static_cast<int>(t);
    const float* row = scores + static_cast<long long>(r) * C;
    const float fv = static_cast<float>(views);
    const float sy = __fdiv_rn(row[y], fv);
    float best = -INFINITY;
    int amax = 0x7fffffff;
    unsigned int ahead = 0;                            // classes ranked before the label
    for (int c0 = lane; c0 < C; c0 += 32 * CM_UNROLL) {
      float v[CM_UNROLL];                              // the loads first: CM_UNROLL in flight per lane
#pragma unroll
      for (int u = 0; u < CM_UNROLL; ++u) v[u] = c0 + 32 * u < C ? row[c0 + 32 * u] : 0.f;
#pragma unroll
      for (int u = 0; u < CM_UNROLL; ++u) {            // in increasing c, as one element per step would
        const int c = c0 + 32 * u;
        if (c < C) {
          const float x = __fdiv_rn(v[u], fv);
          if (x > best) { best = x; amax = c; }
          ahead += (x > sy || (x == sy && c < y)) ? 1u : 0u;
        }
      }
    }
    for (int o = 16; o; o >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int oa = __shfl_xor_sync(0xffffffffu, amax, o);
      if (ob > best || (ob == best && oa < amax)) { best = ob; amax = oa; }
      ahead += __shfl_xor_sync(0xffffffffu, ahead, o);
    }
    if (lane == 0 && amax < C) {
      atomicAdd(M + static_cast<long long>(y) * C + amax, 1ull);
      hit = ahead < 5 ? 1u : 0u;
    }
  }
  if (lane == 0) s_top5[warp] = hit;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long n = 0;
    for (int i = 0; i < CM_ROWS; ++i) n += s_top5[i];
    if (n) atomicAdd(top5, n);
  }
}

void class_metrics(const float* scores, const long long* target, long long* confusion, long long* top5, int B, int C,
                   int views, cudaStream_t s) {
  class_metrics_kernel<<<(B + CM_ROWS - 1) / CM_ROWS, CM_ROWS * 32, 0, s>>>(
      scores, target, reinterpret_cast<unsigned long long*>(confusion), reinterpret_cast<unsigned long long*>(top5), B,
      C, views);
  count_launch();
  check_last("class_metrics");
}

KdParams kd_params(double alpha, double temperature, int B) {
  return KdParams{static_cast<float>(1.0 - alpha), static_cast<float>(alpha * temperature / B),
                  static_cast<float>(alpha * temperature * temperature), static_cast<float>(1.0 / temperature)};
}

// ------------------------------------------------------------- fused head: last Linear + CE + bwd
// K-FUN2+CE (SURVEY 2.5): the funnel's Linear(512, C) (distributedVggf.py:56), cross_entropy (:168),
// Accuracy2 / Average (distributedUtil.py:95-96, :55-58) and the whole backward of that layer in ONE
// launch of one CTA -- seven launches before (GEMM, bias epilogue, CE, bias grad, wgrad GEMM, dgrad
// GEMM, ReLU/dropout-mask epilogue).  C <= 8 classes, K <= 1024 inputs, B <= 256 rows; everything lives
// in shared memory / registers:
//   logits[r][c] = bias[c] + sum_k h[r][k] W[c][k]            (warp per row, fp32 accumulation)
//   loss, argmax == target count, B  -> device meter;  dlogits = (softmax - onehot) * w / norm -> bf16
//   db[c] += sum_r dl[r][c];  dW[c][k] = sum_r dl[r][c] h[r][k]  (+= with accumulate) (thread per k)
//   dh[r][k] = (h[r][k] > 0) * drop_scale * sum_c dl[r][c] W[c][k]  -> bf16     (previous layer's dz)
// Rounding points are those of the unfused path: dlogits are rounded to bf16 before they are used.
constexpr int HEAD_MAXC = 8, HEAD_MAXK = 1024, HEAD_MAXB = 256, HEAD_THREADS = 512;

// SOFT: soft targets as in cross_entropy_kernel<true>; KD: the distillation loss of cross_entropy_kd_kernel, teacher
// logits `tlog` [B][C].  The backward of the layer is unchanged: it takes whichever dlogits the loss made.
template <bool SOFT, bool KD>
__device__ __forceinline__ void head_ce_body(const bf16* __restrict__ h, const bf16* __restrict__ W,
                                             const float* __restrict__ bias, const long long* __restrict__ target,
                                             float* __restrict__ logits, bf16* __restrict__ dlogits, int ldd,
                                             float* __restrict__ dW, float* __restrict__ db, bf16* __restrict__ dh,
                                             float drop_scale, int relu, float* __restrict__ meter,
                                             float* __restrict__ loss_out, int B, int C, int K,
                                             const float* __restrict__ cw, int accumulate, const SoftTargets& st,
                                             const float* __restrict__ tlog, const KdParams& kd) {
  __shared__ float sW[HEAD_MAXC * HEAD_MAXK];
  __shared__ float sdl[HEAD_MAXB * HEAD_MAXC];
  __shared__ float s_loss[32], s_correct[32], s_wsum[32];
  __shared__ float s_total_w;
  float* s_kl = s_wsum;          // KD: the warps' KL terms (s_wsum is free once the normaliser is summed)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  for (int i = threadIdx.x; i < C * K; i += blockDim.x) sW[i] = __bfloat162float(W[i]);

  float wsum_local = 0.f;
  if (cw) {      // class weights: normaliser = sum_i w[target_i]   (same as cross_entropy_kernel)
    for (int r = threadIdx.x; r < B; r += blockDim.x) wsum_local += cw[target[r]];
    for (int o = 16; o; o >>= 1) wsum_local += __shfl_xor_sync(0xffffffffu, wsum_local, o);
    if (lane == 0) s_wsum[warp] = wsum_local;
  }
  __syncthreads();
  if (cw && threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < nwarps; ++i) t += s_wsum[i];
    s_total_w = t;
  }
  __syncthreads();
  const bool by_weight = cw && !(SOFT && st.mix);      // probability targets: divided by B
  const float norm = by_weight ? 1.f / s_total_w : 1.f / static_cast<float>(B);
  const float keep = 1.f - st.eps, eps_c = st.eps / static_cast<float>(C);

  // ---- forward + loss + dlogits ---------------------------------------------------------------
  float loss_acc = 0.f, correct_acc = 0.f, kl_acc = 0.f;
  for (int r = warp; r < B; r += nwarps) {
    float acc[HEAD_MAXC];
#pragma unroll
    for (int c = 0; c < HEAD_MAXC; ++c) acc[c] = 0.f;
    const bf16* hr = h + static_cast<long long>(r) * K;
    for (int k = lane; k < K; k += 32) {
      const float hv = __bfloat162float(hr[k]);
#pragma unroll
      for (int c = 0; c < HEAD_MAXC; ++c)
        if (c < C) acc[c] = fmaf(hv, sW[c * K + k], acc[c]);
    }
#pragma unroll
    for (int c = 0; c < HEAD_MAXC; ++c)
      for (int o = 16; o; o >>= 1) acc[c] += __shfl_xor_sync(0xffffffffu, acc[c], o);
    int t = static_cast<int>(target[r]), tb = t, tmax = t;
    float la = 1.f, lb = 0.f;
    if constexpr (SOFT) soft_row(target, r, B, st, t, tb, la, lb, tmax);
    float mx = -INFINITY;
    int amax = 0;
#pragma unroll
    for (int c = 0; c < HEAD_MAXC; ++c)
      if (c < C) {
        acc[c] += bias[c];
        if (acc[c] > mx) { mx = acc[c]; amax = c; }       // first maximum, like torch.argmax
      }
    float se = 0.f, zt = 0.f;
#pragma unroll
    for (int c = 0; c < HEAD_MAXC; ++c)
      if (c < C) {
        se += __expf(acc[c] - mx);
        if (c == t) zt = acc[c];
      }
    const float lse = mx + __logf(se);
    // KD: the teacher row, its maximum, both log-normalisers at temperature T and the row's KL term
    float u[HEAD_MAXC], mu = -INFINITY, ls = 0.f, lt = 0.f;
    if constexpr (KD) {
      float ss = 0.f, su = 0.f, kl = 0.f;
#pragma unroll
      for (int c = 0; c < HEAD_MAXC; ++c)
        if (c < C) {
          u[c] = tlog[static_cast<long long>(r) * C + c];
          mu = fmaxf(mu, u[c]);
        }
#pragma unroll
      for (int c = 0; c < HEAD_MAXC; ++c)
        if (c < C) {
          ss += __expf((acc[c] - mx) * kd.inv_t);
          su += __expf((u[c] - mu) * kd.inv_t);
        }
      ls = __logf(ss);
      lt = __logf(su);
#pragma unroll
      for (int c = 0; c < HEAD_MAXC; ++c)
        if (c < C) {
          float lps, lpt;
          kd_logs(acc[c], mx, ls, u[c], mu, lt, kd.inv_t, lps, lpt);
          kl += __expf(lpt) * (lpt - lps);
        }
      if (lane == 0) kl_acc += kl;
    }
    float w = cw ? cw[t] : 1.f;
    float qs = 0.f, ql = 0.f;        // SOFT: sum_c q_c and the row's loss sum_c q_c (lse - z_c)
    if constexpr (SOFT) {
#pragma unroll
      for (int c = 0; c < HEAD_MAXC; ++c)
        if (c < C) {
          const float q = soft_q(c, t, tb, la, lb, keep, eps_c, cw);
          qs += q;
          ql += q * (lse - acc[c]);
        }
      w = 1.f;
    }
    if (lane < ldd || lane < C) {
      float g = 0.f, z = 0.f;
#pragma unroll
      for (int c = 0; c < HEAD_MAXC; ++c)
        if (c == lane && c < C) {
          z = acc[c];
          if constexpr (SOFT)
            g = (__expf(acc[c] - lse) * qs - soft_q(c, t, tb, la, lb, keep, eps_c, cw)) * norm;
          else
            g = (__expf(acc[c] - lse) - (c == t ? 1.f : 0.f)) * w * norm;
          if constexpr (KD) g = kd_grad(g, acc[c], mx, ls, u[c], mu, lt, kd);
        }
      if (lane < C) {
        logits[static_cast<long long>(r) * C + lane] = z;
        sdl[r * HEAD_MAXC + lane] = __bfloat162float(__float2bfloat16(g));
      }
      if (dlogits && lane < ldd) dlogits[static_cast<long long>(r) * ldd + lane] = __float2bfloat16(g);
    }
    if (lane == 0) {
      if constexpr (SOFT) {
        loss_acc += ql;
        correct_acc += (amax == tmax) ? 1.f : 0.f;
      } else {
        loss_acc += w * (lse - zt);
        correct_acc += (amax == t) ? 1.f : 0.f;
      }
    }
  }
  if (lane == 0) { s_loss[warp] = loss_acc; s_correct[warp] = correct_acc; }
  if constexpr (KD)
    if (lane == 0) s_kl[warp] = kl_acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float tl = 0.f, tc = 0.f;
    for (int i = 0; i < nwarps; ++i) { tl += s_loss[i]; tc += s_correct[i]; }
    float mean = by_weight ? tl / s_total_w : tl / static_cast<float>(B);
    if constexpr (KD) mean = kd_loss(mean, s_kl, nwarps, B, kd);
    if (meter) {
      atomicAdd(meter + 0, mean * static_cast<float>(B));
      atomicAdd(meter + 1, tc);
      atomicAdd(meter + 2, static_cast<float>(B));
    }
    if (loss_out) *loss_out = mean;
  }
  if (!dW) return;                       // evaluation: forward + metrics only

  // ---- backward of the layer --------------------------------------------------------------------
  if (threadIdx.x < C) {
    float sum = 0.f;
    for (int r = 0; r < B; ++r) sum += sdl[r * HEAD_MAXC + threadIdx.x];
    db[threadIdx.x] += sum;
  }
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    float wk[HEAD_MAXC], gw[HEAD_MAXC];
#pragma unroll
    for (int c = 0; c < HEAD_MAXC; ++c) { wk[c] = c < C ? sW[c * K + k] : 0.f; gw[c] = 0.f; }
    for (int r = 0; r < B; ++r) {
      const float hv = __bfloat162float(h[static_cast<long long>(r) * K + k]);
      float dx = 0.f;
#pragma unroll
      for (int c = 0; c < HEAD_MAXC; ++c)
        if (c < C) {
          const float g = sdl[r * HEAD_MAXC + c];
          gw[c] = fmaf(g, hv, gw[c]);
          dx = fmaf(g, wk[c], dx);
        }
      if (dh) dh[static_cast<long long>(r) * K + k] = __float2bfloat16((!relu || hv > 0.f) ? dx * drop_scale : 0.f);
    }
    // accumulate: a later micro-batch of a gradient-accumulation group adds to the group's dW
#pragma unroll
    for (int c = 0; c < HEAD_MAXC; ++c)
      if (c < C) {
        float* o = dW + static_cast<long long>(c) * K + k;
        *o = accumulate ? *o + gw[c] : gw[c];
      }
  }
}

template <bool SOFT>
__global__ void __launch_bounds__(HEAD_THREADS, 1)
head_ce_kernel(const bf16* __restrict__ h, const bf16* __restrict__ W, const float* __restrict__ bias,
               const long long* __restrict__ target, float* __restrict__ logits, bf16* __restrict__ dlogits, int ldd,
               float* __restrict__ dW, float* __restrict__ db, bf16* __restrict__ dh, float drop_scale, int relu,
               float* __restrict__ meter, float* __restrict__ loss_out, int B, int C, int K,
               const float* __restrict__ cw, int accumulate, SoftTargets st) {
  head_ce_body<SOFT, false>(h, W, bias, target, logits, dlogits, ldd, dW, db, dh, drop_scale, relu, meter, loss_out, B,
                            C, K, cw, accumulate, st, nullptr, KdParams{});
}

template <bool SOFT>
__global__ void __launch_bounds__(HEAD_THREADS, 1)
head_ce_kd_kernel(const bf16* __restrict__ h, const bf16* __restrict__ W, const float* __restrict__ bias,
                  const long long* __restrict__ target, float* __restrict__ logits, bf16* __restrict__ dlogits,
                  int ldd, float* __restrict__ dW, float* __restrict__ db, bf16* __restrict__ dh, float drop_scale,
                  int relu, float* __restrict__ meter, float* __restrict__ loss_out, int B, int C, int K,
                  const float* __restrict__ cw, int accumulate, SoftTargets st, const float* __restrict__ teacher,
                  KdParams kd) {
  head_ce_body<SOFT, true>(h, W, bias, target, logits, dlogits, ldd, dW, db, dh, drop_scale, relu, meter, loss_out, B,
                           C, K, cw, accumulate, st, teacher, kd);
}

bool head_ce_supported(int B, int C, int K) { return C <= HEAD_MAXC && K <= HEAD_MAXK && B <= HEAD_MAXB && B > 0; }

void head_ce_fused(const bf16* h, const bf16* W, const float* bias, const long long* target, float* logits,
                   bf16* dlogits, int ldd, float* dW, float* db, bf16* dh, float drop_scale, bool relu, float* meter,
                   float* loss_out, int B, int C, int K, const float* class_weights, bool accumulate,
                   cudaStream_t s, const SoftTargets* soft) {
  if (!head_ce_supported(B, C, K)) throw std::runtime_error("[b200] head_ce_fused: needs C <= 8, K <= 1024, B <= 256");
  if (ldd > 32) throw std::runtime_error("[b200] head_ce_fused: dlogits row stride must be <= 32");
  if (soft)
    head_ce_kernel<true><<<1, HEAD_THREADS, 0, s>>>(h, W, bias, target, logits, dlogits, ldd, dW, db, dh, drop_scale,
                                                    relu ? 1 : 0, meter, loss_out, B, C, K, class_weights,
                                                    accumulate ? 1 : 0, *soft);
  else
    head_ce_kernel<false><<<1, HEAD_THREADS, 0, s>>>(h, W, bias, target, logits, dlogits, ldd, dW, db, dh, drop_scale,
                                                     relu ? 1 : 0, meter, loss_out, B, C, K, class_weights,
                                                     accumulate ? 1 : 0, SoftTargets{0.f, 1.f, 0.f, 0});
  count_launch();
  check_last("head_ce_fused");
}

void head_ce_kd_fused(const bf16* h, const bf16* W, const float* bias, const long long* target, float* logits,
                      bf16* dlogits, int ldd, float* dW, float* db, bf16* dh, float drop_scale, bool relu, float* meter,
                      float* loss_out, int B, int C, int K, const float* class_weights, bool accumulate,
                      const SoftTargets* soft, const float* teacher, const KdParams& kd, cudaStream_t s) {
  if (!head_ce_supported(B, C, K)) throw std::runtime_error("[b200] head_ce_kd_fused: needs C <= 8, K <= 1024, B <= 256");
  if (ldd > 32) throw std::runtime_error("[b200] head_ce_kd_fused: dlogits row stride must be <= 32");
  if (soft)
    head_ce_kd_kernel<true><<<1, HEAD_THREADS, 0, s>>>(h, W, bias, target, logits, dlogits, ldd, dW, db, dh, drop_scale,
                                                       relu ? 1 : 0, meter, loss_out, B, C, K, class_weights,
                                                       accumulate ? 1 : 0, *soft, teacher, kd);
  else
    head_ce_kd_kernel<false><<<1, HEAD_THREADS, 0, s>>>(h, W, bias, target, logits, dlogits, ldd, dW, db, dh,
                                                        drop_scale, relu ? 1 : 0, meter, loss_out, B, C, K,
                                                        class_weights, accumulate ? 1 : 0,
                                                        SoftTargets{0.f, 1.f, 0.f, 0}, teacher, kd);
  count_launch();
  check_last("head_ce_kd_fused");
}

// ---------------------------------------------------------------------------------- optimizers
EmaCoef ema_coef(double decay, bool first) {
  return EmaCoef{static_cast<float>(decay), static_cast<float>(1.0 - decay), first ? 1 : 0};
}

OptStep make_opt_step(const char* op, OptKind kind, long long n, double lr, double beta1, double beta2, double eps,
                      double momentum, int step, bool first, double grad_scale, double wd,
                      const std::vector<int64_t>& wd_starts, const std::vector<double>& wd_values, double ema_decay,
                      bool ema_first) {
  auto check = [op](bool ok, const auto&... msg) {
    if (ok) return;
    std::ostringstream s;
    ((s << op) << ... << msg);
    throw std::runtime_error(s.str());
  };
  OptStep o{};
  o.kind = kind;
  o.lr = static_cast<float>(lr);
  o.beta1 = static_cast<float>(beta1);
  o.beta2 = static_cast<float>(beta2);
  o.eps = static_cast<float>(eps);
  if (kind != OPT_SGD) {   // from the fp32 betas
    o.bc1_inv = static_cast<float>(1.0 / (1.0 - pow(static_cast<double>(o.beta1), step)));
    o.bc2_inv_sqrt = static_cast<float>(1.0 / sqrt(1.0 - pow(static_cast<double>(o.beta2), step)));
  }
  o.momentum = static_cast<float>(momentum);
  o.first = first ? 1 : 0;
  o.grad_scale = static_cast<float>(grad_scale);
  o.ema = ema_coef(ema_decay, ema_first);
  auto value = [&](double d) { return static_cast<float>(kind == OPT_ADAMW ? 1.0 - lr * d : d); };
  WdSegments& s = o.wd;
  if (wd_starts.empty()) {
    check(wd_values.empty(), ": wd_starts and wd_values go together");
    s.n = 1;
    s.value[0] = value(wd);
    return o;
  }
  check(wd_starts.size() == wd_values.size(), ": wd_starts and wd_values must have the same length");
  check(wd_starts.size() <= static_cast<size_t>(WD_MAX_SEGMENTS), ": at most ", WD_MAX_SEGMENTS,
        " weight-decay segments per launch, got ", wd_starts.size());
  check(wd_starts[0] == 0, ": the first weight-decay segment must start at 0");
  s.n = static_cast<int>(wd_starts.size());
  for (int k = 0; k < s.n; ++k) {
    const int64_t start = wd_starts[k];
    const double d = wd_values[k];
    check(k == 0 || start > wd_starts[k - 1], ": weight-decay segment starts must increase");
    check(start % 4 == 0, ": weight-decay segment starts must be multiples of 4, got ", start);
    check(start < n, ": weight-decay segment start ", start, " lies outside the range of ", n);
    check(std::isfinite(d) && d >= 0.0, ": weight decays must be finite and >= 0, got ", d);
    s.start4[k] = start / 4;
    s.value[k] = value(d);
  }
  return o;
}

// One pass over the flat arena: read grad (fp32 local or bf16 reduced wire), update the fp32 master
// weight and the optimizer state, emit the bf16 shadow used by the GEMMs, and zero the fp32 gradient so
// the red.add wgrad epilogues of the next step start from zero.
// Footprint (same reasoning as allreduce.cu): the update runs on the comm stream UNDER the persistent
// conv kernels of backward.  256 threads x <= 40 registers and no shared memory co-reside with any of
// them, and the grid is capped by optimizer_grid -- a background stream of HBM traffic.  (Round 1
// launched 8 CTAs per SM: at every conv-kernel boundary the high-priority stream filled the SMs with
// optimizer CTAs and the next conv kernel's persistent CTAs started late; bench/step_timeline.py.)
// EMA: also update the weights' moving average `ema` from the new p while it is in registers (one
// more fp32 stream, 8 B per parameter); the EMA = false instantiation is the plain optimizer.
// The step `o` (with its WdSegments) sits in the parameter bank: the thread walks the segments forward
// as its grid-stride loop moves through the range, one compare per iteration for a uniform decay.
template <int KIND, bool EMA>
__device__ __forceinline__ void optimizer_pass(const OptStep& o, float* __restrict__ p, float* __restrict__ m,
                                               float* __restrict__ v, const float* __restrict__ g32,
                                               const bf16* __restrict__ g16, bf16* __restrict__ shadow,
                                               float* __restrict__ gzero, float* __restrict__ ema, long long n4) {
  int seg = 0;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n4;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    while (seg + 1 < o.wd.n && i >= o.wd.start4[seg + 1]) ++seg;
    const float w = o.wd.value[seg];
    // Every stream here is touched exactly once per step: cache-streaming (evict-first) loads and
    // stores, so that ~4 GB of optimizer traffic does not flush the conv kernels' L2-resident operand
    // tiles while it runs under backward (bench/step_timeline.py: +30 % on the 512-channel layers).
    const float4 pv = __ldcs(reinterpret_cast<const float4*>(p) + i);
    const float4 mv = __ldcs(reinterpret_cast<const float4*>(m) + i);
    float4 vv{};
    if constexpr (KIND != OPT_SGD) vv = __ldcs(reinterpret_cast<const float4*>(v) + i);
    float g[4];
    if (g16) {
      const uint2 raw = __ldcs(reinterpret_cast<const uint2*>(g16 + i * 4));
      const float2 a = unpack_bf16x2(raw.x), b = unpack_bf16x2(raw.y);
      g[0] = a.x; g[1] = a.y; g[2] = b.x; g[3] = b.y;
    } else {
      const float4 gv = __ldcs(reinterpret_cast<const float4*>(g32) + i);
      g[0] = gv.x; g[1] = gv.y; g[2] = gv.z; g[3] = gv.w;
    }
    float pp[4] = {pv.x, pv.y, pv.z, pv.w};
    float mm[4] = {mv.x, mv.y, mv.z, mv.w};
    float vs[4] = {vv.x, vv.y, vv.z, vv.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) optimizer_update<KIND>(o, g[k], o.grad_scale, w, pp[k], mm[k], vs[k]);
    __stcs(reinterpret_cast<float4*>(p) + i, make_float4(pp[0], pp[1], pp[2], pp[3]));
    __stcs(reinterpret_cast<float4*>(m) + i, make_float4(mm[0], mm[1], mm[2], mm[3]));
    if constexpr (KIND != OPT_SGD) __stcs(reinterpret_cast<float4*>(v) + i, make_float4(vs[0], vs[1], vs[2], vs[3]));
    if constexpr (EMA) ema_update4(ema + i * 4, pp, o.ema);
    if (shadow)
      __stcs(reinterpret_cast<uint2*>(shadow + i * 4), make_uint2(pack_bf16x2(pp[0], pp[1]), pack_bf16x2(pp[2], pp[3])));
    if (gzero) __stcs(reinterpret_cast<float4*>(gzero) + i, make_float4(0.f, 0.f, 0.f, 0.f));
  }
}

// DECOUPLED: AdamW, the segment values being keep factors instead of L2 decays.
template <bool EMA, bool DECOUPLED>
__global__ void __launch_bounds__(256, 6) adam_kernel(const __grid_constant__ OptStep o, float* __restrict__ p,
    float* __restrict__ m, float* __restrict__ v, const float* __restrict__ g32, const bf16* __restrict__ g16,
    bf16* __restrict__ shadow, float* __restrict__ gzero, float* __restrict__ ema, long long n4) {
  optimizer_pass<DECOUPLED ? OPT_ADAMW : OPT_ADAM, EMA>(o, p, m, v, g32, g16, shadow, gzero, ema, n4);
}

// m is the momentum buffer; v is not used.  SGD has no decoupled form in torch: the decay is L2.
template <bool EMA>
__global__ void __launch_bounds__(256, 6) sgd_kernel(const __grid_constant__ OptStep o, float* __restrict__ p,
    float* __restrict__ m, float* __restrict__ v, const float* __restrict__ g32, const bf16* __restrict__ g16,
    bf16* __restrict__ shadow, float* __restrict__ gzero, float* __restrict__ ema, long long n4) {
  optimizer_pass<OPT_SGD, EMA>(o, p, m, v, g32, g16, shadow, gzero, ema, n4);
}

// The moving average of weights that no optimizer launch covers (--freeze-layers: the frozen suffix of
// the arena, which AveragedModel still averages): ema_update of every element, the update and the
// `first` rule of the optimizer kernels' EMA.  Same footprint as adam_kernel (256 threads, no shared
// memory, evict-first streams, one grid-stride pass).  n need not be a multiple of 4: the last n % 4
// elements go through thread 0 one by one.
__global__ void __launch_bounds__(256, 6) ema_kernel(const float* __restrict__ p, float* __restrict__ ema, long long n,
                                                      const EmaCoef c) {
  const long long n4 = n / 4;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n4;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float4 pv = __ldcs(reinterpret_cast<const float4*>(p) + i);
    const float pp[4] = {pv.x, pv.y, pv.z, pv.w};
    ema_update4(ema + i * 4, pp, c);
  }
  if (blockIdx.x == 0 && threadIdx.x == 0)
    for (long long i = n4 * 4; i < n; ++i) ema[i] = ema_update(ema[i], p[i], c.d, c.a, c.first);
}

using OptKernel = void (*)(OptStep, float*, float*, float*, const float*, const bf16*, bf16*, float*, float*, long long);
static const OptKernel OPT_KERNELS[3][2] = {   // [kind][ema]
    {adam_kernel<false, false>, adam_kernel<true, false>},
    {adam_kernel<false, true>, adam_kernel<true, true>},
    {sgd_kernel<false>, sgd_kernel<true>}};

// One 256-thread CTA per 1024 elements, at most 4 CTAs per SM (Adam and AdamW: B200_ADAM_CTAS_PER_SM,
// tunable without a rebuild), so that the side-stream launches compete with the conv kernels no more than
// that.  Also registers the maximum-shared carve-out of every kernel above, once.
static int optimizer_grid(long long n4, bool adam) {
  static const int adam_per_sm = [] {
    for (const auto& kind : OPT_KERNELS)
      for (OptKernel k : kind) prefer_max_shared_carveout(reinterpret_cast<const void*>(k));
    prefer_max_shared_carveout(reinterpret_cast<const void*>(ema_kernel));
    const char* e = getenv("B200_ADAM_CTAS_PER_SM");
    const int v = e ? atoi(e) : 4;
    return v >= 1 && v <= 16 ? v : 4;
  }();
  const long long cap = static_cast<long long>(sm_count()) * (adam ? adam_per_sm : 4);
  return static_cast<int>(n4 / 256 + 1 < cap ? n4 / 256 + 1 : cap);
}

void optimizer_fused(const OptStep& o, float* p, float* m, float* v, const float* g32, const bf16* g16,
                     bf16* shadow, float* gzero, float* ema, long long n, cudaStream_t s) {
  const char* what = o.kind == OPT_SGD ? "sgd_fused" : "adam_fused";
  if (o.kind != OPT_ADAM && o.kind != OPT_ADAMW && o.kind != OPT_SGD)
    throw std::runtime_error("[b200] optimizer_fused: LAMB and LARS run as layerwise_phase1 / layerwise_phase2");
  if (n % 4) throw std::runtime_error(std::string("[b200] ") + what + ": n must be a multiple of 4");
  const int blocks = optimizer_grid(n / 4, o.kind != OPT_SGD);
  OPT_KERNELS[o.kind][ema != nullptr]<<<blocks, 256, 0, s>>>(o, p, m, v, g32, g16, shadow, gzero, ema, n / 4);
  count_launch();
  check_last(what);
}

// Runs once per EMA step; its cost in the step is measured by bench/freeze_bench.py.
void ema_fused(const float* p, float* ema, long long n, double decay, bool first, cudaStream_t s) {
  if (n <= 0) return;
  ema_kernel<<<optimizer_grid(n / 4, false), 256, 0, s>>>(p, ema, n, ema_coef(decay, first));
  count_launch();
  check_last("ema_fused");
}

// ------------------------------------------------------------------ layer-wise adaptive (LAMB, LARS)
// Same footprint as adam_kernel (256 threads, at most 4 CTAs per SM in all, evict-first streams, the
// maximum-shared carve-out), plus 72 bytes of static shared memory for the block reduction.  Every CTA
// works inside one segment (one tensor): it finds its segment from the CTA table and grid-strides over
// the segment alone, so that its partial sums belong to one tensor.

// The segment of this CTA: the last k with cta0[k] <= blockIdx.x.
__device__ __forceinline__ int lw_segment(const LayerwiseLaunch& L) {
  int k = 0;
  while (k + 1 < L.n && static_cast<int>(blockIdx.x) >= L.cta0[k + 1]) ++k;
  return k;
}

// Sum over the block of (a, b) in a fixed order: a butterfly within each warp, then thread 0 adds the
// eight warp sums in warp order.  The result is valid in thread 0.
__device__ __forceinline__ float2 lw_block_sum(float a, float b, float2* red) {
  for (int o = 16; o; o >>= 1) {
    a = __fadd_rn(a, __shfl_xor_sync(0xffffffffu, a, o));
    b = __fadd_rn(b, __shfl_xor_sync(0xffffffffu, b, o));
  }
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = make_float2(a, b);
  __syncthreads();
  float2 t = make_float2(0.f, 0.f);
  if (threadIdx.x == 0)
    for (int w = 0; w < 8; ++w) t = make_float2(__fadd_rn(t.x, red[w].x), __fadd_rn(t.y, red[w].y));
  return t;
}

__device__ __forceinline__ void lw_load_grad(const float* __restrict__ g32, const bf16* __restrict__ g16, long long i,
                                             float* g) {
  if (g16) {
    const uint2 raw = __ldcs(reinterpret_cast<const uint2*>(g16 + i * 4));
    const float2 a = unpack_bf16x2(raw.x), b = unpack_bf16x2(raw.y);
    g[0] = a.x; g[1] = a.y; g[2] = b.x; g[3] = b.y;
  } else {
    const float4 gv = __ldcs(reinterpret_cast<const float4*>(g32) + i);
    g[0] = gv.x; g[1] = gv.y; g[2] = gv.z; g[3] = gv.w;
  }
}

// Phase 1.  LAMB: m, v updated from g * gscale, partials (sum p^2, sum u^2), gzero cleared.
// LARS: partials (sum p^2, sum (g * gscale)^2); nothing written but the partials.
template <int KIND>
__global__ void __launch_bounds__(256, 6) layerwise_norms_kernel(const __grid_constant__ OptStep o,
    const __grid_constant__ LayerwiseLaunch L, const float* __restrict__ p, float* __restrict__ m,
    float* __restrict__ v, const float* __restrict__ g32, const bf16* __restrict__ g16, float* __restrict__ gzero,
    float* __restrict__ ws) {
  __shared__ float2 red[8];
  const int k = lw_segment(L);
  const int j = static_cast<int>(blockIdx.x) - L.cta0[k];
  const long long stride = static_cast<long long>(L.cta0[k + 1] - L.cta0[k]) * blockDim.x;
  const float wd = L.wd[k];
  float sp = 0.f, sq = 0.f;
  for (long long i = L.start4[k] + static_cast<long long>(j) * blockDim.x + threadIdx.x; i < L.start4[k + 1];
       i += stride) {
    const float4 pv = __ldcs(reinterpret_cast<const float4*>(p) + i);
    const float pp[4] = {pv.x, pv.y, pv.z, pv.w};
    float g[4];
    lw_load_grad(g32, g16, i, g);
    if constexpr (KIND == OPT_LAMB) {
      const float4 mv = __ldcs(reinterpret_cast<const float4*>(m) + i);
      const float4 vv = __ldcs(reinterpret_cast<const float4*>(v) + i);
      float mm[4] = {mv.x, mv.y, mv.z, mv.w}, vs[4] = {vv.x, vv.y, vv.z, vv.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        lamb_moments(__fmul_rn(g[e], o.grad_scale), mm[e], vs[e], o.beta1, o.beta2);
        const float u = lamb_direction(mm[e], vs[e], pp[e], o.bc1_inv, o.bc2_inv_sqrt, o.eps, wd);
        sp = __fmaf_rn(pp[e], pp[e], sp);
        sq = __fmaf_rn(u, u, sq);
      }
      __stcs(reinterpret_cast<float4*>(m) + i, make_float4(mm[0], mm[1], mm[2], mm[3]));
      __stcs(reinterpret_cast<float4*>(v) + i, make_float4(vs[0], vs[1], vs[2], vs[3]));
      if (gzero) __stcs(reinterpret_cast<float4*>(gzero) + i, make_float4(0.f, 0.f, 0.f, 0.f));
    } else {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float gk = __fmul_rn(g[e], o.grad_scale);
        sp = __fmaf_rn(pp[e], pp[e], sp);
        sq = __fmaf_rn(gk, gk, sq);
      }
    }
  }
  const float2 t = lw_block_sum(sp, sq, red);
  if (threadIdx.x == 0) reinterpret_cast<float2*>(ws)[L.slot[k] + j] = t;
}

// Phase 2: the tensor's ratio from its partials (every CTA of the segment adds the same slots in the same
// order), then LAMB: p -= lr (r u) with u recomputed from the stored moments; LARS: lars_update on the
// gradient.  Then the shadow, the EMA and (LARS) the gradient zeroing.
template <int KIND, bool EMA>
__global__ void __launch_bounds__(256, 6) layerwise_update_kernel(const __grid_constant__ OptStep o,
    const __grid_constant__ LayerwiseLaunch L, float* __restrict__ p, float* __restrict__ m,
    const float* __restrict__ v, const float* __restrict__ g32, const bf16* __restrict__ g16,
    bf16* __restrict__ shadow, float* __restrict__ gzero, float* __restrict__ ema, const float* __restrict__ ws,
    float* __restrict__ ratio) {
  __shared__ float2 red[8];
  __shared__ float s_ratio;
  const int k = lw_segment(L);
  float a = 0.f, b = 0.f;
  for (int s = threadIdx.x; s < L.nslots[k]; s += blockDim.x) {
    const float2 w = reinterpret_cast<const float2*>(ws)[L.slot[k] + s];
    a = __fadd_rn(a, w.x);
    b = __fadd_rn(b, w.y);
  }
  const float2 t = lw_block_sum(a, b, red);
  const float wd = L.wd[k];
  if (threadIdx.x == 0) {
    const float r = KIND == OPT_LAMB ? lamb_ratio(t.x, t.y, wd) : lars_ratio(t.x, t.y, wd, L.trust_coeff, L.trust_eps);
    s_ratio = r;
    if (ratio && static_cast<int>(blockIdx.x) == L.cta0[k]) ratio[L.tensor[k]] = r;
  }
  __syncthreads();
  const float r = s_ratio;
  const int j = static_cast<int>(blockIdx.x) - L.cta0[k];
  const long long stride = static_cast<long long>(L.cta0[k + 1] - L.cta0[k]) * blockDim.x;
  for (long long i = L.start4[k] + static_cast<long long>(j) * blockDim.x + threadIdx.x; i < L.start4[k + 1];
       i += stride) {
    const float4 pv = __ldcs(reinterpret_cast<const float4*>(p) + i);
    const float4 mv = __ldcs(reinterpret_cast<const float4*>(m) + i);
    float pp[4] = {pv.x, pv.y, pv.z, pv.w}, mm[4] = {mv.x, mv.y, mv.z, mv.w};
    if constexpr (KIND == OPT_LAMB) {
      const float4 vv = __ldcs(reinterpret_cast<const float4*>(v) + i);
      const float vs[4] = {vv.x, vv.y, vv.z, vv.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float u = lamb_direction(mm[e], vs[e], pp[e], o.bc1_inv, o.bc2_inv_sqrt, o.eps, wd);
        pp[e] = __fmaf_rn(-o.lr, __fmul_rn(r, u), pp[e]);
      }
    } else {
      float g[4];
      lw_load_grad(g32, g16, i, g);
#pragma unroll
      for (int e = 0; e < 4; ++e) lars_update(g[e], o.grad_scale, pp[e], mm[e], o.lr, o.momentum, wd, r, o.first);
      __stcs(reinterpret_cast<float4*>(m) + i, make_float4(mm[0], mm[1], mm[2], mm[3]));
      if (gzero) __stcs(reinterpret_cast<float4*>(gzero) + i, make_float4(0.f, 0.f, 0.f, 0.f));
    }
    __stcs(reinterpret_cast<float4*>(p) + i, make_float4(pp[0], pp[1], pp[2], pp[3]));
    if constexpr (EMA) ema_update4(ema + i * 4, pp, o.ema);
    if (shadow)
      __stcs(reinterpret_cast<uint2*>(shadow + i * 4), make_uint2(pack_bf16x2(pp[0], pp[1]), pack_bf16x2(pp[2], pp[3])));
  }
}

using LwNormsKernel = void (*)(OptStep, LayerwiseLaunch, const float*, float*, float*, const float*, const bf16*,
                               float*, float*);
using LwUpdateKernel = void (*)(OptStep, LayerwiseLaunch, float*, float*, const float*, const float*, const bf16*,
                                bf16*, float*, float*, const float*, float*);
static const LwNormsKernel LW_NORMS[2] = {layerwise_norms_kernel<OPT_LAMB>, layerwise_norms_kernel<OPT_LARS>};
static const LwUpdateKernel LW_UPDATE[2][2] = {   // [lars][ema]
    {layerwise_update_kernel<OPT_LAMB, false>, layerwise_update_kernel<OPT_LAMB, true>},
    {layerwise_update_kernel<OPT_LARS, false>, layerwise_update_kernel<OPT_LARS, true>}};

long long layerwise_max_grid() {
  static const bool once = [] {
    for (auto k : LW_NORMS) prefer_max_shared_carveout(reinterpret_cast<const void*>(k));
    for (const auto& kind : LW_UPDATE)
      for (auto k : kind) prefer_max_shared_carveout(reinterpret_cast<const void*>(k));
    return true;
  }();
  (void)once;
  return static_cast<long long>(sm_count()) * 4;
}

LayerwiseLaunch make_layerwise_launch(const char* op, long long n, const std::vector<int64_t>& starts,
                                      const std::vector<int64_t>& ctas, const std::vector<int64_t>& slots,
                                      const std::vector<int64_t>& nslots, const std::vector<int64_t>& tensors,
                                      const std::vector<double>& wds, double trust_coeff, double trust_eps,
                                      long long max_grid) {
  auto check = [op](bool ok, const auto&... msg) {
    if (ok) return;
    std::ostringstream s;
    ((s << op) << ... << msg);
    throw std::runtime_error(s.str());
  };
  const size_t ns = starts.size();
  check(ns >= 1 && ns <= static_cast<size_t>(LW_MAX_SEGMENTS), ": 1 to ", LW_MAX_SEGMENTS, " segments per launch, got ",
        ns);
  check(ctas.size() == ns && slots.size() == ns && nslots.size() == ns && tensors.size() == ns && wds.size() == ns,
        ": starts, ctas, slots, nslots, tensors and wds must have the same length");
  check(n > 0 && n % 4 == 0, ": n must be a positive multiple of 4, got ", n);
  LayerwiseLaunch L{};
  L.n = static_cast<int>(ns);
  L.trust_coeff = static_cast<float>(trust_coeff);
  L.trust_eps = static_cast<float>(trust_eps);
  long long grid = 0;
  for (size_t k = 0; k < ns; ++k) {
    check(k > 0 || starts[0] == 0, ": the first segment must start at 0");
    check(k == 0 || starts[k] > starts[k - 1], ": segment starts must increase");
    check(starts[k] % 4 == 0 && starts[k] < n, ": segment start ", starts[k], " is not a multiple of 4 inside ", n);
    check(ctas[k] >= 1, ": every segment needs a CTA");
    check(slots[k] >= 0 && nslots[k] >= 0 && tensors[k] >= 0, ": slots, slot counts and tensors must be >= 0");
    check(std::isfinite(wds[k]) && wds[k] >= 0.0, ": weight decays must be finite and >= 0, got ", wds[k]);
    L.cta0[k] = static_cast<int>(grid);
    L.start4[k] = starts[k] / 4;
    L.slot[k] = static_cast<int>(slots[k]);
    L.nslots[k] = static_cast<int>(nslots[k]);
    L.tensor[k] = static_cast<int>(tensors[k]);
    L.wd[k] = static_cast<float>(wds[k]);
    grid += ctas[k];
  }
  check(grid <= max_grid, ": ", grid, " CTAs exceed the cap of ", max_grid);
  L.cta0[ns] = static_cast<int>(grid);
  L.start4[ns] = n / 4;
  return L;
}

void layerwise_phase1(const OptStep& o, const LayerwiseLaunch& L, float* p, float* m, float* v, const float* g32,
                      const bf16* g16, float* gzero, float* ws, cudaStream_t s) {
  if (o.kind != OPT_LAMB && o.kind != OPT_LARS) throw std::runtime_error("[b200] layerwise_phase1: LAMB or LARS");
  layerwise_max_grid();
  LW_NORMS[o.kind == OPT_LARS]<<<L.cta0[L.n], 256, 0, s>>>(o, L, p, m, v, g32, g16, gzero, ws);
  count_launch();
  check_last("layerwise_phase1");
}

void layerwise_phase2(const OptStep& o, const LayerwiseLaunch& L, float* p, float* m, float* v, const float* g32,
                      const bf16* g16, bf16* shadow, float* gzero, float* ema, const float* ws, float* ratio,
                      cudaStream_t s) {
  if (o.kind != OPT_LAMB && o.kind != OPT_LARS) throw std::runtime_error("[b200] layerwise_phase2: LAMB or LARS");
  layerwise_max_grid();
  LW_UPDATE[o.kind == OPT_LARS][ema != nullptr]<<<L.cta0[L.n], 256, 0, s>>>(o, L, p, m, v, g32, g16, shadow, gzero,
                                                                              ema, ws, ratio);
  count_launch();
  check_last("layerwise_phase2");
}

}  // namespace b200
