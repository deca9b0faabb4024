// Memory-bound kernels of the training step: pooling (fwd / fused ReLU+pool backward), adaptive
// average pool, bias gradients, FC epilogues (bias + ReLU + Philox dropout), casts.
// All activations are NHWC bf16; every thread moves 16-byte vectors (8 channels).
#include <stdexcept>
#include <string>

#include "api.h"
#include "ptx.cuh"

namespace b200 {

static inline int ceil_div_ll(long long a, long long b) { return static_cast<int>((a + b - 1) / b); }

// ------------------------------------------------------------------------------------- Philox
// Philox4x32-10 counter RNG: stateless, so the dropout mask of element i is a pure function of
// (seed, offset, i) -- nothing is stored between forward and backward.
__device__ __forceinline__ uint4 philox4x32_10(uint2 key, uint4 ctr) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(M0, ctr.x), lo0 = M0 * ctr.x;
    const uint32_t hi1 = __umulhi(M1, ctr.z), lo1 = M1 * ctr.z;
    ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
    key.x += W0;
    key.y += W1;
  }
  return ctr;
}

// ------------------------------------------------------------------------------------ maxpool
__device__ __forceinline__ void unpack8(const uint4& v, float (&f)[8]) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 t = unpack_bf16x2(w[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  return make_uint4(pack_bf16x2(f[0], f[1]), pack_bf16x2(f[2], f[3]), pack_bf16x2(f[4], f[5]),
                    pack_bf16x2(f[6], f[7]));
}

// Floor mode: the output is floor(H/2) x floor(W/2); at odd H or W the last row / column lies in no
// window and is never read.
__global__ void maxpool2x2_fwd_kernel(const bf16* __restrict__ x, bf16* __restrict__ y, int N, int H,
                                      int W, int C) {
  const int OH = H / 2, OW = W / 2, C8 = C / 8;
  const long long total = static_cast<long long>(N) * OH * OW * C8;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c8 = i % C8;
    long long r = i / C8;
    const int ow = r % OW; r /= OW;
    const int oh = r % OH;
    const int n = r / OH;
    const bf16* base = x + ((static_cast<long long>(n) * H + 2 * oh) * W + 2 * ow) * C + c8 * 8;
    float a[8], b[8], c[8], d[8], o[8];
    unpack8(ld_nc_v4(base), a);
    unpack8(ld_nc_v4(base + C), b);
    unpack8(ld_nc_v4(base + static_cast<long long>(W) * C), c);
    unpack8(ld_nc_v4(base + static_cast<long long>(W) * C + C), d);
#pragma unroll
    for (int k = 0; k < 8; ++k) o[k] = fmaxf(fmaxf(a[k], b[k]), fmaxf(c[k], d[k]));
    *reinterpret_cast<uint4*>(y + ((static_cast<long long>(n) * OH + oh) * OW + ow) * C + c8 * 8) = pack8(o);
  }
}

void maxpool2x2_fwd(const bf16* x, bf16* y, int N, int H, int W, int C, cudaStream_t s) {
  // floor mode (torch's MaxPool2d(2, 2)): an odd last row / column is never read
  if (C % 8 || H < 2 || W < 2) throw std::runtime_error("[b200] maxpool2x2: need C%8==0 and H,W >= 2");
  const long long total = static_cast<long long>(N) * (H / 2) * (W / 2) * (C / 8);
  const int blocks = min(ceil_div_ll(total, 256), sm_count() * 16);
  maxpool2x2_fwd_kernel<<<blocks, 256, 0, s>>>(x, y, N, H, W, C);
  count_launch();
  check_last("maxpool2x2_fwd");
}

// Backward of [ReLU -> maxpool2x2] in one pass: the gradient of a window goes to its first
// maximal element (torch's tie rule) and only if that maximum is positive (ReLU mask).  Optionally
// also accumulates colsum[c] += sum of dz over pixels (the conv layer's bias gradient): the grid
// stride is a multiple of C/8, so a thread always sees the same 8 channels and keeps them in
// registers; one shared-memory reduction and C global atomics per block at the end.
// ODD (odd H or W, floor mode): the last row / column lies in no window and its dz is stored as 0,
// by the threads of the last window row / column; the even-size kernel is the ODD = false body.
template <bool ODD>
__device__ __forceinline__ void maxpool2x2_relu_bwd_body(const bf16* __restrict__ y, const bf16* __restrict__ dp,
                                                         bf16* __restrict__ dz, float* __restrict__ colsum, int N,
                                                         int H, int W, int C) {
  extern __shared__ float s_sum[];      // [C] when colsum
  const int OH = H / 2, OW = W / 2, C8 = C / 8;
  const long long total = static_cast<long long>(N) * OH * OW * C8;
  float bsum[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (colsum) {
    for (int i = threadIdx.x; i < C; i += blockDim.x) s_sum[i] = 0.f;
    __syncthreads();
  }
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c8 = i % C8;
    long long r = i / C8;
    const int ow = r % OW; r /= OW;
    const int oh = r % OH;
    const int n = r / OH;
    const long long o00 = ((static_cast<long long>(n) * H + 2 * oh) * W + 2 * ow) * C + c8 * 8;
    const long long rowstride = static_cast<long long>(W) * C;
    float a[8], b[8], c[8], d[8], g[8];
    unpack8(ld_nc_v4(y + o00), a);
    unpack8(ld_nc_v4(y + o00 + C), b);
    unpack8(ld_nc_v4(y + o00 + rowstride), c);
    unpack8(ld_nc_v4(y + o00 + rowstride + C), d);
    unpack8(ld_nc_v4(dp + ((static_cast<long long>(n) * OH + oh) * OW + ow) * C + c8 * 8), g);
    float ra[8], rb[8], rc[8], rd[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const float m = fmaxf(fmaxf(a[k], b[k]), fmaxf(c[k], d[k]));
      const float gg = m > 0.f ? g[k] : 0.f;
      const bool ia = a[k] == m;
      const bool ib = !ia && b[k] == m;
      const bool ic = !ia && !ib && c[k] == m;
      const bool id = !ia && !ib && !ic;
      ra[k] = ia ? gg : 0.f; rb[k] = ib ? gg : 0.f; rc[k] = ic ? gg : 0.f; rd[k] = id ? gg : 0.f;
      bsum[k] += gg;
    }
    *reinterpret_cast<uint4*>(dz + o00) = pack8(ra);
    *reinterpret_cast<uint4*>(dz + o00 + C) = pack8(rb);
    *reinterpret_cast<uint4*>(dz + o00 + rowstride) = pack8(rc);
    *reinterpret_cast<uint4*>(dz + o00 + rowstride + C) = pack8(rd);
    if constexpr (ODD) {
      const uint4 z = make_uint4(0u, 0u, 0u, 0u);
      const bool last_h = (H & 1) && oh == OH - 1, last_w = (W & 1) && ow == OW - 1;
      if (last_h) {
        *reinterpret_cast<uint4*>(dz + o00 + 2 * rowstride) = z;
        *reinterpret_cast<uint4*>(dz + o00 + 2 * rowstride + C) = z;
      }
      if (last_w) {
        *reinterpret_cast<uint4*>(dz + o00 + 2 * C) = z;
        *reinterpret_cast<uint4*>(dz + o00 + rowstride + 2 * C) = z;
      }
      if (last_h && last_w) *reinterpret_cast<uint4*>(dz + o00 + 2 * rowstride + 2 * C) = z;
    }
  }
  if (colsum) {
    const int c8 = (blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x) % C8;
#pragma unroll
    for (int k = 0; k < 8; ++k) atomicAdd(&s_sum[c8 * 8 + k], bsum[k]);
    __syncthreads();
    for (int i = threadIdx.x; i < C; i += blockDim.x)
      if (s_sum[i] != 0.f) atomicAdd(colsum + i, s_sum[i]);
  }
}

__global__ void maxpool2x2_relu_bwd_kernel(const bf16* __restrict__ y, const bf16* __restrict__ dp,
                                           bf16* __restrict__ dz, float* __restrict__ colsum, int N, int H,
                                           int W, int C) {
  maxpool2x2_relu_bwd_body<false>(y, dp, dz, colsum, N, H, W, C);
}
__global__ void maxpool2x2_relu_bwd_odd_kernel(const bf16* __restrict__ y, const bf16* __restrict__ dp,
                                               bf16* __restrict__ dz, float* __restrict__ colsum, int N, int H,
                                               int W, int C) {
  maxpool2x2_relu_bwd_body<true>(y, dp, dz, colsum, N, H, W, C);
}

void maxpool2x2_relu_bwd(const bf16* y, const bf16* dp, bf16* dz, float* colsum, int N, int H, int W,
                         int C, cudaStream_t s) {
  if (C % 8 || H < 2 || W < 2) throw std::runtime_error("[b200] maxpool2x2_bwd: need C%8==0 and H,W >= 2");
  if (colsum && 256 % (C / 8) != 0)
    throw std::runtime_error("[b200] maxpool2x2_bwd: fused column sum needs C/8 to divide 256");
  const long long total = static_cast<long long>(N) * (H / 2) * (W / 2) * (C / 8);
  const int blocks = min(ceil_div_ll(total, 256), sm_count() * 16);
  const size_t smem = colsum ? C * sizeof(float) : 0;
  if ((H | W) & 1)
    maxpool2x2_relu_bwd_odd_kernel<<<blocks, 256, smem, s>>>(y, dp, dz, colsum, N, H, W, C);
  else
    maxpool2x2_relu_bwd_kernel<<<blocks, 256, smem, s>>>(y, dp, dz, colsum, N, H, W, C);
  count_launch();
  check_last("maxpool2x2_relu_bwd");
}

// Backward of the pool fused into the conv epilogue (ConvPolicy::epilogue_pool).  One
// thread = one pooled pixel x 8 channels: reads 16 B of dp and the chunk's mask words, writes the
// four 16-byte pieces of dz.  Reads 3/8 of a full-resolution tensor instead of 1 1/2.
__global__ void unpool2x2_kernel(const bf16* __restrict__ dp, const uint32_t* __restrict__ mask,
                                 bf16* __restrict__ dz, float* __restrict__ colsum, int N, int H, int W,
                                 int C) {
  extern __shared__ float s_sum[];      // [C] when colsum
  const int OH = H / 2, OW = W / 2, C8 = C / 8, C32 = C / 32;
  const long long total = static_cast<long long>(N) * OH * OW * C8;
  float bsum[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (colsum) {
    for (int i = threadIdx.x; i < C; i += blockDim.x) s_sum[i] = 0.f;
    __syncthreads();
  }
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c8 = i % C8;
    long long r = i / C8;                                   // pooled pixel index
    const long long ppix = r;
    const int ow = r % OW; r /= OW;
    const int oh = r % OH;
    const int n = r / OH;
    const uint4 mk = *reinterpret_cast<const uint4*>(mask + (ppix * C32 + (c8 >> 2)) * 4);
    const int sh = (c8 & 3) * 8;
    const uint32_t b0 = mk.x >> sh, b1 = mk.y >> sh, pos = mk.z >> sh;
    float g[8], ra[8], rb[8], rc[8], rd[8];
    unpack8(ld_nc_v4(dp + ppix * C + c8 * 8), g);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const float gg = ((pos >> k) & 1u) ? g[k] : 0.f;
      const uint32_t idx = ((b0 >> k) & 1u) | (((b1 >> k) & 1u) << 1);
      ra[k] = idx == 0u ? gg : 0.f; rb[k] = idx == 1u ? gg : 0.f;
      rc[k] = idx == 2u ? gg : 0.f; rd[k] = idx == 3u ? gg : 0.f;
      bsum[k] += gg;
    }
    const long long o00 = ((static_cast<long long>(n) * H + 2 * oh) * W + 2 * ow) * C + c8 * 8;
    const long long rowstride = static_cast<long long>(W) * C;
    *reinterpret_cast<uint4*>(dz + o00) = pack8(ra);
    *reinterpret_cast<uint4*>(dz + o00 + C) = pack8(rb);
    *reinterpret_cast<uint4*>(dz + o00 + rowstride) = pack8(rc);
    *reinterpret_cast<uint4*>(dz + o00 + rowstride + C) = pack8(rd);
  }
  if (colsum) {
    const int c8 = (blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x) % C8;
#pragma unroll
    for (int k = 0; k < 8; ++k) atomicAdd(&s_sum[c8 * 8 + k], bsum[k]);
    __syncthreads();
    for (int i = threadIdx.x; i < C; i += blockDim.x)
      if (s_sum[i] != 0.f) atomicAdd(colsum + i, s_sum[i]);
  }
}

void unpool2x2(const bf16* dp, const uint32_t* mask, bf16* dz, float* colsum, int N, int H, int W, int C,
               cudaStream_t s) {
  if (C % 32 || H % 2 || W % 2) throw std::runtime_error("[b200] unpool2x2: need C%32==0 and even H,W");
  if (colsum && 256 % (C / 8) != 0)
    throw std::runtime_error("[b200] unpool2x2: fused column sum needs C/8 to divide 256");
  const long long total = static_cast<long long>(N) * (H / 2) * (W / 2) * (C / 8);
  const int blocks = min(ceil_div_ll(total, 256), sm_count() * 16);
  unpool2x2_kernel<<<blocks, 256, colsum ? C * sizeof(float) : 0, s>>>(dp, mask, dz, colsum, N, H, W, C);
  count_launch();
  check_last("unpool2x2");
}

// ---------------------------------------------------------------------- adaptive average pool
__device__ __forceinline__ int ap_start(int o, int in, int out) { return (o * in) / out; }
__device__ __forceinline__ int ap_end(int o, int in, int out) { return ((o + 1) * in + out - 1) / out; }

__global__ void adaptive_avgpool_fwd_kernel(const bf16* __restrict__ x, bf16* __restrict__ y, int N,
                                            int H, int W, int C, int OH, int OW) {
  const int C8 = C / 8;
  const long long total = static_cast<long long>(N) * OH * OW * C8;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c8 = i % C8;
    long long r = i / C8;
    const int ow = r % OW; r /= OW;
    const int oh = r % OH;
    const int n = r / OH;
    const int h0 = ap_start(oh, H, OH), h1 = ap_end(oh, H, OH);
    const int w0 = ap_start(ow, W, OW), w1 = ap_end(ow, W, OW);
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int h = h0; h < h1; ++h)
      for (int w = w0; w < w1; ++w) {
        float v[8];
        unpack8(ld_nc_v4(x + ((static_cast<long long>(n) * H + h) * W + w) * C + c8 * 8), v);
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[k] += v[k];
      }
    const float inv = 1.f / static_cast<float>((h1 - h0) * (w1 - w0));
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] *= inv;
    *reinterpret_cast<uint4*>(y + ((static_cast<long long>(n) * OH + oh) * OW + ow) * C + c8 * 8) = pack8(acc);
  }
}

__global__ void adaptive_avgpool_bwd_kernel(const bf16* __restrict__ dy, bf16* __restrict__ dx, int N,
                                            int H, int W, int C, int OH, int OW) {
  const int C8 = C / 8;
  const long long total = static_cast<long long>(N) * H * W * C8;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c8 = i % C8;
    long long r = i / C8;
    const int w = r % W; r /= W;
    const int h = r % H;
    const int n = r / H;
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int oh = 0; oh < OH; ++oh) {
      const int h0 = ap_start(oh, H, OH), h1 = ap_end(oh, H, OH);
      if (h < h0 || h >= h1) continue;
      for (int ow = 0; ow < OW; ++ow) {
        const int w0 = ap_start(ow, W, OW), w1 = ap_end(ow, W, OW);
        if (w < w0 || w >= w1) continue;
        float v[8];
        unpack8(ld_nc_v4(dy + ((static_cast<long long>(n) * OH + oh) * OW + ow) * C + c8 * 8), v);
        const float inv = 1.f / static_cast<float>((h1 - h0) * (w1 - w0));
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[k] += v[k] * inv;
      }
    }
    *reinterpret_cast<uint4*>(dx + ((static_cast<long long>(n) * H + h) * W + w) * C + c8 * 8) = pack8(acc);
  }
}

void adaptive_avgpool_fwd(const bf16* x, bf16* y, int N, int H, int W, int C, int OH, int OW,
                          cudaStream_t s) {
  if (C % 8) throw std::runtime_error("[b200] adaptive_avgpool: C%8 != 0");
  const long long total = static_cast<long long>(N) * OH * OW * (C / 8);
  adaptive_avgpool_fwd_kernel<<<min(ceil_div_ll(total, 256), sm_count() * 16), 256, 0, s>>>(x, y, N, H, W, C, OH, OW);
  count_launch();
  check_last("adaptive_avgpool_fwd");
}
void adaptive_avgpool_bwd(const bf16* dy, bf16* dx, int N, int H, int W, int C, int OH, int OW,
                          cudaStream_t s) {
  if (C % 8) throw std::runtime_error("[b200] adaptive_avgpool: C%8 != 0");
  const long long total = static_cast<long long>(N) * H * W * (C / 8);
  adaptive_avgpool_bwd_kernel<<<min(ceil_div_ll(total, 256), sm_count() * 16), 256, 0, s>>>(dy, dx, N, H, W, C, OH, OW);
  count_launch();
  check_last("adaptive_avgpool_bwd");
}

// ---------------------------------------------------------------------------------- bias grad
// db[c] += scale * sum_r dz[r][c].  Block = CG column groups (8 channels each) x RL row lanes.
// PARTIAL: block x stores its row of sums to db[x][C] instead (the sum inside a block has a fixed order;
// only the order in which the blocks' atomics arrive does not), for splitk_reduce to add up in block order.
template <bool PARTIAL>
__global__ void bias_grad_kernel(const bf16* __restrict__ dz, float* __restrict__ db, long long rows,
                                 int C, float scale, int CG, int RL, long long rows_per_block) {
  extern __shared__ float red[];      // [RL][CG*8]
  const int cg = threadIdx.x % CG;
  const int rl = threadIdx.x / CG;
  const int col8 = blockIdx.y * CG + cg;
  const bool active = col8 * 8 < C;
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  const long long r0 = blockIdx.x * rows_per_block;
  const long long r1 = min(rows, r0 + rows_per_block);
  if (active) {
    long long r = r0 + rl;
    // 4 independent 16-byte loads in flight per thread
    for (; r + 3LL * RL < r1; r += 4LL * RL) {
      uint4 raw[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) raw[u] = ld_nc_v4(dz + (r + static_cast<long long>(u) * RL) * C + col8 * 8);
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        float v[8];
        unpack8(raw[u], v);
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[k] += v[k];
      }
    }
    for (; r < r1; r += RL) {
      float v[8];
      unpack8(ld_nc_v4(dz + r * C + col8 * 8), v);
#pragma unroll
      for (int k = 0; k < 8; ++k) acc[k] += v[k];
    }
  }
#pragma unroll
  for (int k = 0; k < 8; ++k) red[(rl * CG + cg) * 8 + k] = acc[k];
  __syncthreads();
  if (rl == 0 && active) {
    for (int j = 1; j < RL; ++j)
#pragma unroll
      for (int k = 0; k < 8; ++k) acc[k] += red[(j * CG + cg) * 8 + k];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      if constexpr (PARTIAL) db[static_cast<long long>(blockIdx.x) * C + col8 * 8 + k] = acc[k] * scale;
      else atomicAdd(db + col8 * 8 + k, acc[k] * scale);
    }
  }
}
// Generic fallback (C not a multiple of 8, e.g. the 3-class logits): one thread per channel.
__global__ void bias_grad_small_kernel(const bf16* __restrict__ dz, float* __restrict__ db,
                                       long long rows, int C, int ld, float scale) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float acc = 0.f;
  for (long long r = 0; r < rows; ++r) acc += __bfloat162float(dz[r * ld + c]);
  atomicAdd(db + c, acc * scale);
}

// Block shape and row blocks of bias_grad for `rows` x C on `sms` SMs; returns the row blocks (grid.x).
static int bias_grad_shape(long long rows, int C, int sms, int* CG, int* RL, long long* rpb) {
  const int c8 = C / 8;
  *CG = c8 < 256 ? c8 : 256;
  *RL = 256 / *CG;
  if (*RL < 1) *RL = 1;
  long long nblk = (rows + *RL * 16 - 1) / (*RL * 16);
  const long long cap = static_cast<long long>(sms) * 8 / ((c8 + *CG - 1) / *CG);
  if (nblk > cap) nblk = cap;
  if (nblk < 1) nblk = 1;
  *rpb = (rows + nblk - 1) / nblk;
  return static_cast<int>((rows + *rpb - 1) / *rpb);
}
int colsum_partial_blocks(long long rows, int C, int sms) {
  int CG, RL;
  long long rpb;
  return bias_grad_shape(rows, C, sms, &CG, &RL, &rpb);
}

template <bool PARTIAL>
static int bias_grad_launch(const bf16* dz, float* db, long long ws_elems, long long rows, int C, float scale,
                            cudaStream_t s) {
  if (C % 8 != 0) throw std::runtime_error("[b200] bias_grad: C%8 != 0 (use bias_grad_ld)");
  int CG, RL;
  long long rpb;
  const int blocks = bias_grad_shape(rows, C, sm_count(), &CG, &RL, &rpb);
  if (PARTIAL && (!db || ws_elems < static_cast<long long>(blocks) * C))
    throw std::runtime_error("[b200] colsum_partial: the workspace must hold " + std::to_string(blocks) +
                             " rows of " + std::to_string(C) + " floats");
  const int threads = CG * RL;
  dim3 grid(blocks, (C / 8 + CG - 1) / CG);
  bias_grad_kernel<PARTIAL><<<grid, threads, threads * 8 * sizeof(float), s>>>(dz, db, rows, C, scale, CG, RL, rpb);
  count_launch();
  check_last(PARTIAL ? "colsum_partial" : "bias_grad");
  return blocks;
}
void bias_grad(const bf16* dz, float* db, long long rows, int C, float scale, cudaStream_t s) {
  bias_grad_launch<false>(dz, db, 0, rows, C, scale, s);
}
int colsum_partial(const bf16* dz, float* ws, long long ws_elems, long long rows, int C, float scale, cudaStream_t s) {
  return bias_grad_launch<true>(dz, ws, ws_elems, rows, C, scale, s);
}

// ------------------------------------------------------------------------- split-K reduction
// dst[i] = (accumulate ? dst[i] : 0) + alpha * (((ws[0][i] + ws[1][i]) + ws[2][i]) + ...): the slices a
// PARTIAL epilogue stored, added in split order.  Every add and the product round to fp32 on their own
// (no contraction into an FMA), so the result is a function of the slices alone.  Bandwidth-bound: one
// float4 per thread and pass, four slices' loads in flight, the workspace read once and not kept in L2.
__device__ __forceinline__ uint64_t l2_evict_first_policy() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ float4 ld_evict_first_v4(const float* p, uint64_t pol) {
  float4 v;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.f32 {%0, %1, %2, %3}, [%4], %5;"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p), "l"(pol));
  return v;
}
__device__ __forceinline__ void add4(float4& a, const float4& b) {
  a.x = __fadd_rn(a.x, b.x); a.y = __fadd_rn(a.y, b.y); a.z = __fadd_rn(a.z, b.z); a.w = __fadd_rn(a.w, b.w);
}
__global__ void __launch_bounds__(256)
splitk_reduce_kernel(const float* __restrict__ ws, float* __restrict__ dst, long long n, long long slice,
                     int splits, float alpha, int accumulate) {
  const long long n4 = n / 4;
  const uint64_t pol = l2_evict_first_policy();
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n4;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float* src = ws + i * 4;
    float4 acc = ld_evict_first_v4(src, pol);
    int k = 1;
    for (; k + 4 <= splits; k += 4) {
      float4 v[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) v[u] = ld_evict_first_v4(src + (k + u) * slice, pol);
#pragma unroll
      for (int u = 0; u < 4; ++u) add4(acc, v[u]);
    }
    for (; k < splits; ++k) add4(acc, ld_evict_first_v4(src + k * slice, pol));
    acc = make_float4(__fmul_rn(alpha, acc.x), __fmul_rn(alpha, acc.y), __fmul_rn(alpha, acc.z), __fmul_rn(alpha, acc.w));
    float4* o = reinterpret_cast<float4*>(dst) + i;
    if (accumulate) {
      float4 d = *o;
      add4(d, acc);
      acc = d;
    }
    *o = acc;
  }
  if (blockIdx.x == 0) {                // scalar tail
    for (long long i = n4 * 4 + threadIdx.x; i < n; i += blockDim.x) {
      float acc = ws[i];
      for (int k = 1; k < splits; ++k) acc = __fadd_rn(acc, ws[i + k * slice]);
      acc = __fmul_rn(alpha, acc);
      dst[i] = accumulate ? __fadd_rn(dst[i], acc) : acc;
    }
  }
}

void splitk_reduce(const float* ws, long long ws_elems, float* dst, long long n, long long slice, int splits,
                   float alpha, bool accumulate, cudaStream_t s) {
  if (n <= 0 || splits < 1 || slice < n || slice % 4 != 0)
    throw std::runtime_error("[b200] splitk_reduce: needs n > 0, splits >= 1 and a slice stride >= n in whole float4s");
  if (!ws || !dst || (reinterpret_cast<uintptr_t>(ws) & 15) || (reinterpret_cast<uintptr_t>(dst) & 15))
    throw std::runtime_error("[b200] splitk_reduce: the workspace and the destination must be 16-byte aligned");
  if (ws_elems < (splits - 1) * slice + n)
    throw std::runtime_error("[b200] splitk_reduce: the workspace holds " + std::to_string(ws_elems) + " floats, " +
                             std::to_string(splits) + " slices need " + std::to_string((splits - 1) * slice + n));
  splitk_reduce_kernel<<<min(ceil_div_ll(n / 4 + 1, 256), sm_count() * 8), 256, 0, s>>>(ws, dst, n, slice, splits, alpha,
                                                                                      accumulate ? 1 : 0);
  count_launch();
  check_last("splitk_reduce");
}
void bias_grad_ld(const bf16* dz, float* db, long long rows, int C, int ld, float scale,
                  cudaStream_t s) {
  bias_grad_small_kernel<<<(C + 127) / 128, 128, 0, s>>>(dz, db, rows, C, ld, scale);
  count_launch();
  check_last("bias_grad_ld");
}

// ------------------------------------------------------------------------------ FC epilogues
// y = dropout(relu(acc + bias)); written as bf16 (ld = ldy) and/or fp32; acc optionally cleared so
// the split-K red.add GEMM of the next step starts from zero.
__global__ void fc_bias_act_kernel(float* __restrict__ acc, const float* __restrict__ bias,
                                   bf16* __restrict__ y, float* __restrict__ y_f32, int B, int N,
                                   int ldy, int relu, float drop_p, unsigned long long seed,
                                   unsigned long long offset, int clear) {
  const long long total = static_cast<long long>(B) * N;
  const long long quads = (total + 3) / 4;
  const float keep_scale = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  for (long long q = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; q < quads;
       q += static_cast<long long>(gridDim.x) * blockDim.x) {
    uint4 rnd = make_uint4(0, 0, 0, 0);
    if (drop_p > 0.f)
      rnd = philox4x32_10(make_uint2(static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32)),
                          make_uint4(static_cast<uint32_t>(q), static_cast<uint32_t>(q >> 32),
                                     static_cast<uint32_t>(offset), static_cast<uint32_t>(offset >> 32)));
    const uint32_t rr[4] = {rnd.x, rnd.y, rnd.z, rnd.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const long long i = q * 4 + j;
      if (i >= total) break;
      const int b = static_cast<int>(i / N), n = static_cast<int>(i % N);
      float v = acc[i] + (bias ? bias[n] : 0.f);
      if (clear) acc[i] = 0.f;
      if (relu) v = fmaxf(v, 0.f);
      if (drop_p > 0.f) {
        const float u = (rr[j] >> 8) * (1.0f / 16777216.0f);
        v = u < drop_p ? 0.f : v * keep_scale;
      }
      if (y) y[static_cast<long long>(b) * ldy + n] = __float2bfloat16(v);
      if (y_f32) y_f32[i] = v;
    }
  }
}

void fc_bias_act(float* acc, const float* bias, bf16* y, float* y_f32, int B, int N, bool relu,
                 float drop_p, unsigned long long seed, unsigned long long offset, bool clear,
                 cudaStream_t s) {
  const long long quads = (static_cast<long long>(B) * N + 3) / 4;
  fc_bias_act_kernel<<<min(ceil_div_ll(quads, 256), sm_count() * 8), 256, 0, s>>>(
      acc, bias, y, y_f32, B, N, N, relu ? 1 : 0, drop_p, seed, offset, clear ? 1 : 0);
  count_launch();
  check_last("fc_bias_act");
}

// dz = acc * [act > 0] / (1 - p).  `act` is the layer's *post-dropout* output, so act > 0 encodes
// both the ReLU mask and the dropout keep-mask.
__global__ void fc_grad_act_kernel(float* __restrict__ acc, const bf16* __restrict__ act,
                                   bf16* __restrict__ dz, long long total, int relu, float scale,
                                   int clear) {
  const long long n4 = total / 4;       // 16-byte fp32 / 8-byte bf16 vectors
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n4;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float4 v = reinterpret_cast<float4*>(acc)[i];
    if (clear) reinterpret_cast<float4*>(acc)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (relu) {
      const uint2 a = *reinterpret_cast<const uint2*>(act + i * 4);
      const float2 a0 = unpack_bf16x2(a.x), a1 = unpack_bf16x2(a.y);
      v.x = a0.x > 0.f ? v.x * scale : 0.f;
      v.y = a0.y > 0.f ? v.y * scale : 0.f;
      v.z = a1.x > 0.f ? v.z * scale : 0.f;
      v.w = a1.y > 0.f ? v.w * scale : 0.f;
    }
    *reinterpret_cast<uint2*>(dz + i * 4) = make_uint2(pack_bf16x2(v.x, v.y), pack_bf16x2(v.z, v.w));
  }
  if (blockIdx.x == 0) {                // scalar tail
    for (long long i = n4 * 4 + threadIdx.x; i < total; i += blockDim.x) {
      float v = acc[i];
      if (clear) acc[i] = 0.f;
      if (relu) v = __bfloat162float(act[i]) > 0.f ? v * scale : 0.f;
      dz[i] = __float2bfloat16(v);
    }
  }
}

void fc_grad_act(float* acc, const bf16* act, bf16* dz, int B, int N, bool relu, float drop_p,
                 unsigned long long, unsigned long long, bool clear, cudaStream_t s) {
  const long long total = static_cast<long long>(B) * N;
  const float scale = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  if ((reinterpret_cast<uintptr_t>(acc) & 15) || (reinterpret_cast<uintptr_t>(dz) & 7) ||
      (act && (reinterpret_cast<uintptr_t>(act) & 7)))
    throw std::runtime_error("[b200] fc_grad_act: buffers must be 16-byte (fp32) / 8-byte (bf16) aligned");
  fc_grad_act_kernel<<<min(ceil_div_ll(total / 4 + 1, 256), sm_count() * 8), 256, 0, s>>>(acc, act, dz, total,
                                                                                   relu ? 1 : 0, scale, clear ? 1 : 0);
  count_launch();
  check_last("fc_grad_act");
}

// -------------------------------------------------------------------------------------- casts
__global__ void cast_f32_to_bf16_kernel(const float* __restrict__ x, bf16* __restrict__ y, long long n) {
  const long long n4 = n / 4;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n4;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float4 v = *reinterpret_cast<const float4*>(x + i * 4);
    *reinterpret_cast<uint2*>(y + i * 4) = make_uint2(pack_bf16x2(v.x, v.y), pack_bf16x2(v.z, v.w));
  }
  if (blockIdx.x == 0 && threadIdx.x < n % 4) y[n4 * 4 + threadIdx.x] = __float2bfloat16(x[n4 * 4 + threadIdx.x]);
}
__global__ void cast_bf16_to_f32_kernel(const bf16* __restrict__ x, float* __restrict__ y, long long n) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    y[i] = __bfloat162float(x[i]);
}
void cast_f32_to_bf16(const float* x, bf16* y, long long n, cudaStream_t s) {
  cast_f32_to_bf16_kernel<<<min(ceil_div_ll(n / 4 + 1, 256), sm_count() * 8), 256, 0, s>>>(x, y, n);
  count_launch();
  check_last("cast_f32_to_bf16");
}
void cast_bf16_to_f32(const bf16* x, float* y, long long n, cudaStream_t s) {
  cast_bf16_to_f32_kernel<<<min(ceil_div_ll(n, 256), sm_count() * 8), 256, 0, s>>>(x, y, n);
  count_launch();
  check_last("cast_bf16_to_f32");
}

// ------------------------------------------------------------------------ co-residency probe
// bench/interference.py: a thin (256 threads, <= 40 registers, no shared memory) background kernel that
// exercises ONE resource, to find out what a comm-stream CTA sharing an SM with a persistent wgmma
// conv CTA takes away from it.  mode 0: dependent FMA chain (issue slots only), 1: streaming 16-byte
// loads, 2: streaming 16-byte stores, 3: load + store, 4: sqrt / divide chain (MUFU),
// 5: sleep (resident warps that issue almost nothing).
__global__ void __launch_bounds__(256, 6)
probe_background_kernel(float4* __restrict__ buf, long long n4, int mode, int reps, float* __restrict__ sink) {
  float acc = threadIdx.x * 1e-6f;
  for (int r = 0; r < reps; ++r) {
    if (mode == 0) {
      for (int k = 0; k < 4096; ++k) acc = fmaf(acc, 1.000001f, 1e-7f);
    } else if (mode == 4) {
      for (int k = 0; k < 1024; ++k) acc = sqrtf(acc + 1.5f) / (acc + 2.5f);
    } else if (mode == 5) {
      for (int k = 0; k < 64; ++k) __nanosleep(1000);
    } else {
      for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n4;
           i += static_cast<long long>(gridDim.x) * blockDim.x) {
        if (mode == 1) {
          const float4 v = __ldcs(buf + i);
          acc += v.x + v.w;
        } else if (mode == 2) {
          __stcs(buf + i, make_float4(acc, 0.f, 0.f, 0.f));
        } else {
          float4 v = __ldcs(buf + i);
          v.x += 1.f;
          __stcs(buf + i, v);
        }
      }
    }
  }
  if (acc == 12345.678f) *sink = acc;
}
void probe_background(float* buf, long long n, int mode, int ctas, int reps, float* sink, cudaStream_t s) {
  static const bool carve = [] {
    const char* e = getenv("B200_PROBE_CARVEOUT");
    if (e && e[0] == '1') prefer_max_shared_carveout(reinterpret_cast<const void*>(probe_background_kernel));
    return true;
  }();
  (void)carve;
  probe_background_kernel<<<ctas, 256, 0, s>>>(reinterpret_cast<float4*>(buf), n / 4, mode, reps, sink);
  count_launch();
  check_last("probe_background");
}

}  // namespace b200
