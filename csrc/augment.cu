// Fused input transform (K-AUG): the reference's six PIL/torchvision stages
// (distributedVggf.py:88-95 / :103-108) evaluated as one coordinate chain per output pixel, reading
// the decoded uint8 HWC source and writing normalised bf16 either as NHWC (C padded) or directly
// as the layer-0 im2col matrix [N*OH*OW][kpad] (k = (kh*3+kw)*3 + c) that feeds the wgmma GEMM
// -- the 3-channel tensor never exists in HBM in that mode.
// The arithmetic mirrors data/transforms.py::augment_reference (the oracle in the tests).
#include <stdexcept>

#include "api.h"
#include "ptx.cuh"

namespace b200 {

struct AugGeom {
  int N, SH, SW, RH, RW, OH, OW;
  float mean[3], inv_std[3];
};

// Test-time augmentation views (TtaView in api.h): the origin (y0, x0) of an OH x OW crop of the RH x RW
// resized image, and whether the crop is taken from its horizontal mirror (the chain's flip, applied after
// the crop offset, is exactly that).  Centre origins round half to even, as torchvision's center_crop.
__device__ __forceinline__ void view_origin(int view, int RH, int RW, int OH, int OW, int& y0, int& x0, bool& flip) {
  const int pos = view & 7;
  const int cy = __float2int_rn((RH - OH) * 0.5f), cx = __float2int_rn((RW - OW) * 0.5f);
  y0 = pos == TtaTopLeft || pos == TtaTopRight ? 0 : (pos == TtaBottomLeft || pos == TtaBottomRight ? RH - OH : cy);
  x0 = pos == TtaTopLeft || pos == TtaBottomLeft ? 0
       : (pos == TtaTopRight || pos == TtaBottomRight ? RW - OW : (pos == TtaCentreMirror ? RW - OW - cx : cx));
  flip = (view & TtaFlip) != 0;
}

// Normalised value of output pixel (oy, ox) of sample n, all 3 channels.
__device__ __forceinline__ void aug_sample(const uint8_t* __restrict__ src, const float* __restrict__ prm,
                                           const AugGeom& g, int oy, int ox, float (&out)[3]) {
  const float top = prm[0], left = prm[1], ch = prm[2], cw = prm[3], cs = prm[4], sn = prm[5];
  const bool flip = prm[6] > 0.5f;
  const int off_y = __float2int_rn((g.RH - g.OH) * 0.5f);
  const int off_x = __float2int_rn((g.RW - g.OW) * 0.5f);
  const float ay = static_cast<float>(oy + off_y);
  float ax = static_cast<float>(ox + off_x);
  if (flip) ax = static_cast<float>(g.RW - 1) - ax;
  const float cx = g.RW * 0.5f, cy = g.RH * 0.5f;
  const float dx = ax + 0.5f - cx, dy = ay + 0.5f - cy;
  const float rx = floorf(cs * dx - sn * dy + cx);
  const float ry = floorf(sn * dx + cs * dy + cy);
  if (rx < 0.f || rx >= g.RW || ry < 0.f || ry >= g.RH) {   // rotation fill = 0 (pre-normalise)
#pragma unroll
    for (int c = 0; c < 3; ++c) out[c] = (0.f - g.mean[c]) * g.inv_std[c];
    return;
  }
  float sy = (ry + 0.5f) * (ch / g.RH) - 0.5f;
  float sx = (rx + 0.5f) * (cw / g.RW) - 0.5f;
  sy = fminf(fmaxf(sy, 0.f), ch - 1.f);
  sx = fminf(fmaxf(sx, 0.f), cw - 1.f);
  const float y0 = floorf(sy), x0 = floorf(sx);
  const float wy = sy - y0, wx = sx - x0;
  const float y1 = fminf(y0 + 1.f, ch - 1.f), x1 = fminf(x0 + 1.f, cw - 1.f);
  const int iy0 = min(max(static_cast<int>(y0 + top), 0), g.SH - 1);
  const int iy1 = min(max(static_cast<int>(y1 + top), 0), g.SH - 1);
  const int ix0 = min(max(static_cast<int>(x0 + left), 0), g.SW - 1);
  const int ix1 = min(max(static_cast<int>(x1 + left), 0), g.SW - 1);
  const uint8_t* p00 = src + (static_cast<long long>(iy0) * g.SW + ix0) * 3;
  const uint8_t* p01 = src + (static_cast<long long>(iy0) * g.SW + ix1) * 3;
  const uint8_t* p10 = src + (static_cast<long long>(iy1) * g.SW + ix0) * 3;
  const uint8_t* p11 = src + (static_cast<long long>(iy1) * g.SW + ix1) * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float v = p00[c] * (1.f - wy) * (1.f - wx) + p01[c] * (1.f - wy) * wx +
                    p10[c] * wy * (1.f - wx) + p11[c] * wy * wx;
    out[c] = (v * (1.f / 255.f) - g.mean[c]) * g.inv_std[c];
  }
}

// aug_sample for the crop at (off_y, off_x) of the resized image (of its mirror with `flip`).  A copy rather than
// the body of aug_sample: sharing it moves registers in the kernels that call aug_sample.
__device__ __forceinline__ void aug_sample_at(const uint8_t* __restrict__ src, const float* __restrict__ prm,
                                              const AugGeom& g, int oy, int ox, int off_y, int off_x, bool flip,
                                              float (&out)[3]) {
  const float top = prm[0], left = prm[1], ch = prm[2], cw = prm[3], cs = prm[4], sn = prm[5];
  const float ay = static_cast<float>(oy + off_y);
  float ax = static_cast<float>(ox + off_x);
  if (flip) ax = static_cast<float>(g.RW - 1) - ax;
  const float cx = g.RW * 0.5f, cy = g.RH * 0.5f;
  const float dx = ax + 0.5f - cx, dy = ay + 0.5f - cy;
  const float rx = floorf(cs * dx - sn * dy + cx);
  const float ry = floorf(sn * dx + cs * dy + cy);
  if (rx < 0.f || rx >= g.RW || ry < 0.f || ry >= g.RH) {   // rotation fill = 0 (pre-normalise)
#pragma unroll
    for (int c = 0; c < 3; ++c) out[c] = (0.f - g.mean[c]) * g.inv_std[c];
    return;
  }
  float sy = (ry + 0.5f) * (ch / g.RH) - 0.5f;
  float sx = (rx + 0.5f) * (cw / g.RW) - 0.5f;
  sy = fminf(fmaxf(sy, 0.f), ch - 1.f);
  sx = fminf(fmaxf(sx, 0.f), cw - 1.f);
  const float y0 = floorf(sy), x0 = floorf(sx);
  const float wy = sy - y0, wx = sx - x0;
  const float y1 = fminf(y0 + 1.f, ch - 1.f), x1 = fminf(x0 + 1.f, cw - 1.f);
  const int iy0 = min(max(static_cast<int>(y0 + top), 0), g.SH - 1);
  const int iy1 = min(max(static_cast<int>(y1 + top), 0), g.SH - 1);
  const int ix0 = min(max(static_cast<int>(x0 + left), 0), g.SW - 1);
  const int ix1 = min(max(static_cast<int>(x1 + left), 0), g.SW - 1);
  const uint8_t* p00 = src + (static_cast<long long>(iy0) * g.SW + ix0) * 3;
  const uint8_t* p01 = src + (static_cast<long long>(iy0) * g.SW + ix1) * 3;
  const uint8_t* p10 = src + (static_cast<long long>(iy1) * g.SW + ix0) * 3;
  const uint8_t* p11 = src + (static_cast<long long>(iy1) * g.SW + ix1) * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float v = p00[c] * (1.f - wy) * (1.f - wx) + p01[c] * (1.f - wy) * wx +
                    p10[c] * wy * (1.f - wx) + p11[c] * wy * wx;
    out[c] = (v * (1.f / 255.f) - g.mean[c]) * g.inv_std[c];
  }
}

// mode 0: NHWC bf16, C padded to `pad` (pad in {4, 8}); one thread per output pixel.
// MIX (augment_mixed): MixNone is the plain transform.  The partner of sample n is n-1 mod N.
//   MixCutMix: a pixel inside the box evaluates the partner's chain (its source and params), one
//              evaluation per pixel either way.
//   MixMixUp:  both chains, blended in fp32 as lam * x_n + (1 - lam) * x_partner, rounded to bf16 once.
template <int MIX>
__global__ void augment_nhwc_kernel(const uint8_t* __restrict__ src, const float* __restrict__ params,
                                    bf16* __restrict__ out, AugGeom g, int pad, MixParams mix) {
  const long long total = static_cast<long long>(g.N) * g.OH * g.OW;
  const long long img = static_cast<long long>(g.SH) * g.SW * 3;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int ox = i % g.OW;
    const int oy = (i / g.OW) % g.OH;
    int n = static_cast<int>(i / (static_cast<long long>(g.OW) * g.OH));
    float v[3];
    if constexpr (MIX == MixCutMix) {
      if (ox >= mix.x1 && ox < mix.x2 && oy >= mix.y1 && oy < mix.y2) n = n == 0 ? g.N - 1 : n - 1;
    }
    aug_sample(src + n * img, params + n * 8, g, oy, ox, v);
    if constexpr (MIX == MixMixUp) {
      const int p = n == 0 ? g.N - 1 : n - 1;
      float w[3];
      aug_sample(src + p * img, params + p * 8, g, oy, ox, w);
#pragma unroll
      for (int c = 0; c < 3; ++c) v[c] = __fadd_rn(__fmul_rn(mix.lam, v[c]), __fmul_rn(mix.lam_b, w[c]));
    }
    bf16* o = out + i * pad;
    if (pad == 4) {          // one 8-byte store per pixel
      *reinterpret_cast<uint2*>(o) = make_uint2(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], 0.f));
    } else {
      o[0] = __float2bfloat16(v[0]);
      o[1] = __float2bfloat16(v[1]);
      o[2] = __float2bfloat16(v[2]);
      for (int c = 3; c < pad; ++c) o[c] = __float2bfloat16(0.f);
    }
  }
}

// mode 1: im2col rows for the 3x3/pad-1 first convolution.  One thread per (pixel, 8-element
// chunk of the row): it evaluates the transform at the (up to 4) taps its chunk covers (0 outside
// the image: conv zero padding acts on the *normalised* tensor) and issues ONE 16-byte store, so a
// warp writes 512 contiguous bytes.  Chunks beyond k = 27 are the zero tail.
__global__ void augment_im2col_kernel(const uint8_t* __restrict__ src, const float* __restrict__ params,
                                      bf16* __restrict__ out, AugGeom g, int kpad) {
  const int chunks = kpad / 8;
  const long long total = static_cast<long long>(g.N) * g.OH * g.OW * chunks;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int chunk = static_cast<int>(i % chunks);
    const long long pix = i / chunks;
    float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    const int k0 = chunk * 8;
    if (k0 < 27) {
      const int ox = pix % g.OW;
      const int oy = (pix / g.OW) % g.OH;
      const int n = static_cast<int>(pix / (static_cast<long long>(g.OW) * g.OH));
      const uint8_t* img = src + static_cast<long long>(n) * g.SH * g.SW * 3;
      const float* prm = params + n * 8;
      const int tap_lo = k0 / 3;
      const int tap_hi = min((k0 + 7) / 3, 8);
      for (int tap = tap_lo; tap <= tap_hi; ++tap) {
        const int yy = oy + tap / 3 - 1, xx = ox + tap % 3 - 1;
        float s3[3] = {0.f, 0.f, 0.f};
        if (yy >= 0 && yy < g.OH && xx >= 0 && xx < g.OW) aug_sample(img, prm, g, yy, xx, s3);
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const int k = tap * 3 + c - k0;
          if (k >= 0 && k < 8) v[k] = s3[c];
        }
      }
    }
    const uint4 pk = make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]),
                                pack_bf16x2(v[4], v[5]), pack_bf16x2(v[6], v[7]));
    *reinterpret_cast<uint4*>(out + pix * kpad + k0) = pk;
  }
}

void augment_fused(const uint8_t* src, const float* params, bf16* out, int N, int SH, int SW, int RH,
                   int RW, int OH, int OW, int mode, int pad, const float* mean, const float* stdv,
                   cudaStream_t s) {
  AugGeom g;
  g.N = N; g.SH = SH; g.SW = SW; g.RH = RH; g.RW = RW; g.OH = OH; g.OW = OW;
  for (int c = 0; c < 3; ++c) { g.mean[c] = mean[c]; g.inv_std[c] = 1.f / stdv[c]; }
  const long long pixels = static_cast<long long>(N) * OH * OW;
  if (mode == 0) {
    const int blocks = static_cast<int>((pixels + 255) / 256 < sm_count() * 16 ? (pixels + 255) / 256 : sm_count() * 16);
    augment_nhwc_kernel<MixNone><<<blocks, 256, 0, s>>>(src, params, out, g, pad, MixParams{});
  } else {
    if (pad < 32 || pad % 8) throw std::runtime_error("[b200] augment_fused: kpad must be a multiple of 8, >= 32");
    const long long total = pixels * (pad / 8);
    const int blocks = static_cast<int>((total + 255) / 256 < sm_count() * 32 ? (total + 255) / 256 : sm_count() * 32);
    augment_im2col_kernel<<<blocks, 256, 0, s>>>(src, params, out, g, pad);
  }
  count_launch();
  check_last("augment_fused");
}

void augment_mixed(const uint8_t* src, const float* params, bf16* out, int N, int SH, int SW, int RH, int RW,
                   int OH, int OW, int pad, const float* mean, const float* stdv, const MixParams& mix,
                   cudaStream_t s) {
  if (mix.kind != MixMixUp && mix.kind != MixCutMix) throw std::runtime_error("[b200] augment_mixed: kind is MixUp or CutMix");
  AugGeom g;
  g.N = N; g.SH = SH; g.SW = SW; g.RH = RH; g.RW = RW; g.OH = OH; g.OW = OW;
  for (int c = 0; c < 3; ++c) { g.mean[c] = mean[c]; g.inv_std[c] = 1.f / stdv[c]; }
  const long long pixels = static_cast<long long>(N) * OH * OW;
  const int blocks = static_cast<int>((pixels + 255) / 256 < sm_count() * 16 ? (pixels + 255) / 256 : sm_count() * 16);
  if (mix.kind == MixMixUp)
    augment_nhwc_kernel<MixMixUp><<<blocks, 256, 0, s>>>(src, params, out, g, pad, mix);
  else
    augment_nhwc_kernel<MixCutMix><<<blocks, 256, 0, s>>>(src, params, out, g, pad, mix);
  count_launch();
  check_last("augment_mixed");
}

// One test-time augmentation view into NHWC4: aug_sample_at at the view's origin, the view's flip combined with
// the sample's own.  A kernel of its own, so that augment_nhwc_kernel's instantiations keep their code.
__global__ void augment_view_nhwc_kernel(const uint8_t* __restrict__ src, const float* __restrict__ params,
                                         bf16* __restrict__ out, AugGeom g, int view) {
  int y0, x0;
  bool vflip;
  view_origin(view, g.RH, g.RW, g.OH, g.OW, y0, x0, vflip);
  const long long total = static_cast<long long>(g.N) * g.OH * g.OW;
  const long long img = static_cast<long long>(g.SH) * g.SW * 3;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int ox = i % g.OW;
    const int oy = (i / g.OW) % g.OH;
    const int n = static_cast<int>(i / (static_cast<long long>(g.OW) * g.OH));
    const float* prm = params + n * 8;
    float v[3];
    aug_sample_at(src + n * img, prm, g, oy, ox, y0, x0, (prm[6] > 0.5f) != vflip, v);
    *reinterpret_cast<uint2*>(out + i * 4) = make_uint2(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], 0.f));
  }
}

void augment_view(const uint8_t* src, const float* params, bf16* out, int N, int SH, int SW, int RH, int RW, int OH,
                  int OW, int view, const float* mean, const float* stdv, cudaStream_t s) {
  AugGeom g;
  g.N = N; g.SH = SH; g.SW = SW; g.RH = RH; g.RW = RW; g.OH = OH; g.OW = OW;
  for (int c = 0; c < 3; ++c) { g.mean[c] = mean[c]; g.inv_std[c] = 1.f / stdv[c]; }
  const long long pixels = static_cast<long long>(N) * OH * OW;
  const int blocks = static_cast<int>((pixels + 255) / 256 < sm_count() * 16 ? (pixels + 255) / 256 : sm_count() * 16);
  augment_view_nhwc_kernel<<<blocks, 256, 0, s>>>(src, params, out, g, view);
  count_launch();
  check_last("augment_view");
}

// ------------------------------------------------------------------ ragged batches, Pillow resampling
// Images of any size.  The crop box is resized with Pillow's BILINEAR filter (libImaging/Resample.c),
// which widens to the whole footprint when it shrinks: per axis scale = in/out, support = max(scale, 1),
// fp64 triangle weights normalised by their sum, then 22-bit fixed point.  Like Pillow, the horizontal
// pass rounds to uint8 before the vertical pass, so both passes are exact integer arithmetic and the
// fp64 operations below are spelled with _rn intrinsics so that nvcc contracts none of them.
// data/transforms.py::ragged_reference is the oracle.
struct RaggedGeom {
  int N, OH, OW;
  float mean[3], stdv[3];
};

constexpr int kPilBits = 22;

struct PilAxis {
  double scale, support, ss;
  int in;
};

__device__ __forceinline__ PilAxis pil_axis(int in, int out) {
  PilAxis a;
  a.scale = __ddiv_rn(static_cast<double>(in), static_cast<double>(out));
  a.support = a.scale < 1.0 ? 1.0 : a.scale;
  a.ss = __ddiv_rn(1.0, a.support);
  a.in = in;
  return a;
}

// Input window [lo, lo + n) of output index i, and the sum of its unnormalised weights.
struct PilWindow {
  double center, ww;
  int lo, n;
};

__device__ __forceinline__ double pil_weight(const PilAxis& a, const PilWindow& w, int x) {
  const double t = fabs(__dmul_rn(__dadd_rn(__dsub_rn(static_cast<double>(x + w.lo), w.center), 0.5), a.ss));
  return t < 1.0 ? __dsub_rn(1.0, t) : 0.0;
}

__device__ __forceinline__ PilWindow pil_window(const PilAxis& a, int i) {
  PilWindow w;
  w.center = __dmul_rn(static_cast<double>(i) + 0.5, a.scale);
  w.lo = max(static_cast<int>(__dadd_rn(__dsub_rn(w.center, a.support), 0.5)), 0);
  w.n = min(static_cast<int>(__dadd_rn(__dadd_rn(w.center, a.support), 0.5)), a.in) - w.lo;
  w.ww = 0.0;
  for (int x = 0; x < w.n; ++x) w.ww = __dadd_rn(w.ww, pil_weight(a, w, x));
  return w;
}

__device__ __forceinline__ int pil_fixed(const PilAxis& a, const PilWindow& w, int x) {
  double k = pil_weight(a, w, x);
  if (w.ww != 0.0) k = __ddiv_rn(k, w.ww);
  return static_cast<int>(__dadd_rn(0.5, __dmul_rn(k, static_cast<double>(1 << kPilBits))));
}

__device__ __forceinline__ uint8_t pil_clip8(int acc) { return static_cast<uint8_t>(min(max(acc >> kPilBits, 0), 255)); }

// (rx, ry) in the RH x RW resized image of output pixel (oy, ox): centre crop, flip, nearest rotation,
// each float operation rounded on its own, as augment_reference evaluates it with torch ops.
__device__ __forceinline__ void ragged_chain(const float* prm, int RH, int RW, int OH, int OW, int oy, int ox,
                                             float& rx, float& ry) {
  const float cs = prm[4], sn = prm[5];
  const float ay = static_cast<float>(oy + __float2int_rn((RH - OH) * 0.5f));
  float ax = static_cast<float>(ox + __float2int_rn((RW - OW) * 0.5f));
  if (prm[6] > 0.5f) ax = static_cast<float>(RW - 1) - ax;
  const float cx = RW * 0.5f, cy = RH * 0.5f;
  const float dx = __fsub_rn(__fadd_rn(ax, 0.5f), cx), dy = __fsub_rn(__fadd_rn(ay, 0.5f), cy);
  rx = floorf(__fadd_rn(__fsub_rn(__fmul_rn(cs, dx), __fmul_rn(sn, dy)), cx));
  ry = floorf(__fadd_rn(__fadd_rn(__fmul_rn(sn, dx), __fmul_rn(cs, dy)), cy));
}


// ragged_chain for the crop at (y0, x0), of the mirror with `flip` (a copy, for the reason given at aug_sample_at).
__device__ __forceinline__ void ragged_chain_at(const float* prm, int RH, int RW, int y0, int x0, bool flip, int oy,
                                                int ox, float& rx, float& ry) {
  const float cs = prm[4], sn = prm[5];
  const float ay = static_cast<float>(oy + y0);
  float ax = static_cast<float>(ox + x0);
  if (flip) ax = static_cast<float>(RW - 1) - ax;
  const float cx = RW * 0.5f, cy = RH * 0.5f;
  const float dx = __fsub_rn(__fadd_rn(ax, 0.5f), cx), dy = __fsub_rn(__fadd_rn(ay, 0.5f), cy);
  rx = floorf(__fadd_rn(__fsub_rn(__fmul_rn(cs, dx), __fmul_rn(sn, dy)), cx));
  ry = floorf(__fadd_rn(__fadd_rn(__fmul_rn(sn, dx), __fmul_rn(cs, dy)), cy));
}

// Per-image state shared by a block: every block of both passes works on one image (blockIdx.y).
struct RaggedImage {
  long long off, inter;       // byte offsets of the source and of its intermediate
  int H, W, RH, RW, top, left, ch, cw;
  int rx0, rx1, ry0, ry1;     // resized pixels the output reads (rx0 > rx1: none)
};

__device__ void load_ragged_image(const long long* __restrict__ geom, const float* __restrict__ params, int n,
                                  int OH, int OW, RaggedImage& im) {
  const long long* g = geom + n * 5;
  im.off = g[0];
  im.H = static_cast<int>(g[1]); im.W = static_cast<int>(g[2]);
  im.RH = static_cast<int>(g[3]); im.RW = static_cast<int>(g[4]);
  long long inter = 0;       // the intermediates of the batch's images lie back to back, H x RW x 3 each
  for (int i = 0; i < n; ++i) inter += geom[i * 5 + 1] * geom[i * 5 + 4] * 3;
  im.inter = inter;
  const float* p = params + n * 8;
  im.top = static_cast<int>(p[0]); im.left = static_cast<int>(p[1]);
  im.ch = static_cast<int>(p[2]); im.cw = static_cast<int>(p[3]);
  // the chain is monotone in ox and in oy (each rounded operation is), so the corners bound it
  float x0 = 3.4e38f, x1 = -3.4e38f, y0 = 3.4e38f, y1 = -3.4e38f;
  for (int c = 0; c < 4; ++c) {
    float rx, ry;
    ragged_chain(p, im.RH, im.RW, OH, OW, (c >> 1) * (OH - 1), (c & 1) * (OW - 1), rx, ry);
    x0 = fminf(x0, rx); x1 = fmaxf(x1, rx); y0 = fminf(y0, ry); y1 = fmaxf(y1, ry);
  }
  im.rx0 = static_cast<int>(fmaxf(x0, 0.f)); im.rx1 = static_cast<int>(fminf(x1, im.RW - 1.f));
  im.ry0 = static_cast<int>(fmaxf(y0, 0.f)); im.ry1 = static_cast<int>(fminf(y1, im.RH - 1.f));
  if (im.ry0 > im.ry1) im.rx1 = im.rx0 - 1;
}

// Pass 1: rows of the crop box that the vertical filter reads x the resized columns the output reads,
// filtered horizontally into inter[crop row][RW][3] (uint8).
__global__ void augment_ragged_h_kernel(const uint8_t* __restrict__ src, const long long* __restrict__ geom,
                                        const float* __restrict__ params, uint8_t* __restrict__ inter, RaggedGeom g) {
  __shared__ RaggedImage im;
  if (threadIdx.x == 0) load_ragged_image(geom, params, blockIdx.y, g.OH, g.OW, im);
  __syncthreads();
  if (im.rx0 > im.rx1) return;
  const PilAxis va = pil_axis(im.ch, im.RH), ha = pil_axis(im.cw, im.RW);
  const PilWindow first = pil_window(va, im.ry0), last = pil_window(va, im.ry1);
  const int r0 = first.lo, rows = last.lo + last.n - first.lo, cols = im.rx1 - im.rx0 + 1;
  const long long total = static_cast<long long>(rows) * cols;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int r = r0 + static_cast<int>(i / cols), x = im.rx0 + static_cast<int>(i % cols);
    const PilWindow w = pil_window(ha, x);
    const uint8_t* s = src + im.off + (static_cast<long long>(im.top + r) * im.W + im.left + w.lo) * 3;
    int a0 = 1 << (kPilBits - 1), a1 = a0, a2 = a0;
    for (int t = 0; t < w.n; ++t) {
      const int k = pil_fixed(ha, w, t);
      a0 += s[t * 3] * k; a1 += s[t * 3 + 1] * k; a2 += s[t * 3 + 2] * k;
    }
    uint8_t* o = inter + im.inter + (static_cast<long long>(r) * im.RW + x) * 3;
    o[0] = pil_clip8(a0); o[1] = pil_clip8(a1); o[2] = pil_clip8(a2);
  }
}

// Normalised value of output pixel (oy, ox) of a ragged image: chain -> (rx, ry), vertical filter down
// column rx of the intermediate -> uint8 -> normalise.
__device__ __forceinline__ void ragged_pixel(const RaggedImage& im, const PilAxis& va, const float* prm,
                                             const uint8_t* __restrict__ inter, const RaggedGeom& g, int oy, int ox,
                                             float (&o)[3]) {
  float rx, ry;
  ragged_chain(prm, im.RH, im.RW, g.OH, g.OW, oy, ox, rx, ry);
  float v[3] = {0.f, 0.f, 0.f};
  if (rx >= 0.f && rx < im.RW && ry >= 0.f && ry < im.RH) {     // rotation fill = 0 (pre-normalise)
    const PilWindow w = pil_window(va, static_cast<int>(ry));
    const long long stride = static_cast<long long>(im.RW) * 3;
    const uint8_t* s = inter + im.inter + w.lo * stride + static_cast<int>(rx) * 3;
    int a0 = 1 << (kPilBits - 1), a1 = a0, a2 = a0;
    for (int t = 0; t < w.n; ++t) {
      const int k = pil_fixed(va, w, t);
      a0 += s[t * stride] * k; a1 += s[t * stride + 1] * k; a2 += s[t * stride + 2] * k;
    }
    v[0] = pil_clip8(a0); v[1] = pil_clip8(a1); v[2] = pil_clip8(a2);
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) o[c] = __fdiv_rn(__fsub_rn(__fdiv_rn(v[c], 255.f), g.mean[c]), g.stdv[c]);
}

// ragged_pixel after the chain: the vertical filter at (rx, ry) (a copy, as ragged_chain_at).
__device__ __forceinline__ void ragged_sample(const RaggedImage& im, const PilAxis& va, const uint8_t* __restrict__ inter,
                                              const RaggedGeom& g, float rx, float ry, float (&o)[3]) {
  float v[3] = {0.f, 0.f, 0.f};
  if (rx >= 0.f && rx < im.RW && ry >= 0.f && ry < im.RH) {     // rotation fill = 0 (pre-normalise)
    const PilWindow w = pil_window(va, static_cast<int>(ry));
    const long long stride = static_cast<long long>(im.RW) * 3;
    const uint8_t* s = inter + im.inter + w.lo * stride + static_cast<int>(rx) * 3;
    int a0 = 1 << (kPilBits - 1), a1 = a0, a2 = a0;
    for (int t = 0; t < w.n; ++t) {
      const int k = pil_fixed(va, w, t);
      a0 += s[t * stride] * k; a1 += s[t * stride + 1] * k; a2 += s[t * stride + 2] * k;
    }
    v[0] = pil_clip8(a0); v[1] = pil_clip8(a1); v[2] = pil_clip8(a2);
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) o[c] = __fdiv_rn(__fsub_rn(__fdiv_rn(v[c], 255.f), g.mean[c]), g.stdv[c]);
}

// Pass 2: one thread per output pixel: ragged_pixel, one 8-byte NHWC4 store.  MIX as for
// augment_nhwc_kernel: the partner's intermediate covers every (oy, ox) of its own output, so pass 1
// needs no change.
template <int MIX>
__global__ void augment_ragged_v_kernel(const long long* __restrict__ geom, const float* __restrict__ params,
                                        const uint8_t* __restrict__ inter, bf16* __restrict__ out, RaggedGeom g,
                                        MixParams mix) {
  __shared__ RaggedImage im, pim;
  const int n = blockIdx.y, p = n == 0 ? g.N - 1 : n - 1;
  if (threadIdx.x == 0) load_ragged_image(geom, params, n, g.OH, g.OW, im);
  if (MIX != MixNone && threadIdx.x == 32) load_ragged_image(geom, params, p, g.OH, g.OW, pim);
  __syncthreads();
  const PilAxis va = pil_axis(im.ch, im.RH);
  PilAxis pva = va;
  if constexpr (MIX != MixNone) pva = pil_axis(pim.ch, pim.RH);
  const int pixels = g.OH * g.OW;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < pixels; i += gridDim.x * blockDim.x) {
    const int oy = i / g.OW, ox = i % g.OW;
    float o[3];
    if constexpr (MIX == MixCutMix) {
      if (ox >= mix.x1 && ox < mix.x2 && oy >= mix.y1 && oy < mix.y2)
        ragged_pixel(pim, pva, params + p * 8, inter, g, oy, ox, o);
      else
        ragged_pixel(im, va, params + n * 8, inter, g, oy, ox, o);
    } else {
      ragged_pixel(im, va, params + n * 8, inter, g, oy, ox, o);
    }
    if constexpr (MIX == MixMixUp) {
      float w[3];
      ragged_pixel(pim, pva, params + p * 8, inter, g, oy, ox, w);
#pragma unroll
      for (int c = 0; c < 3; ++c) o[c] = __fadd_rn(__fmul_rn(mix.lam, o[c]), __fmul_rn(mix.lam_b, w[c]));
    }
    *reinterpret_cast<uint2*>(out + (static_cast<long long>(n) * pixels + i) * 4) =
        make_uint2(pack_bf16x2(o[0], o[1]), pack_bf16x2(o[2], 0.f));
  }
}

void augment_ragged(const uint8_t* src, const long long* geom, const float* params, uint8_t* inter, bf16* out,
                    int N, int OH, int OW, int grid_x, const float* mean, const float* stdv, cudaStream_t s,
                    const MixParams* mix) {
  RaggedGeom g;
  g.N = N; g.OH = OH; g.OW = OW;
  for (int c = 0; c < 3; ++c) { g.mean[c] = mean[c]; g.stdv[c] = stdv[c]; }
  const dim3 grid(grid_x, N);
  augment_ragged_h_kernel<<<grid, 256, 0, s>>>(src, geom, params, inter, g);
  if (!mix || mix->kind == MixNone)
    augment_ragged_v_kernel<MixNone><<<grid, 256, 0, s>>>(geom, params, inter, out, g, MixParams{});
  else if (mix->kind == MixMixUp)
    augment_ragged_v_kernel<MixMixUp><<<grid, 256, 0, s>>>(geom, params, inter, out, g, *mix);
  else
    augment_ragged_v_kernel<MixCutMix><<<grid, 256, 0, s>>>(geom, params, inter, out, g, *mix);
  count_launch(2);
  check_last("augment_ragged");
}

// ---- test-time augmentation views of a ragged batch: pass 1 once over the columns and rows every view reads,
// then pass 2 once per view.  Separate kernels, so that augment_ragged's keep their code.
// load_ragged_image with the bounds of the union of the views' chains (the corners of each bound it).
__device__ void load_ragged_image_views(const long long* __restrict__ geom, const float* __restrict__ params, int n,
                                        int OH, int OW, const TtaViews& views, RaggedImage& im) {
  load_ragged_image(geom, params, n, OH, OW, im);
  const float* p = params + n * 8;
  float x0 = 3.4e38f, x1 = -3.4e38f, y0 = 3.4e38f, y1 = -3.4e38f;
  for (int v = 0; v < views.n; ++v) {
    int oy0, ox0;
    bool flip;
    view_origin(static_cast<int>((views.codes >> (4 * v)) & 15u), im.RH, im.RW, OH, OW, oy0, ox0, flip);
    for (int c = 0; c < 4; ++c) {
      float rx, ry;
      ragged_chain_at(p, im.RH, im.RW, oy0, ox0, (p[6] > 0.5f) != flip, (c >> 1) * (OH - 1), (c & 1) * (OW - 1), rx, ry);
      x0 = fminf(x0, rx); x1 = fmaxf(x1, rx); y0 = fminf(y0, ry); y1 = fmaxf(y1, ry);
    }
  }
  im.rx0 = static_cast<int>(fmaxf(x0, 0.f)); im.rx1 = static_cast<int>(fminf(x1, im.RW - 1.f));
  im.ry0 = static_cast<int>(fmaxf(y0, 0.f)); im.ry1 = static_cast<int>(fminf(y1, im.RH - 1.f));
  if (im.ry0 > im.ry1) im.rx1 = im.rx0 - 1;
}

// Pass 1 of augment_ragged_h_kernel over the union of the views.
__global__ void augment_ragged_views_h_kernel(const uint8_t* __restrict__ src, const long long* __restrict__ geom,
                                              const float* __restrict__ params, uint8_t* __restrict__ inter,
                                              RaggedGeom g, TtaViews views) {
  __shared__ RaggedImage im;
  if (threadIdx.x == 0) load_ragged_image_views(geom, params, blockIdx.y, g.OH, g.OW, views, im);
  __syncthreads();
  if (im.rx0 > im.rx1) return;
  const PilAxis va = pil_axis(im.ch, im.RH), ha = pil_axis(im.cw, im.RW);
  const PilWindow first = pil_window(va, im.ry0), last = pil_window(va, im.ry1);
  const int r0 = first.lo, rows = last.lo + last.n - first.lo, cols = im.rx1 - im.rx0 + 1;
  const long long total = static_cast<long long>(rows) * cols;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int r = r0 + static_cast<int>(i / cols), x = im.rx0 + static_cast<int>(i % cols);
    const PilWindow w = pil_window(ha, x);
    const uint8_t* s = src + im.off + (static_cast<long long>(im.top + r) * im.W + im.left + w.lo) * 3;
    int a0 = 1 << (kPilBits - 1), a1 = a0, a2 = a0;
    for (int t = 0; t < w.n; ++t) {
      const int k = pil_fixed(ha, w, t);
      a0 += s[t * 3] * k; a1 += s[t * 3 + 1] * k; a2 += s[t * 3 + 2] * k;
    }
    uint8_t* o = inter + im.inter + (static_cast<long long>(r) * im.RW + x) * 3;
    o[0] = pil_clip8(a0); o[1] = pil_clip8(a1); o[2] = pil_clip8(a2);
  }
}

// Pass 2 for one view: the chain at the view's origin, the view's flip combined with the sample's own.
__global__ void augment_ragged_view_v_kernel(const long long* __restrict__ geom, const float* __restrict__ params,
                                             const uint8_t* __restrict__ inter, bf16* __restrict__ out, RaggedGeom g,
                                             int view) {
  __shared__ RaggedImage im;
  const int n = blockIdx.y;
  if (threadIdx.x == 0) load_ragged_image(geom, params, n, g.OH, g.OW, im);
  __syncthreads();
  const PilAxis va = pil_axis(im.ch, im.RH);
  const float* prm = params + n * 8;
  int y0, x0;
  bool vflip;
  view_origin(view, im.RH, im.RW, g.OH, g.OW, y0, x0, vflip);
  const bool flip = (prm[6] > 0.5f) != vflip;
  const int pixels = g.OH * g.OW;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < pixels; i += gridDim.x * blockDim.x) {
    const int oy = i / g.OW, ox = i % g.OW;
    float rx, ry, o[3];
    ragged_chain_at(prm, im.RH, im.RW, y0, x0, flip, oy, ox, rx, ry);
    ragged_sample(im, va, inter, g, rx, ry, o);
    *reinterpret_cast<uint2*>(out + (static_cast<long long>(n) * pixels + i) * 4) =
        make_uint2(pack_bf16x2(o[0], o[1]), pack_bf16x2(o[2], 0.f));
  }
}

void augment_ragged_view(const uint8_t* src, const long long* geom, const float* params, uint8_t* inter, bf16* out,
                         int N, int OH, int OW, int grid_x, const float* mean, const float* stdv, int view,
                         const TtaViews* pass1, cudaStream_t s) {
  RaggedGeom g;
  g.N = N; g.OH = OH; g.OW = OW;
  for (int c = 0; c < 3; ++c) { g.mean[c] = mean[c]; g.stdv[c] = stdv[c]; }
  const dim3 grid(grid_x, N);
  if (pass1) {
    augment_ragged_views_h_kernel<<<grid, 256, 0, s>>>(src, geom, params, inter, g, *pass1);
    count_launch();
  }
  augment_ragged_view_v_kernel<<<grid, 256, 0, s>>>(geom, params, inter, out, g, view);
  count_launch();
  check_last("augment_ragged_view");
}

// im2col of an already-normalised NHWC (3 channels padded to cpad = 4) bf16 image: the second half
// of the two-pass input path (augment -> 8-byte pixels, 25 MB, stays in L2 -> im2col rows).  One
// thread per (pixel, 8-element chunk): up to four 8-byte pixel loads, one 16-byte store.
__global__ void im2col3x3_c3_kernel(const bf16* __restrict__ x, bf16* __restrict__ out, int N, int H, int W,
                                    int cpad, int kpad) {
  const int chunks = kpad / 8;
  const long long total = static_cast<long long>(N) * H * W * chunks;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int chunk = static_cast<int>(i % chunks);
    const long long pix = i / chunks;
    const int k0 = chunk * 8;
    uint32_t h[8];                                   // bf16 bit patterns, compile-time indexed only
    if (k0 < 27) {
      const int w = pix % W;
      const int hh = (pix / W) % H;
      const long long img = (pix / (static_cast<long long>(W) * H)) * H * W;
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const int k = k0 + e;
        const int tap = k / 3, c = k - 3 * tap;
        const int yy = hh + tap / 3 - 1, xx = w + tap % 3 - 1;
        uint2 px = make_uint2(0u, 0u);
        if (k < 27 && yy >= 0 && yy < H && xx >= 0 && xx < W)
          px = __ldg(reinterpret_cast<const uint2*>(x + (img + static_cast<long long>(yy) * W + xx) * 4));
        h[e] = c == 0 ? (px.x & 0xffffu) : (c == 1 ? (px.x >> 16) : (px.y & 0xffffu));
      }
    } else {
#pragma unroll
      for (int e = 0; e < 8; ++e) h[e] = 0u;
    }
    const uint4 pk = make_uint4(h[0] | (h[1] << 16), h[2] | (h[3] << 16), h[4] | (h[5] << 16), h[6] | (h[7] << 16));
    *reinterpret_cast<uint4*>(out + pix * kpad + k0) = pk;
  }
}

void im2col3x3_c3(const bf16* x, bf16* out, int N, int H, int W, int cpad, int kpad, cudaStream_t s) {
  if (cpad != 4 || kpad % 8 || kpad < 32) throw std::runtime_error("[b200] im2col3x3_c3: cpad must be 4, kpad a multiple of 8 >= 32");
  const long long total = static_cast<long long>(N) * H * W * (kpad / 8);
  const int blocks = static_cast<int>((total + 255) / 256 < sm_count() * 32 ? (total + 255) / 256 : sm_count() * 32);
  im2col3x3_c3_kernel<<<blocks, 256, 0, s>>>(x, out, N, H, W, cpad, kpad);
  count_launch();
  check_last("im2col3x3_c3");
}

__global__ void nchw_f32_to_nhwc_bf16_kernel(const float* __restrict__ x, bf16* __restrict__ y, int N, int C,
                                             int H, int W, int cpad) {
  const long long total = static_cast<long long>(N) * H * W;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long hw = i % (static_cast<long long>(H) * W);
    const long long n = i / (static_cast<long long>(H) * W);
    for (int c = 0; c < cpad; ++c) {
      const float v = c < C ? x[(n * C + c) * H * W + hw] : 0.f;
      y[i * cpad + c] = __float2bfloat16(v);
    }
  }
}

void nchw_f32_to_nhwc_bf16(const float* x, bf16* y, int N, int C, int H, int W, int cpad, cudaStream_t s) {
  const long long total = static_cast<long long>(N) * H * W;
  const int blocks = static_cast<int>((total + 255) / 256 < sm_count() * 16 ? (total + 255) / 256 : sm_count() * 16);
  nchw_f32_to_nhwc_bf16_kernel<<<blocks, 256, 0, s>>>(x, y, N, C, H, W, cpad);
  count_launch();
  check_last("nchw_f32_to_nhwc_bf16");
}

}  // namespace b200
