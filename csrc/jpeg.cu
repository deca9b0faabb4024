// Device half of the streaming JPEG pipeline (--pipeline stream): the host threads stop at the quantised
// coefficients (csrc/jpeg_decode.cpp); these two launches turn a batch of them into the uint8 HWC images
// augment_ragged reads, at each image's geometry offset.  The result is Pillow's decode bit for bit: the
// arithmetic is libjpeg's (jidctint.c's JDCT_ISLOW IDCT with its range-limit table, jdsample.c's fancy
// upsampling, jdcolor.c's fixed-point YCbCr -> RGB), restated in data/jpeg.py, the reference of the tests.
// No atomics: every output byte is written by exactly one thread.
#include <stdexcept>

#include "api.h"
#include "jpeg.h"

namespace b200 {

namespace {

constexpr int kIdctBlocks = 16;           // 8x8 blocks per CTA, 8 threads each

// One jidctint pass over 8 values; outputs descaled by `shift` (libjpeg's DESCALE: add half, shift right).
// 64-bit products, as libjpeg's JLONG.
__device__ __forceinline__ void idct8(const long long* in, long long* out, int shift) {
  const long long c0298 = 2446, c0390 = 3196, c0541 = 4433, c0765 = 6270, c0899 = 7373, c1175 = 9633, c1501 = 12299,
            c1847 = 15137, c1961 = 16069, c2053 = 16819, c2562 = 20995, c3072 = 25172;
  long long z2 = in[2], z3 = in[6];
  long long z1 = (z2 + z3) * c0541;
  const long long tmp2 = z1 - z3 * c1847, tmp3 = z1 + z2 * c0765;
  const long long tmp0 = (in[0] + in[4]) * 8192, tmp1 = (in[0] - in[4]) * 8192;
  const long long tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
  long long t0 = in[7], t1 = in[5], t2 = in[3], t3 = in[1];
  z1 = t0 + t3;
  z2 = t1 + t2;
  z3 = t0 + t2;
  long long z4 = t1 + t3;
  const long long z5 = (z3 + z4) * c1175;
  t0 *= c0298; t1 *= c2053; t2 *= c3072; t3 *= c1501;
  z1 *= -c0899; z2 *= -c2562;
  z3 = z3 * -c1961 + z5;
  z4 = z4 * -c0390 + z5;
  t0 += z1 + z3; t1 += z2 + z4; t2 += z2 + z3; t3 += z1 + z4;
  const long long r = 1ll << (shift - 1);
  out[0] = (tmp10 + t3 + r) >> shift; out[7] = (tmp10 - t3 + r) >> shift;
  out[1] = (tmp11 + t2 + r) >> shift; out[6] = (tmp11 - t2 + r) >> shift;
  out[2] = (tmp12 + t1 + r) >> shift; out[5] = (tmp12 - t1 + r) >> shift;
  out[3] = (tmp13 + t0 + r) >> shift; out[4] = (tmp13 - t0 + r) >> shift;
}

// libjpeg's post-IDCT range-limit table, indexed with x & 1023 (x: the descaled sample before +128).
__device__ __forceinline__ unsigned range_limit(long long x) {
  const int t = (int)(x & 1023);
  return t < 128 ? t + 128 : (t < 512 ? 255 : (t < 896 ? 0 : t - 896));
}

__device__ __forceinline__ int sample(const uint8_t* __restrict__ plane, int bw, int x, int y) {
  return plane[((long long)((y >> 3) * bw + (x >> 3)) << 6) | ((y & 7) << 3) | (x & 7)];
}

// Chroma at full-resolution pixel (x, y) of an H x W image with luma sampling (hmax, vmax): jdsample.c's
// h2v1 / h2v2 fancy upsampling over the real ceil(W / hmax) x ceil(H / vmax) samples, replication when the
// component is at most two samples wide.
__device__ __forceinline__ int chroma(const uint8_t* __restrict__ pl, int bw, int x, int y, int H, int W, int hmax,
                                      int vmax) {
  if (hmax == 1) return sample(pl, bw, x, y);
  const int cw = (W + 1) >> 1, k = x >> 1;
  if (cw <= 2) return sample(pl, bw, k, y / vmax);
  const bool odd = x & 1;
  if (vmax == 1) {
    const int c = sample(pl, bw, k, y);
    if (!odd) return k == 0 ? c : (3 * c + sample(pl, bw, k - 1, y) + 1) >> 2;
    return k == cw - 1 ? c : (3 * c + sample(pl, bw, k + 1, y) + 2) >> 2;
  }
  const int ch = (H + 1) >> 1, ky = y >> 1;
  const int ny = (y & 1) ? min(ky + 1, ch - 1) : max(ky - 1, 0);
  const int cs = 3 * sample(pl, bw, k, ky) + sample(pl, bw, k, ny);
  if (!odd) return k == 0 ? (4 * cs + 8) >> 4 : (3 * cs + 3 * sample(pl, bw, k - 1, ky) + sample(pl, bw, k - 1, ny) + 8) >> 4;
  return k == cw - 1 ? (4 * cs + 7) >> 4
                     : (3 * cs + 3 * sample(pl, bw, k + 1, ky) + sample(pl, bw, k + 1, ny) + 7) >> 4;
}

}  // namespace

// Launch 1: dequantise + IDCT every 8x8 block of the batch into the block-major sample planes.  Thread t of a
// block's eight does column t, then row t.
__global__ void __launch_bounds__(8 * kIdctBlocks) jpeg_idct_kernel(const int16_t* __restrict__ coef,
                                                                    const int* __restrict__ quant,
                                                                    const int* __restrict__ desc, int k,
                                                                    long long total, uint8_t* __restrict__ planes) {
  __shared__ int ws[kIdctBlocks][64];     // jidctint's int workspace
  const int g = threadIdx.x >> 3, t = threadIdx.x & 7;
  const long long blk = (long long)blockIdx.x * kIdctBlocks + g;
  const bool live = blk < total;
  if (live) {
    int lo = 0, hi = k - 1;               // last image whose first block is <= blk
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (desc[mid * kJpegDesc + 3] <= blk) lo = mid; else hi = mid - 1;
    }
    const int* d = desc + lo * kJpegDesc;
    const long long local = blk - d[3], n0 = (long long)d[5] * d[8], n1 = (long long)d[6] * d[9];
    const int c = local < n0 ? 0 : (local < n0 + n1 ? 1 : 2);
    const int* q = quant + d[11 + c] * 64;
    const int16_t* src = coef + blk * 64;
    long long in[8], out[8];
#pragma unroll
    for (int r = 0; r < 8; ++r) in[r] = (long long)src[r * 8 + t] * q[r * 8 + t];
    idct8(in, out, 11);                   // CONST_BITS - PASS1_BITS
#pragma unroll
    for (int r = 0; r < 8; ++r) ws[g][r * 8 + t] = (int)out[r];
  }
  __syncthreads();
  if (live) {
    long long in[8], out[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) in[j] = ws[g][t * 8 + j];
    idct8(in, out, 18);                   // CONST_BITS + PASS1_BITS + 3
    uint2 v;
    v.x = range_limit(out[0]) | range_limit(out[1]) << 8 | range_limit(out[2]) << 16 | range_limit(out[3]) << 24;
    v.y = range_limit(out[4]) | range_limit(out[5]) << 8 | range_limit(out[6]) << 16 | range_limit(out[7]) << 24;
    *reinterpret_cast<uint2*>(planes + blk * 64 + t * 8) = v;
  }
}

// Launch 2: upsampling + colour conversion (grey: replicated), HWC uint8 at geom's offset; raw-RGB members are
// copied.  blockIdx.y: the image; the x blocks stride over its pixels.
__global__ void __launch_bounds__(256) jpeg_color_kernel(const uint8_t* __restrict__ planes,
                                                         const uint8_t* __restrict__ raw, const int* __restrict__ desc,
                                                         const long long* __restrict__ geom, uint8_t* __restrict__ out) {
  const int i = blockIdx.y;
  const int* d = desc + i * kJpegDesc;
  const long long off = geom[i * 5];
  const int H = (int)geom[i * 5 + 1], W = (int)geom[i * 5 + 2];
  const long long HW = (long long)H * W;
  const int n = d[0];
  const uint8_t* p0 = planes + (long long)d[3] * 64;
  const uint8_t* p1 = p0 + (long long)d[5] * d[8] * 64;
  const uint8_t* p2 = p1 + (long long)d[6] * d[9] * 64;
  uint8_t* dst = out + off;
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < HW; p += (long long)gridDim.x * blockDim.x) {
    uint8_t* o = dst + p * 3;
    if (n == 0) {
      const uint8_t* s = raw + d[4] + p * 3;
      o[0] = s[0]; o[1] = s[1]; o[2] = s[2];
      continue;
    }
    const int y = (int)(p / W), x = (int)(p - (long long)y * W);
    const int Y = sample(p0, d[5], x, y);
    if (n == 1) {
      o[0] = o[1] = o[2] = (uint8_t)Y;
      continue;
    }
    const int cb = chroma(p1, d[6], x, y, H, W, d[1], d[2]) - 128, cr = chroma(p2, d[7], x, y, H, W, d[1], d[2]) - 128;
    const int r = Y + ((91881 * cr + 32768) >> 16);                   // jdcolor.c, SCALEBITS 16
    const int gg = Y + ((-22554 * cb + 32768 - 46802 * cr) >> 16);
    const int b = Y + ((116130 * cb + 32768) >> 16);
    o[0] = (uint8_t)min(max(r, 0), 255);
    o[1] = (uint8_t)min(max(gg, 0), 255);
    o[2] = (uint8_t)min(max(b, 0), 255);
  }
}

void jpeg_decode(const int16_t* coef, const int* quant, const int* desc, const long long* geom, const uint8_t* raw,
                 uint8_t* planes, uint8_t* out, int k, long long total_blocks, int grid_x, cudaStream_t s) {
  int launches = 1;
  if (total_blocks > 0) {
    jpeg_idct_kernel<<<(unsigned)((total_blocks + kIdctBlocks - 1) / kIdctBlocks), 8 * kIdctBlocks, 0, s>>>(
        coef, quant, desc, k, total_blocks, planes);
    ++launches;
  }
  jpeg_color_kernel<<<dim3(grid_x, k), 256, 0, s>>>(planes, raw, desc, geom, out);
  count_launch(launches);
  check_last("jpeg_decode");
}

}  // namespace b200
