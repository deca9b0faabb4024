// PowerSGD gradient compression (Vogels et al. 2019; torch's powerSGD_hook) over the fp32 gradient arena.
//
// One compressed tensor is its native row-major gradient range, an n x m matrix.  Per update:
//   psgd_orthogonalize(Q)          Q [m][r] orthonormal columns (modified Gram-Schmidt)
//   psgd_project                   M = g * s + e (written over e), P = M Q   [n][r]
//   (all-reduce P)  psgd_orthogonalize(P)
//   psgd_backproject               Q = M^T P                                 [m][r]
//   (all-reduce Q)  psgd_decompress  G = alpha P Q^T written over g, e = M - G
// Every kernel runs on the comm stream under the convolution backward, so all of them keep the side-stream
// footprint: 256 threads, at most 40 registers (__launch_bounds__(256, 6)), no stack, at most 1 KB of
// static shared memory (block reductions only), the maximum-shared carve-out, and evict-first streaming
// (__ldcs / __stcs) over the n x m operands, which are touched once per pass.  P and Q are small (L2
// resident) and read through the read-only path.  The rank is a template (1..8): the per-thread
// accumulators are r floats, and r = 8 is what fits the register budget.
//
// Every reduction has a fixed order (warp butterflies, then warps 0..7 in order, row splits through
// splitk_reduce in split order), so a launch gives the same bits every time it sees the same inputs.
#include <stdexcept>
#include <string>

#include "api.h"

namespace b200 {

namespace {

constexpr int PT = 256;            // threads per CTA
constexpr int PW = PT / 32;        // warps per CTA

// Row r (R floats, 16-byte aligned when R % 4 == 0) of a small [rows][R] matrix through the read-only path.
template <int R>
__device__ __forceinline__ void load_row(const float* __restrict__ x, long long r, float (&v)[R]) {
  if constexpr (R % 4 == 0) {
#pragma unroll
    for (int k = 0; k < R / 4; ++k) {
      const float4 t = __ldg(reinterpret_cast<const float4*>(x + r * R) + k);
      v[4 * k] = t.x;
      v[4 * k + 1] = t.y;
      v[4 * k + 2] = t.z;
      v[4 * k + 3] = t.w;
    }
  } else {
#pragma unroll
    for (int k = 0; k < R; ++k) v[k] = __ldg(x + r * R + k);
  }
}

// V consecutive floats (V = 2 or 4), evict-first.
template <int V>
__device__ __forceinline__ void ld_stream(const float* x, float (&v)[V]) {
  if constexpr (V == 4) {
    const float4 t = __ldcs(reinterpret_cast<const float4*>(x));
    v[0] = t.x, v[1] = t.y, v[2] = t.z, v[3] = t.w;
  } else {
    const float2 t = __ldcs(reinterpret_cast<const float2*>(x));
    v[0] = t.x, v[1] = t.y;
  }
}
template <int V>
__device__ __forceinline__ void st_stream(float* x, const float (&v)[V]) {
  if constexpr (V == 4)
    __stcs(reinterpret_cast<float4*>(x), make_float4(v[0], v[1], v[2], v[3]));
  else
    __stcs(reinterpret_cast<float2*>(x), make_float2(v[0], v[1]));
}
// Columns per thread and pass of project / decompress: each column takes one Q row of R registers, so
// the wider ranks move 8 bytes per operand instead of 16 to stay inside 40 registers.
template <int R>
constexpr int vec_width() { return R >= 4 ? 2 : 4; }

// Sum of v over the CTA, in a fixed order: xor butterflies within each warp, then warps 0..PW-1.  The
// result is in out[0..R) for every thread on return.  red: PW x R floats of shared memory.
template <int R>
__device__ __forceinline__ void block_sum(float (&v)[R], float* red, float* out) {
#pragma unroll
  for (int k = 0; k < R; ++k) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
  }
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < R; ++k) red[warp * R + k] = v[k];
  }
  __syncthreads();
  if (threadIdx.x < R) {
    float s = red[threadIdx.x];
#pragma unroll
    for (int w = 1; w < PW; ++w) s = __fadd_rn(s, red[w * R + threadIdx.x]);
    out[threadIdx.x] = s;
  }
  __syncthreads();
}

// ---------------------------------------------------------------------------------- project
// One CTA per row (grid-stride): M[i][:] = g[i][:] * s + e[i][:] (one rounding per operation, as torch's
// mean followed by the error add), stored over e; P[i][:] = M[i][:] Q.
template <int R>
__global__ void __launch_bounds__(PT, 6) psgd_project_kernel(const float* __restrict__ g, float* __restrict__ e,
                                                              const float* __restrict__ q, float* __restrict__ p,
                                                              int n, int m, float s) {
  __shared__ float red[PW * R];
  __shared__ float res[R];
  constexpr int V = vec_width<R>();
  const int mv_n = m / V;
  for (int i = blockIdx.x; i < n; i += gridDim.x) {
    const float* gi = g + static_cast<long long>(i) * m;
    float* ei = e + static_cast<long long>(i) * m;
    float acc[R];
#pragma unroll
    for (int k = 0; k < R; ++k) acc[k] = 0.f;
    for (int j = threadIdx.x; j < mv_n; j += PT) {
      float gv[V], mv[V];
      ld_stream<V>(gi + j * V, gv);
      ld_stream<V>(ei + j * V, mv);
#pragma unroll
      for (int c = 0; c < V; ++c) mv[c] = __fadd_rn(__fmul_rn(gv[c], s), mv[c]);
      st_stream<V>(ei + j * V, mv);
#pragma unroll
      for (int c = 0; c < V; ++c) {
        float qv[R];
        load_row<R>(q, static_cast<long long>(j) * V + c, qv);
#pragma unroll
        for (int k = 0; k < R; ++k) acc[k] = fmaf(mv[c], qv[k], acc[k]);
      }
    }
    block_sum<R>(acc, red, res);
    if (threadIdx.x < R) p[static_cast<long long>(i) * R + threadIdx.x] = res[threadIdx.x];
  }
}

// ------------------------------------------------------------------------------ back-project
// Column j of a row split: ws[split][j][:] = sum over the split's rows i (in order) of M[i][j] P[i][:].
// One thread per column, 256 columns per CTA, blockIdx.y = split; splitk_reduce adds the splits in order.
template <int R>
__global__ void __launch_bounds__(PT, 6) psgd_backproject_kernel(const float* __restrict__ M,
                                                                  const float* __restrict__ p, float* __restrict__ ws,
                                                                  int n, int m, int rows_per_split, long long slice) {
  const int j = blockIdx.x * PT + threadIdx.x;
  if (j >= m) return;
  const int i0 = blockIdx.y * rows_per_split;
  const int i1 = min(n, i0 + rows_per_split);
  float acc[R];
#pragma unroll
  for (int k = 0; k < R; ++k) acc[k] = 0.f;
  const float* col = M + j;
#pragma unroll(R > 4 ? 2 : 4)
  for (int i = i0; i < i1; ++i) {
    const float x = __ldcs(col + static_cast<long long>(i) * m);
    float pv[R];
    load_row<R>(p, i, pv);
#pragma unroll
    for (int k = 0; k < R; ++k) acc[k] = fmaf(x, pv[k], acc[k]);
  }
  float* out = ws + blockIdx.y * slice + static_cast<long long>(j) * R;
#pragma unroll
  for (int k = 0; k < R; ++k) out[k] = acc[k];
}

// ----------------------------------------------------------------------------- orthogonalize
// Modified Gram-Schmidt over the R columns of one [rows][R] matrix per CTA, as torch's
// _orthogonalize_gram_schmidt: for each column i, normalise it, then subtract its projection from every later
// column.  A column of norm 0 stays 0 (torch would divide 0 by 0).  2R passes over the matrix; the column
// norm of i + 1 is gathered in the subtraction pass of column i.
template <int R>
__global__ void __launch_bounds__(PT, 6) psgd_orthogonalize_kernel(float* __restrict__ x_all, int rows) {
  __shared__ float red[PW * R];
  __shared__ float res[R];
  float* x = x_all + static_cast<long long>(blockIdx.x) * rows * R;
  float part[R];
#pragma unroll
  for (int k = 0; k < R; ++k) part[k] = 0.f;
  for (int t = threadIdx.x; t < rows; t += PT) part[0] = fmaf(x[t * R], x[t * R], part[0]);
  block_sum<R>(part, red, res);
  float nrm2 = res[0];
#pragma unroll
  for (int i = 0; i < R; ++i) {
    const float nrm = sqrtf(nrm2);
#pragma unroll
    for (int k = 0; k < R; ++k) part[k] = 0.f;
    for (int t = threadIdx.x; t < rows; t += PT) {
      float* row = x + static_cast<long long>(t) * R;
      const float xi = nrm > 0.f ? __fdiv_rn(row[i], nrm) : 0.f;
      row[i] = xi;
#pragma unroll
      for (int k = i + 1; k < R; ++k) part[k] = fmaf(xi, row[k], part[k]);
    }
    if (i + 1 == R) break;
    block_sum<R>(part, red, res);
    float d[R];
#pragma unroll
    for (int k = 0; k < R; ++k) d[k] = res[k];
    float ss[1] = {0.f};
    for (int t = threadIdx.x; t < rows; t += PT) {
      float* row = x + static_cast<long long>(t) * R;
      const float xi = row[i];
#pragma unroll
      for (int k = i + 1; k < R; ++k) row[k] = __fsub_rn(row[k], __fmul_rn(d[k], xi));
      ss[0] = fmaf(row[i + 1], row[i + 1], ss[0]);
    }
    block_sum<1>(ss, red, res);
    nrm2 = res[0];
  }
}

// ------------------------------------------------------------------------------- decompress
// One CTA per row (grid-stride): G[i][j] = alpha * (P[i][:] . Q[j][:]) stored over g, e[i][j] = M[i][j] - G[i][j]
// (M is what psgd_project left in e).
template <int R>
__global__ void __launch_bounds__(PT, 6) psgd_decompress_kernel(const float* __restrict__ p,
                                                                 const float* __restrict__ q, float* __restrict__ g,
                                                                 float* __restrict__ e, int n, int m, float alpha) {
  constexpr int V = vec_width<R>();
  const int mv_n = m / V;
  __shared__ float pv[R];            // P[i][:], read as broadcasts: R registers fewer than a private copy
  for (int i = blockIdx.x; i < n; i += gridDim.x) {
    if (threadIdx.x < R) pv[threadIdx.x] = p[static_cast<long long>(i) * R + threadIdx.x];
    __syncthreads();
    float* gi = g + static_cast<long long>(i) * m;
    float* ei = e + static_cast<long long>(i) * m;
    for (int j = threadIdx.x; j < mv_n; j += PT) {
      float mv[V], gc[V];
      ld_stream<V>(ei + j * V, mv);
#pragma unroll
      for (int c = 0; c < V; ++c) {
        float qv[R];
        load_row<R>(q, static_cast<long long>(j) * V + c, qv);
        float a = 0.f;
#pragma unroll
        for (int k = 0; k < R; ++k) a = fmaf(pv[k], qv[k], a);
        gc[c] = __fmul_rn(a, alpha);
        mv[c] = __fsub_rn(mv[c], gc[c]);
      }
      st_stream<V>(gi + j * V, gc);
      st_stream<V>(ei + j * V, mv);
    }
    __syncthreads();                  // pv is rewritten for the next row
  }
}

template <int R>
void carve_all() {
  prefer_max_shared_carveout(reinterpret_cast<const void*>(psgd_project_kernel<R>));
  prefer_max_shared_carveout(reinterpret_cast<const void*>(psgd_backproject_kernel<R>));
  prefer_max_shared_carveout(reinterpret_cast<const void*>(psgd_orthogonalize_kernel<R>));
  prefer_max_shared_carveout(reinterpret_cast<const void*>(psgd_decompress_kernel<R>));
}

void carve_once() {
  static const bool done = [] {
    carve_all<1>();
    carve_all<2>();
    carve_all<3>();
    carve_all<4>();
    carve_all<5>();
    carve_all<6>();
    carve_all<7>();
    carve_all<8>();
    return true;
  }();
  (void)done;
}

void check_shape(const char* op, int n, int m, int rank) {
  if (rank < 1 || rank > PSGD_MAX_RANK)
    throw std::runtime_error(std::string("[b200] ") + op + ": rank must lie in [1, 8]: each thread keeps r fp32 "
                             "accumulators, and more than 8 do not fit the 40-register budget of a comm-stream kernel");
  if (n < 1 || m < 4 || m % 4)
    throw std::runtime_error(std::string("[b200] ") + op + ": needs n >= 1 rows and m >= 4 columns, m a multiple of 4");
}

void check_ptr(const char* op, const void* ptr) {
  if (!ptr || (reinterpret_cast<uintptr_t>(ptr) & 15))
    throw std::runtime_error(std::string("[b200] ") + op + ": operands must be non-null and 16-byte aligned");
}

// Rows per CTA-row-split of the back-projection: about four CTAs per SM over the grid.
int backproject_rows(int n, int m, int sms) {
  const int tiles = (m + PT - 1) / PT;
  int splits = (4 * sms + tiles - 1) / tiles;
  splits = splits < 1 ? 1 : (splits > n ? n : splits);
  return (n + splits - 1) / splits;
}

template <typename F>
void dispatch(int rank, F&& f) {
  switch (rank) {
    case 1: f(std::integral_constant<int, 1>()); break;
    case 2: f(std::integral_constant<int, 2>()); break;
    case 3: f(std::integral_constant<int, 3>()); break;
    case 4: f(std::integral_constant<int, 4>()); break;
    case 5: f(std::integral_constant<int, 5>()); break;
    case 6: f(std::integral_constant<int, 6>()); break;
    case 7: f(std::integral_constant<int, 7>()); break;
    default: f(std::integral_constant<int, 8>()); break;
  }
}

int row_grid(int n) {
  const int cap = sm_count() * 6;
  return n < cap ? n : cap;
}

}  // namespace

int psgd_backproject_splits(int n, int m, int sms) {
  const int rps = backproject_rows(n, m, sms);
  return (n + rps - 1) / rps;
}

long long psgd_workspace_elems(int n, int m, int rank, int sms) {
  return psgd_backproject_splits(n, m, sms) * workspace_slice(static_cast<long long>(m) * rank);
}

void psgd_project(const float* g, float* e, const float* q, float* p, int n, int m, int rank, float scale,
                  cudaStream_t s) {
  check_shape("psgd_project", n, m, rank);
  for (const void* t : {static_cast<const void*>(g), static_cast<const void*>(e), static_cast<const void*>(q),
                        static_cast<const void*>(p)})
    check_ptr("psgd_project", t);
  carve_once();
  dispatch(rank, [&](auto r) {
    psgd_project_kernel<decltype(r)::value><<<row_grid(n), PT, 0, s>>>(g, e, q, p, n, m, scale);
  });
  count_launch();
  check_last("psgd_project");
}

void psgd_backproject(const float* M, const float* p, float* q, float* ws, long long ws_elems, int n, int m, int rank,
                      cudaStream_t s) {
  check_shape("psgd_backproject", n, m, rank);
  for (const void* t : {static_cast<const void*>(M), static_cast<const void*>(p), static_cast<const void*>(q),
                        static_cast<const void*>(ws)})
    check_ptr("psgd_backproject", t);
  const int sms = sm_count();
  const int rps = backproject_rows(n, m, sms);
  const int splits = (n + rps - 1) / rps;
  const long long slice = workspace_slice(static_cast<long long>(m) * rank);
  if (ws_elems < splits * slice)
    throw std::runtime_error("[b200] psgd_backproject: the workspace holds " + std::to_string(ws_elems) +
                             " floats, the launch needs " + std::to_string(splits * slice));
  carve_once();
  const dim3 grid((m + PT - 1) / PT, splits);
  dispatch(rank, [&](auto r) {
    psgd_backproject_kernel<decltype(r)::value><<<grid, PT, 0, s>>>(M, p, ws, n, m, rps, slice);
  });
  count_launch();
  check_last("psgd_backproject");
  splitk_reduce(ws, ws_elems, q, static_cast<long long>(m) * rank, slice, splits, 1.f, false, s);
}

void psgd_orthogonalize(float* x, int rows, int count, int rank, cudaStream_t s) {
  check_shape("psgd_orthogonalize", count, 4, rank);
  if (rows < rank)
    throw std::runtime_error("[b200] psgd_orthogonalize: needs at least as many rows as columns");
  check_ptr("psgd_orthogonalize", x);
  carve_once();
  dispatch(rank, [&](auto r) { psgd_orthogonalize_kernel<decltype(r)::value><<<count, PT, 0, s>>>(x, rows); });
  count_launch();
  check_last("psgd_orthogonalize");
}

void psgd_decompress(const float* p, const float* q, float* g, float* e, int n, int m, int rank, float alpha,
                     cudaStream_t s) {
  check_shape("psgd_decompress", n, m, rank);
  for (const void* t : {static_cast<const void*>(p), static_cast<const void*>(q), static_cast<const void*>(g),
                        static_cast<const void*>(e)})
    check_ptr("psgd_decompress", t);
  carve_once();
  dispatch(rank, [&](auto r) {
    psgd_decompress_kernel<decltype(r)::value><<<row_grid(n), PT, 0, s>>>(p, q, g, e, n, m, alpha);
  });
  count_launch();
  check_last("psgd_decompress");
}

}  // namespace b200
