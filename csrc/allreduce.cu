// Fused gradient all-reduce over NVLink peer memory (K-AR) -- no NCCL on this path.
//
// What the reference gets from DDP's Reducer + a gloo ring (distributedVggf.py:225, SURVEY N3/N4):
// grad <- (1/ws) * sum over ranks, per bucket, overlapped with the rest of backward.  Here one
// kernel per bucket does, on a side stream while backward keeps running:
//
//   pack     wire[i] = bf16(grad_f32[i] * 1/ws)            local fp32 arena -> symmetric wire
//   barrier  CTA b of every rank handshakes with CTA b of every peer (flags in peer memory,
//            st.release.sys / ld.acquire.sys); CTAs never wait for other CTAs of the same GPU
//   reduce   one-shot : every rank loads chunk b from all peers, sums in fp32, keeps it locally
//            two-shot : rank r loads its 1/ws sub-slice of chunk b from all peers, sums in fp32,
//                       and pushes the bf16 result into every peer's wire (reduce-scatter +
//                       all-gather in one pass, 2(ws-1)/ws bytes per element on the wire)
//            NVLS     : rank r issues multimem.ld_reduce (the switch adds the ws copies with fp32
//                       accumulation) on its sub-slice and multimem.st broadcasts the result
//   barrier  everybody is done reading / writing my wire
//   unpack   optional fp32 write-back into the arena (the fused Adam can read the bf16 wire
//            directly instead)
//
// Work decomposition: the bucket is cut into G chunks (one per CTA), each chunk into `world`
// cells; cell (b, r) is reduced by CTA b of rank r.  A chunk is only ever touched by the CTAs
// with the same index, which is what makes the per-CTA handshake sufficient.
#include <cmath>
#include <stdexcept>

#include "adam.cuh"
#include "api.h"
#include "ptx.cuh"

namespace b200 {

// Footprint: the comm stream's CTAs run WHILE the persistent wgmma kernels of backward hold every
// SM.  A 256-thread CTA capped at 40 registers (10 240) and no shared memory fits next to a
// persistent CTA only where that leaves 10 240 registers free.  None of the wgmma kernels does:
// umma_kernel, conv_halo_kernel and wgrad_halo64_kernel are 512-thread CTAs at 128 registers
// (65 536, redistributed between their warpgroups with setmaxnreg), and conv0_kernel has 640
// threads.  `cuobjdump --dump-resource-usage` on the
// library lists each kernel's count.  Where a conv CTA fills the SM, reduction CTAs wait for it to
// finish; thin CTAs (bytes in flight = CTAs x 256 threads x UNR x 16 B) still keep the footprint of
// each small.
constexpr int AR_MAX_CTAS = 128;
constexpr int AR_THREADS = 256;
constexpr int AR_MIN_BLOCKS = 6;                                // __launch_bounds__ -> <= 40 registers
constexpr int AR_SLOT_WORDS = 2 * AR_MAX_CTAS * AR_MAX_WORLD;   // two phases per slot

__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

__device__ __forceinline__ uint32_t* flag_ptr(uint32_t* pad, int slot, int phase, int cta, int src) {
  return pad + ((static_cast<long long>(slot) * 2 + phase) * AR_MAX_CTAS + cta) * AR_MAX_WORLD + src;
}

// Handshake between the CTAs with index `cta` on all ranks.  Thread t < world talks to peer t.
__device__ __forceinline__ void cta_barrier_all_ranks(const CommCtx& c, int slot, int phase, int cta,
                                                      uint32_t epoch) {
  __syncthreads();
  if (threadIdx.x < c.world) {
    const int peer = threadIdx.x;
    fence_acq_rel_sys();
    st_release_sys(flag_ptr(c.signal_ptrs[peer], slot, phase, cta, c.rank), epoch);
    const uint32_t* mine = flag_ptr(c.signal_ptrs[c.rank], slot, phase, cta, peer);
    // Bounded by WALL CLOCK (%globaltimer), not by a spin count: a peer may legitimately be late by
    // seconds (rank 0 writing a checkpoint, a slow first batch) -- the limit is minutes and
    // configurable (B200_BARRIER_TIMEOUT_S), and only a genuinely dead peer trips it.
    unsigned int spins = 0;
    unsigned long long t0 = 0;
    while (static_cast<int>(ld_acquire_sys(mine) - epoch) < 0) {
      if ((++spins & 1023u) == 0) {
        const unsigned long long now = globaltimer_ns();
        if (t0 == 0) t0 = now;
        if (now - t0 > c.timeout_ns) {
          printf("[b200] cross-GPU barrier timeout rank=%d peer=%d slot=%d phase=%d cta=%d epoch=%u seen=%u\n",
                 c.rank, peer, slot, phase, cta, epoch, ld_relaxed_sys(mine));
          __trap();
        }
      }
    }
  }
  __syncthreads();
}

__device__ __forceinline__ uint4 ld_v4(const void* p) {
  uint4 v;
  asm volatile("ld.global.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p)
               : "memory");
  return v;
}

__device__ __forceinline__ void accum_bf16x8(float (&acc)[8], const uint4& v) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 f = unpack_bf16x2(w[i]);
    acc[2 * i] += f.x;
    acc[2 * i + 1] += f.y;
  }
}

struct ArArgs {
  CommCtx c;
  const float* grad;       // local fp32 arena (nullptr: wire already holds the packed data)
  float* grad_out;         // optional fp32 write-back
  long long start;         // element offset of the bucket inside arena and wire
  long long n;             // elements (multiple of 8)
  float inv_world;
  int slot;
  uint32_t epoch;
};

// One 16-byte wire vector = 8 bf16 (WIRE32 = false) or 4 fp32 (WIRE32 = true).
template <int ALGO, bool WIRE32>
__global__ void __launch_bounds__(AR_THREADS, AR_MIN_BLOCKS) allreduce_kernel(const ArArgs a) {
  constexpr int EPV = WIRE32 ? 4 : 8;                 // elements per vector
  const CommCtx& c = a.c;
  const int b = blockIdx.x, G = gridDim.x, world = c.world, rank = c.rank;
  const long long nvec = a.n / EPV;
  const long long cell = (nvec + static_cast<long long>(G) * world - 1) / (static_cast<long long>(G) * world);
  const long long chunk0 = min(nvec, static_cast<long long>(b) * world * cell);
  const long long chunk1 = min(nvec, static_cast<long long>(b + 1) * world * cell);
  uint8_t* my_wire = reinterpret_cast<uint8_t*>(c.wire_ptrs[rank]) + a.start * (WIRE32 ? 4 : 2);

  // ---- pack: fp32 arena -> wire (scaled, rounded once) -----------------------------------------
  constexpr int UNR = 4;        // independent 16-byte wire transactions in flight per thread
  constexpr int PUNR = 2;       // pack: 2 x 32 fp32 bytes in flight per thread (register budget)
  if (a.grad) {
    const float* g = a.grad + a.start;
    const float s = a.inv_world;
    long long v = chunk0 + threadIdx.x;
    if constexpr (!WIRE32) {
      for (; v + (PUNR - 1) * AR_THREADS < chunk1; v += PUNR * AR_THREADS) {
        float4 x0[PUNR], x1[PUNR];
#pragma unroll
        for (int u = 0; u < PUNR; ++u) {
          x0[u] = __ldcs(reinterpret_cast<const float4*>(g + (v + u * AR_THREADS) * 8));      // read once: streaming
          x1[u] = __ldcs(reinterpret_cast<const float4*>(g + (v + u * AR_THREADS) * 8 + 4));
        }
#pragma unroll
        for (int u = 0; u < PUNR; ++u)
          st_v4(my_wire + (v + u * AR_THREADS) * 16,
                make_uint4(pack_bf16x2(x0[u].x * s, x0[u].y * s), pack_bf16x2(x0[u].z * s, x0[u].w * s),
                           pack_bf16x2(x1[u].x * s, x1[u].y * s), pack_bf16x2(x1[u].z * s, x1[u].w * s)));
      }
    }
    for (; v < chunk1; v += AR_THREADS) {
      if constexpr (WIRE32) {
        float4 x = *reinterpret_cast<const float4*>(g + v * 4);
        x.x *= s; x.y *= s; x.z *= s; x.w *= s;
        *reinterpret_cast<float4*>(my_wire + v * 16) = x;
      } else {
        const float4 x0 = *reinterpret_cast<const float4*>(g + v * 8);
        const float4 x1 = *reinterpret_cast<const float4*>(g + v * 8 + 4);
        st_v4(my_wire + v * 16, make_uint4(pack_bf16x2(x0.x * s, x0.y * s), pack_bf16x2(x0.z * s, x0.w * s),
                                           pack_bf16x2(x1.x * s, x1.y * s), pack_bf16x2(x1.z * s, x1.w * s)));
      }
    }
  }
  cta_barrier_all_ranks(c, a.slot, 0, b, a.epoch);

  // ---- reduce ---------------------------------------------------------------------------------
  if constexpr (ALGO == AR_ONESHOT) {
    // every rank reduces the whole chunk; result goes to the local fp32 arena (never to the wire,
    // which peers are still reading).
    float* out = a.grad_out + a.start;
    for (long long v = chunk0 + threadIdx.x; v < chunk1; v += AR_THREADS) {
      if constexpr (WIRE32) {
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int peer = 0; peer < world; ++peer) {   // fixed order: bit-identical sums on every rank
          const uint4 raw = ld_v4(reinterpret_cast<const uint8_t*>(c.wire_ptrs[peer]) + a.start * 4 + v * 16);
          acc.x += __uint_as_float(raw.x); acc.y += __uint_as_float(raw.y);
          acc.z += __uint_as_float(raw.z); acc.w += __uint_as_float(raw.w);
        }
        *reinterpret_cast<float4*>(out + v * 4) = acc;
      } else {
        float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        for (int peer = 0; peer < world; ++peer)
          accum_bf16x8(acc, ld_v4(reinterpret_cast<const uint8_t*>(c.wire_ptrs[peer]) + a.start * 2 + v * 16));
        *reinterpret_cast<float4*>(out + v * 8) = make_float4(acc[0], acc[1], acc[2], acc[3]);
        *reinterpret_cast<float4*>(out + v * 8 + 4) = make_float4(acc[4], acc[5], acc[6], acc[7]);
      }
    }
    cta_barrier_all_ranks(c, a.slot, 1, b, a.epoch);
    return;
  }

  const long long cell0 = min(chunk1, chunk0 + static_cast<long long>(rank) * cell);
  const long long cell1 = min(chunk1, cell0 + cell);
  if constexpr (ALGO == AR_TWOSHOT) {
    for (long long v = cell0 + threadIdx.x; v < cell1; v += AR_THREADS) {
      const long long boff = a.start * (WIRE32 ? 4 : 2) + v * 16;
      uint4 res;
      if constexpr (WIRE32) {
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int p = 0; p < world; ++p) {
          const int peer = (rank + p) % world;
          const uint4 raw = ld_v4(reinterpret_cast<const uint8_t*>(c.wire_ptrs[peer]) + boff);
          acc.x += __uint_as_float(raw.x); acc.y += __uint_as_float(raw.y);
          acc.z += __uint_as_float(raw.z); acc.w += __uint_as_float(raw.w);
        }
        res = make_uint4(__float_as_uint(acc.x), __float_as_uint(acc.y), __float_as_uint(acc.z), __float_as_uint(acc.w));
      } else {
        float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        int p = 0;
        for (; p + 4 <= world; p += 4) {          // four peer loads in flight, then accumulate
          uint4 r4[4];
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            int peer = rank + p + u;
            if (peer >= world) peer -= world;
            r4[u] = ld_v4(reinterpret_cast<const uint8_t*>(c.wire_ptrs[peer]) + boff);
          }
#pragma unroll
          for (int u = 0; u < 4; ++u) accum_bf16x8(acc, r4[u]);
        }
        for (; p < world; ++p) {
          int peer = rank + p;
          if (peer >= world) peer -= world;
          accum_bf16x8(acc, ld_v4(reinterpret_cast<const uint8_t*>(c.wire_ptrs[peer]) + boff));
        }
        res = make_uint4(pack_bf16x2(acc[0], acc[1]), pack_bf16x2(acc[2], acc[3]),
                         pack_bf16x2(acc[4], acc[5]), pack_bf16x2(acc[6], acc[7]));
      }
      for (int p = 0; p < world; ++p) {
        const int peer = (rank + p) % world;
        st_v4(reinterpret_cast<uint8_t*>(c.wire_ptrs[peer]) + boff, res);
      }
    }
  } else {   // AR_NVLS: the switch reduces and broadcasts
    uint8_t* mc = reinterpret_cast<uint8_t*>(c.wire_mc) + a.start * (WIRE32 ? 4 : 2);
    long long v = cell0 + threadIdx.x;
    if constexpr (!WIRE32) {
      for (; v + (UNR - 1) * AR_THREADS < cell1; v += UNR * AR_THREADS) {
        uint4 r[UNR];
#pragma unroll
        for (int u = 0; u < UNR; ++u) r[u] = multimem_ld_reduce_bf16x8(mc + (v + u * AR_THREADS) * 16);
#pragma unroll
        for (int u = 0; u < UNR; ++u) multimem_st_v4(mc + (v + u * AR_THREADS) * 16, r[u]);
      }
    }
    for (; v < cell1; v += AR_THREADS) {
      if constexpr (WIRE32) {
        const float4 r = multimem_ld_reduce_f32x4(mc + v * 16);
        multimem_st_v4(mc + v * 16, make_uint4(__float_as_uint(r.x), __float_as_uint(r.y),
                                               __float_as_uint(r.z), __float_as_uint(r.w)));
      } else {
        multimem_st_v4(mc + v * 16, multimem_ld_reduce_bf16x8(mc + v * 16));
      }
    }
  }
  cta_barrier_all_ranks(c, a.slot, 1, b, a.epoch);

  // ---- unpack (optional): wire -> fp32 arena ----------------------------------------------------
  if (a.grad_out) {
    float* out = a.grad_out + a.start;
    long long v = chunk0 + threadIdx.x;
    if constexpr (!WIRE32) {
      for (; v + (UNR - 1) * AR_THREADS < chunk1; v += UNR * AR_THREADS) {
        uint4 raw[UNR];
#pragma unroll
        for (int u = 0; u < UNR; ++u) raw[u] = ld_v4(my_wire + (v + u * AR_THREADS) * 16);
#pragma unroll
        for (int u = 0; u < UNR; ++u) {
          const float2 f0 = unpack_bf16x2(raw[u].x), f1 = unpack_bf16x2(raw[u].y), f2 = unpack_bf16x2(raw[u].z),
                       f3 = unpack_bf16x2(raw[u].w);
          float* o = out + (v + u * AR_THREADS) * 8;
          *reinterpret_cast<float4*>(o) = make_float4(f0.x, f0.y, f1.x, f1.y);
          *reinterpret_cast<float4*>(o + 4) = make_float4(f2.x, f2.y, f3.x, f3.y);
        }
      }
    }
    for (; v < chunk1; v += AR_THREADS) {
      const uint4 raw = ld_v4(my_wire + v * 16);
      if constexpr (WIRE32) {
        *reinterpret_cast<uint4*>(out + v * 4) = raw;
      } else {
        const float2 f0 = unpack_bf16x2(raw.x), f1 = unpack_bf16x2(raw.y), f2 = unpack_bf16x2(raw.z),
                     f3 = unpack_bf16x2(raw.w);
        *reinterpret_cast<float4*>(out + v * 8) = make_float4(f0.x, f0.y, f1.x, f1.y);
        *reinterpret_cast<float4*>(out + v * 8 + 4) = make_float4(f2.x, f2.y, f3.x, f3.y);
      }
    }
  }
}

// CTAs of a launch: at least ~2 vectors per thread per cell, otherwise fewer (latency-bound small
// buckets).  Exposed so that the host can reproduce which rank owns which cell (zero1_step).
int allreduce_grid(long long n, int world, int max_ctas, bool wire_fp32) {
  const long long nvec = n / (wire_fp32 ? 4 : 8);
  int G = max_ctas <= 0 ? 48 : max_ctas;
  if (G > AR_MAX_CTAS) G = AR_MAX_CTAS;
  const long long want = nvec / (static_cast<long long>(AR_THREADS) * world) + 1;
  if (want < G) G = static_cast<int>(want);
  return G < 1 ? 1 : G;
}

void allreduce_fused(const CommCtx& ctx, const float* grad_f32, float* grad_out_f32, long long start,
                     long long n, float inv_world, int algo, bool wire_fp32, int slot, uint32_t epoch,
                     int max_ctas, cudaStream_t s) {
  if (ctx.world > AR_MAX_WORLD) throw std::runtime_error("[b200] allreduce_fused: world too large");
  if (n % 8 || start % 8) throw std::runtime_error("[b200] allreduce_fused: range must be 8-element aligned");
  if (algo == AR_ONESHOT && !grad_out_f32)
    throw std::runtime_error("[b200] allreduce_fused: one-shot needs an fp32 output");
  if (algo == AR_NVLS && !ctx.wire_mc)
    throw std::runtime_error("[b200] allreduce_fused: NVLS requested but no multicast mapping");
  ArArgs a;
  a.c = ctx; a.grad = grad_f32; a.grad_out = grad_out_f32; a.start = start; a.n = n;
  a.inv_world = inv_world; a.slot = slot; a.epoch = epoch;
  const int G = allreduce_grid(n, ctx.world, max_ctas, wire_fp32);
  static const bool carve = [] {
    prefer_max_shared_carveout(reinterpret_cast<const void*>(allreduce_kernel<AR_ONESHOT, false>));
    prefer_max_shared_carveout(reinterpret_cast<const void*>(allreduce_kernel<AR_ONESHOT, true>));
    prefer_max_shared_carveout(reinterpret_cast<const void*>(allreduce_kernel<AR_TWOSHOT, false>));
    prefer_max_shared_carveout(reinterpret_cast<const void*>(allreduce_kernel<AR_TWOSHOT, true>));
    prefer_max_shared_carveout(reinterpret_cast<const void*>(allreduce_kernel<AR_NVLS, false>));
    prefer_max_shared_carveout(reinterpret_cast<const void*>(allreduce_kernel<AR_NVLS, true>));
    return true;
  }();
  (void)carve;
#define AR_LAUNCH(ALGO)                                                           \
  if (wire_fp32) allreduce_kernel<ALGO, true><<<G, AR_THREADS, 0, s>>>(a);        \
  else allreduce_kernel<ALGO, false><<<G, AR_THREADS, 0, s>>>(a);
  switch (algo) {
    case AR_ONESHOT: AR_LAUNCH(AR_ONESHOT) break;
    case AR_TWOSHOT: AR_LAUNCH(AR_TWOSHOT) break;
    case AR_NVLS: AR_LAUNCH(AR_NVLS) break;
    default: throw std::runtime_error("[b200] allreduce_fused: unknown algorithm");
  }
#undef AR_LAUNCH
  count_launch();
  check_last("allreduce_fused");
}

// ------------------------------------------------------------ fused reduce-scatter + Adam + all-gather
// EXPERIMENTAL (--zero1).  The two-shot variant has run on one H100 80GB HBM3 with emulated ranks
// (tests/test_collectives_gpu.py, world 1 .. 16): owned cells, Adam state, wires and shadows bit for
// bit, nothing written outside its range.  The handshake between real peers and the NVLS variant run
// only in test_multigpu.py, on a host with several GPUs.
//
// ZeRO-1 in ONE kernel per bucket, over peer memory: the compute step (the optimizer) sits between
// the two halves of the collective instead of after it.
//
//   pack      wire = bf16(grad * 1/ws), fp32 gradient range re-zeroed            (as allreduce_kernel)
//   barrier
//   per cell  rank r owns cell (b, r):  g = sum over ranks of the cell (NVLS multimem.ld_reduce, or
//             peer loads), Adam on ITS fp32 master / moments only, new weight -> bf16 ->
//             multimem.st (or peer stores) into every rank's wire at the same offset
//   barrier
//   copy      wire -> local bf16 weight shadow (every rank, whole chunk)
//
// Versus all-reduce + replicated Adam: the optimizer's 24 B/parameter of HBM traffic shrink by the
// world size (by a factor of ws), the wire carries new weights instead
// of averaged gradients (same bytes), and every replica ends with bit-identical bf16 weights by
// construction.  The fp32 master and moments of a cell live on its owner only (gathered for
// checkpoints by NativeEngine.prepare_export).  The reduced gradient is rounded to bf16 once, exactly
// like the wire of allreduce_kernel, and both paths apply adam_update (adam.cuh), so they produce the
// same update bit for bit.
struct Zero1Args {
  CommCtx c;
  float* grad;             // local fp32 arena (nullptr: wire already holds the packed data)
  float* p; float* m; float* v;
  bf16* shadow;
  float* ema;              // moving average of the weights (zero1_kernel<..., true, ...>)
  long long start, n;
  float inv_world;
  int slot;
  uint32_t epoch;
  OptStep o;               // Adam or AdamW, one decay (o.wd.value[0]) for the whole range
};

template <bool EMA, bool DECOUPLED>
__device__ __forceinline__ uint4 zero1_adam8(const Zero1Args& a, long long elem, const uint4& gred) {
  const uint32_t gw[4] = {gred.x, gred.y, gred.z, gred.w};
  float g[8];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 f = unpack_bf16x2(gw[i]);
    g[2 * i] = f.x; g[2 * i + 1] = f.y;
  }
  float pp[8], mm[8], vv[8];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const float4 p4 = __ldcs(reinterpret_cast<const float4*>(a.p + elem + 4 * h));   // streaming: see adam_kernel
    const float4 m4 = __ldcs(reinterpret_cast<const float4*>(a.m + elem + 4 * h));
    const float4 v4 = __ldcs(reinterpret_cast<const float4*>(a.v + elem + 4 * h));
    pp[4 * h] = p4.x; pp[4 * h + 1] = p4.y; pp[4 * h + 2] = p4.z; pp[4 * h + 3] = p4.w;
    mm[4 * h] = m4.x; mm[4 * h + 1] = m4.y; mm[4 * h + 2] = m4.z; mm[4 * h + 3] = m4.w;
    vv[4 * h] = v4.x; vv[4 * h + 1] = v4.y; vv[4 * h + 2] = v4.z; vv[4 * h + 3] = v4.w;
  }
#pragma unroll
  for (int k = 0; k < 8; ++k)            // the update of adam_kernel at grad_scale 1, bit for bit
    optimizer_update<DECOUPLED ? OPT_ADAMW : OPT_ADAM>(a.o, g[k], 1.f, a.o.wd.value[0], pp[k], mm[k], vv[k]);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    __stcs(reinterpret_cast<float4*>(a.p + elem + 4 * h), make_float4(pp[4 * h], pp[4 * h + 1], pp[4 * h + 2], pp[4 * h + 3]));
    __stcs(reinterpret_cast<float4*>(a.m + elem + 4 * h), make_float4(mm[4 * h], mm[4 * h + 1], mm[4 * h + 2], mm[4 * h + 3]));
    __stcs(reinterpret_cast<float4*>(a.v + elem + 4 * h), make_float4(vv[4 * h], vv[4 * h + 1], vv[4 * h + 2], vv[4 * h + 3]));
    // one half at a time: 4 more live floats next to the Adam state
    if constexpr (EMA) ema_update4(a.ema + elem + 4 * h, pp + 4 * h, a.o.ema);
  }
  return make_uint4(pack_bf16x2(pp[0], pp[1]), pack_bf16x2(pp[2], pp[3]), pack_bf16x2(pp[4], pp[5]),
                    pack_bf16x2(pp[6], pp[7]));
}

// 128 threads x <= 80 registers (the Adam state of 8 parameters lives in registers between the
// reduce and the broadcast) = 10 240 registers: the same footprint as allreduce_kernel, so these CTAs
// also co-reside with every conv kernel of backward.  EMA: the owner also updates the moving average of
// its cells (non-owned cells of `ema` are not touched; prepare_ema gathers them like prepare_export).
// DECOUPLED: AdamW.  ZeRO-1 buckets hold one FC weight each, so one decay covers the whole range.
constexpr int Z1_THREADS = 128;
constexpr int Z1_MIN_BLOCKS = 6;
template <int ALGO, bool EMA, bool DECOUPLED>
__global__ void __launch_bounds__(Z1_THREADS, Z1_MIN_BLOCKS) zero1_kernel(const Zero1Args a) {
  static_assert(ALGO == AR_TWOSHOT || ALGO == AR_NVLS, "the owner-computes step needs a reduce-scatter");
  const CommCtx& c = a.c;
  const int b = blockIdx.x, G = gridDim.x, world = c.world, rank = c.rank;
  const long long nvec = a.n / 8;
  const long long cell = (nvec + static_cast<long long>(G) * world - 1) / (static_cast<long long>(G) * world);
  const long long chunk0 = min(nvec, static_cast<long long>(b) * world * cell);
  const long long chunk1 = min(nvec, static_cast<long long>(b + 1) * world * cell);
  uint8_t* my_wire = reinterpret_cast<uint8_t*>(c.wire_ptrs[rank]) + a.start * 2;

  if (a.grad) {                         // pack + re-zero the fp32 gradient range for the next step
    float* g = a.grad + a.start;
    const float s = a.inv_world;
    for (long long v = chunk0 + threadIdx.x; v < chunk1; v += Z1_THREADS) {
      const float4 x0 = *reinterpret_cast<const float4*>(g + v * 8);
      const float4 x1 = *reinterpret_cast<const float4*>(g + v * 8 + 4);
      *reinterpret_cast<float4*>(g + v * 8) = make_float4(0.f, 0.f, 0.f, 0.f);
      *reinterpret_cast<float4*>(g + v * 8 + 4) = make_float4(0.f, 0.f, 0.f, 0.f);
      st_v4(my_wire + v * 16, make_uint4(pack_bf16x2(x0.x * s, x0.y * s), pack_bf16x2(x0.z * s, x0.w * s),
                                         pack_bf16x2(x1.x * s, x1.y * s), pack_bf16x2(x1.z * s, x1.w * s)));
    }
  }
  cta_barrier_all_ranks(c, a.slot, 0, b, a.epoch);

  const long long cell0 = min(chunk1, chunk0 + static_cast<long long>(rank) * cell);
  const long long cell1 = min(chunk1, cell0 + cell);
  if constexpr (ALGO == AR_NVLS) {
    uint8_t* mc = reinterpret_cast<uint8_t*>(c.wire_mc) + a.start * 2;
    // software pipeline: the switch reduction of the NEXT vector is in flight while this one's Adam
    // state (96 bytes of p, m, v) is loaded, updated and stored
    long long v = cell0 + threadIdx.x;
    uint4 gnext = make_uint4(0, 0, 0, 0);
    if (v < cell1) gnext = multimem_ld_reduce_bf16x8(mc + v * 16);       // switch adds, fp32 accumulate
    for (; v < cell1; v += Z1_THREADS) {
      const uint4 gred = gnext;
      if (v + Z1_THREADS < cell1) gnext = multimem_ld_reduce_bf16x8(mc + (v + Z1_THREADS) * 16);
      multimem_st_v4(mc + v * 16, zero1_adam8<EMA, DECOUPLED>(a, a.start + v * 8, gred));
    }
  } else {
    for (long long v = cell0 + threadIdx.x; v < cell1; v += Z1_THREADS) {
      const long long boff = a.start * 2 + v * 16;
      float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      for (int p = 0; p < world; ++p) {
        const int peer = (rank + p) % world;
        accum_bf16x8(acc, ld_v4(reinterpret_cast<const uint8_t*>(c.wire_ptrs[peer]) + boff));
      }
      const uint4 gred = make_uint4(pack_bf16x2(acc[0], acc[1]), pack_bf16x2(acc[2], acc[3]),
                                    pack_bf16x2(acc[4], acc[5]), pack_bf16x2(acc[6], acc[7]));
      const uint4 w8 = zero1_adam8<EMA, DECOUPLED>(a, a.start + v * 8, gred);
      for (int p = 0; p < world; ++p) {
        const int peer = (rank + p) % world;
        st_v4(reinterpret_cast<uint8_t*>(c.wire_ptrs[peer]) + boff, w8);
      }
    }
  }
  cta_barrier_all_ranks(c, a.slot, 1, b, a.epoch);

  bf16* sh = a.shadow + a.start;        // every rank: new weights of the whole chunk -> local shadow
  for (long long v = chunk0 + threadIdx.x; v < chunk1; v += Z1_THREADS)
    __stcs(reinterpret_cast<uint4*>(sh + v * 8), ld_v4(my_wire + v * 16));
}

void zero1_step(const CommCtx& ctx, const OptStep& o, float* grad_f32, float* p, float* m, float* v, bf16* shadow,
                float* ema, long long start, long long n, float inv_world, int algo, int slot, uint32_t epoch,
                int max_ctas, cudaStream_t s) {
  if (ctx.world > AR_MAX_WORLD) throw std::runtime_error("[b200] zero1_step: world too large");
  if (n % 8 || start % 8) throw std::runtime_error("[b200] zero1_step: range must be 8-element aligned");
  if (algo == AR_NVLS && !ctx.wire_mc) throw std::runtime_error("[b200] zero1_step: NVLS needs a multicast mapping");
  if (algo != AR_NVLS && algo != AR_TWOSHOT) throw std::runtime_error("[b200] zero1_step: two-shot or NVLS only");
  if (o.kind == OPT_SGD || o.wd.n != 1 || o.grad_scale != 1.f)
    throw std::runtime_error("[b200] zero1_step: Adam or AdamW with one weight decay and grad_scale 1 only");
  Zero1Args a;
  a.c = ctx; a.grad = grad_f32; a.p = p; a.m = m; a.v = v; a.shadow = shadow; a.ema = ema; a.start = start; a.n = n;
  a.inv_world = inv_world; a.slot = slot; a.epoch = epoch; a.o = o;
  const int G = allreduce_grid(n, ctx.world, max_ctas, false);
  using Kernel = void (*)(const Zero1Args);
  static const Kernel kernels[2][2][2] = {   // [NVLS][EMA][DECOUPLED]
      {{zero1_kernel<AR_TWOSHOT, false, false>, zero1_kernel<AR_TWOSHOT, false, true>},
       {zero1_kernel<AR_TWOSHOT, true, false>, zero1_kernel<AR_TWOSHOT, true, true>}},
      {{zero1_kernel<AR_NVLS, false, false>, zero1_kernel<AR_NVLS, false, true>},
       {zero1_kernel<AR_NVLS, true, false>, zero1_kernel<AR_NVLS, true, true>}}};
  static const bool carve = [] {
    for (const auto& by_ema : kernels)
      for (const auto& by_kind : by_ema)
        for (Kernel k : by_kind) prefer_max_shared_carveout(reinterpret_cast<const void*>(k));
    return true;
  }();
  (void)carve;
  kernels[algo == AR_NVLS][ema != nullptr][o.kind == OPT_ADAMW]<<<G, Z1_THREADS, 0, s>>>(a);
  count_launch();
  check_last("zero1_step");
}

// ------------------------------------------------------------------------------------ broadcast
// K-BCAST (DDP's constructor sync, distributedVggf.py:225): root stages fp32 data in its wire
// buffer, everybody pulls it over NVLink.  Called on chunks that fit the wire buffer.
__global__ void __launch_bounds__(AR_THREADS, 1)
broadcast_kernel(const CommCtx c, float* data, long long n, int root, int slot, uint32_t epoch) {
  const int b = blockIdx.x, G = gridDim.x;
  const long long nvec = n / 4;
  const long long per = (nvec + G - 1) / G;
  const long long v0 = min(nvec, b * per), v1 = min(nvec, v0 + per);
  uint8_t* root_wire = reinterpret_cast<uint8_t*>(c.wire_ptrs[root]);
  if (c.rank == root)
    for (long long v = v0 + threadIdx.x; v < v1; v += AR_THREADS)
      st_v4(root_wire + v * 16, *reinterpret_cast<const uint4*>(data + v * 4));
  cta_barrier_all_ranks(c, slot, 0, b, epoch);
  if (c.rank != root)
    for (long long v = v0 + threadIdx.x; v < v1; v += AR_THREADS)
      *reinterpret_cast<uint4*>(data + v * 4) = ld_v4(root_wire + v * 16);
  cta_barrier_all_ranks(c, slot, 1, b, epoch);
}

void broadcast_fused(const CommCtx& ctx, float* data_f32, long long n, int root, int slot,
                     uint32_t epoch, cudaStream_t s) {
  if (n % 4) throw std::runtime_error("[b200] broadcast_fused: n must be a multiple of 4");
  broadcast_kernel<<<32, AR_THREADS, 0, s>>>(ctx, data_f32, n, root, slot, epoch);
  count_launch();
  check_last("broadcast_fused");
}

__global__ void barrier_kernel(const CommCtx c, int slot, uint32_t epoch) {
  cta_barrier_all_ranks(c, slot, 0, 0, epoch);
}
void device_barrier(const CommCtx& ctx, int slot, uint32_t epoch, cudaStream_t s) {
  barrier_kernel<<<1, 32, 0, s>>>(ctx, slot, epoch);
  count_launch();
  check_last("device_barrier");
}

int allreduce_signal_words(int slots) { return slots * AR_SLOT_WORDS; }

}  // namespace b200
