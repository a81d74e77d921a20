// norm.cu — K5: GroupNorm(32) statistics / apply(+SiLU) over NHWC bf16 and LayerNorm over token rows.
// HBM-bound glue: 128-bit loads, fp32 statistics, warp-shuffle / shared-memory reductions, deterministic
// (no floating-point atomics to global memory: per-chunk partials are summed in a fixed order).
// Replaces diffusers GroupNorm / LayerNorm call sites inside ResnetBlock2D, Transformer2DModel and
// BasicTransformerBlock (reached from mixofshow/pipelines/pipeline_edlora.py:277).
#include <stdlib.h>

#include <type_traits>

#include "common.h"
#include "tc.cuh"

namespace mos {

constexpr int GN_GROUPS = 32;

// GroupNorm statistics are centred.  Raw sums of x and x^2 lose the variance to cancellation once the group's mean is large
// against its spread (E[x^2] - mean^2 in fp32), and sums about any one element p lose it once that element lies far from
// the group's mean (the error grows with ((p - mean) / std)^2; the top-left pixel, where the zero padding of 3x3
// convolutions leaves its mark, can lie up to sqrt(n) std away).  So:
//  - the cluster kernel sums x - p and (x - p)^2 about p, the group's first element in the sample's first row (which keeps
//    constant groups exact).  When p lies more than 4 std from the mean, it sums x - m and (x - m)^2 about that mean m
//    in a second pass over the slab it holds in shared memory;
//  - the statistics kernel of the fallback and the backward keeps a running (mean, M2) per thread and channel (Welford)
//    and writes one (mean, M2) per (chunk, group); gn_merge_chunks merges the chunks about the first chunk's mean and
//    adds their centred terms.
// Every merge runs in a fixed order, so the statistics are bitwise reproducible.

template <bool F16>
__device__ __forceinline__ float gn_pivot(const __nv_bfloat16* x, long long ldx, int b, int HW, int c0) {
  return ld16<F16>(x + (long long)b * HW * ldx + c0);
}

// partial[b][chunk][g][2] = (mean, M2 = sum of (x - mean)^2) over rows [chunk*rows_per_chunk, ...) of batch b
template <bool F16>
__global__ void gn_stats_kernel(const __nv_bfloat16* __restrict__ x, long long ldx, int HW, int C,
                                int rows_per_chunk, float* __restrict__ partial) {
  extern __shared__ float red[];  // [blockDim][16]: per-thread channel means / M2
  pdl_wait();
  pdl_launch_dependents();
  const int oct = C / 8, cpg = C / GN_GROUPS;
  const int b = blockIdx.y, chunk = blockIdx.x, nchunks = gridDim.x;
  const int lanes = blockDim.x / oct;  // row lanes; blockDim is a multiple of oct
  const int o = threadIdx.x % oct, rl = threadIdx.x / oct;
  const int r0 = chunk * rows_per_chunk, r1 = min(HW, r0 + rows_per_chunk);
  float m[8], m2[8];   // Welford: running mean and sum of squared deviations of the thread's rows, per channel
  int cnt = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) m[i] = m2[i] = 0.f;
  const __nv_bfloat16* base = x + ((long long)b * HW) * ldx + o * 8;
  for (int rb = r0 + rl; rb < r1; rb += 4 * lanes) {
    uint4 u4[4];   // four independent 16-byte loads in flight per thread
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int r = rb + k * lanes;
      u4[k] = r < r1 ? __ldg(reinterpret_cast<const uint4*>(base + (long long)r * ldx)) : make_uint4(0, 0, 0, 0);
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (rb + k * lanes >= r1) continue;
      const float inv = __frcp_rn((float)(++cnt));
      const uint32_t w[4] = {u4[k].x, u4[k].y, u4[k].z, u4[k].w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 f = unpack16x2<F16>(w[i]);
        const float d0 = f.x - m[2 * i], d1 = f.y - m[2 * i + 1];
        m[2 * i] = fmaf(d0, inv, m[2 * i]);
        m[2 * i + 1] = fmaf(d1, inv, m[2 * i + 1]);
        m2[2 * i] = fmaf(d0, f.x - m[2 * i], m2[2 * i]);
        m2[2 * i + 1] = fmaf(d1, f.y - m[2 * i + 1], m2[2 * i + 1]);
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    red[threadIdx.x * 16 + i] = m[i];
    red[threadIdx.x * 16 + 8 + i] = m2[i];
  }
  __syncthreads();
  if (threadIdx.x < GN_GROUPS) {  // fixed order -> bitwise reproducible statistics
    // Row lane l holds the (mean, M2) of rows r0 + l + j * lanes: q0 or q0 + 1 of them.  The group's mean is the first
    // partial's mean plus the weighted mean of the differences to it; M2 = sum of (M2 + rows * (mean_l,c - mean)^2).
    const int g = threadIdx.x, rows = r1 - r0, q0 = rows / lanes, rem = rows - q0 * lanes;
    const float m0 = red[((g * cpg) >> 3) * 16 + ((g * cpg) & 7)];   // lane 0 holds at least one row
    float s = 0.f;
    for (int c = g * cpg; c < (g + 1) * cpg; ++c) {
      for (int l = 0; l < lanes; ++l) s = fmaf((float)(q0 + (l < rem)), red[(l * oct + (c >> 3)) * 16 + (c & 7)] - m0, s);
    }
    const float mu = m0 + s / ((float)rows * (float)cpg);
    float q = 0.f;
    for (int c = g * cpg; c < (g + 1) * cpg; ++c) {
      for (int l = 0; l < lanes; ++l) {
        const float* t = red + (l * oct + (c >> 3)) * 16 + (c & 7);
        const float d = t[0] - mu;
        q += fmaf((float)(q0 + (l < rem)) * d, d, t[8]);
      }
    }
    float* dst = partial + (((long long)b * nchunks + chunk) * GN_GROUPS + g) * 2;
    dst[0] = mu;
    dst[1] = q;
  }
}

// mean / rstd of the (sample, group) pairs of batch b from the per-chunk (mean, M2) of gn_stats_kernel, on threads
// [0, 128): 4 threads per group over strided chunks, then a shuffle tree (fixed order).  The mean is the first chunk's
// mean plus the row-weighted mean of the differences to it, which keeps a constant group exact; the variance adds each
// chunk's M2 and its centred term rows * cpg * (mean_c - mean)^2.
__device__ __forceinline__ void gn_merge_chunks(const float* __restrict__ partial, int nchunks, int rows_per_chunk,
                                                int b, int HW, int cpg, float eps, float* mean, float* rstd) {
  if (threadIdx.x < GN_GROUPS * 4) {
    const int g = threadIdx.x >> 2, sub = threadIdx.x & 3;
    const float2* pg = reinterpret_cast<const float2*>(partial) + (long long)b * nchunks * GN_GROUPS + g;
    const float m0 = __ldg(pg).x;
    float s = 0.f;
    for (int c = sub; c < nchunks; c += 4) {
      const float rows = (float)(min(HW, (c + 1) * rows_per_chunk) - c * rows_per_chunk);
      s = fmaf(rows, __ldg(pg + (long long)c * GN_GROUPS).x - m0, s);
    }
#pragma unroll
    for (int d = 2; d > 0; d >>= 1) s += __shfl_xor_sync(0xffffffffu, s, d);
    const float mu = m0 + s / (float)HW;
    float q = 0.f;
    for (int c = sub; c < nchunks; c += 4) {
      const float n = (float)(min(HW, (c + 1) * rows_per_chunk) - c * rows_per_chunk) * (float)cpg;
      const float2 v = __ldg(pg + (long long)c * GN_GROUPS);
      const float d = v.x - mu;
      q += fmaf(n * d, d, v.y);
    }
#pragma unroll
    for (int d = 2; d > 0; d >>= 1) q += __shfl_xor_sync(0xffffffffu, q, d);
    if (sub == 0) {
      mean[g] = mu;
      rstd[g] = rsqrtf(fmaxf(q / ((float)HW * (float)cpg), 0.f) + eps);
    }
  }
}

template <bool F16>
__global__ void gn_apply_kernel(const __nv_bfloat16* __restrict__ x, long long ldx, int HW, int C,
                                const float* __restrict__ partial, int nchunks, const float* __restrict__ gamma,
                                const float* __restrict__ beta, float eps, int silu_act, int rows_per_block,
                                __nv_bfloat16* __restrict__ y, long long ldy) {
  __shared__ float mean[GN_GROUPS], rstd[GN_GROUPS];
  pdl_wait();
  pdl_launch_dependents();
  const int b = blockIdx.y;
  const int cpg = C / GN_GROUPS;
  gn_merge_chunks(partial, nchunks, rows_per_block, b, HW, cpg, eps, mean, rstd);   // blockDim >= 160 always
  __syncthreads();
  const int oct = C / 8;
  const int lanes = blockDim.x / oct;
  const int o = threadIdx.x % oct, rl = threadIdx.x / oct;
  if (rl >= lanes) return;
  // y = (x - mean) * (gamma * rstd) + beta: folding the mean into the shift would cancel when |mean| * rstd is large
  float sc[8], mu[8], sh[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    int c = o * 8 + i, g = c / cpg;
    sc[i] = __ldg(gamma + c) * rstd[g];
    mu[i] = mean[g];
    sh[i] = __ldg(beta + c);
  }
  const int r0 = blockIdx.x * rows_per_block, r1 = min(HW, r0 + rows_per_block);
  const __nv_bfloat16* xb = x + ((long long)b * HW) * ldx + o * 8;
  __nv_bfloat16* yb = y + ((long long)b * HW) * ldy + o * 8;
  for (int rb = r0 + rl; rb < r1; rb += 4 * lanes) {
    uint4 u4[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int r = rb + k * lanes;
      if (r < r1) u4[k] = __ldg(reinterpret_cast<const uint4*>(xb + (long long)r * ldx));
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int r = rb + k * lanes;
      if (r < r1) {
        const uint32_t w[4] = {u4[k].x, u4[k].y, u4[k].z, u4[k].w};
        float v[8];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          float2 f = unpack16x2<F16>(w[i]);
          v[2 * i] = (f.x - mu[2 * i]) * sc[2 * i] + sh[2 * i];
          v[2 * i + 1] = (f.y - mu[2 * i + 1]) * sc[2 * i + 1] + sh[2 * i + 1];
        }
        if (silu_act) {
#pragma unroll
          for (int i = 0; i < 8; ++i) v[i] = silu(v[i]);
        }
        uint4 out;
        out.x = pack16x2<F16>(v[0], v[1]);
        out.y = pack16x2<F16>(v[2], v[3]);
        out.z = pack16x2<F16>(v[4], v[5]);
        out.w = pack16x2<F16>(v[6], v[7]);
        *reinterpret_cast<uint4*>(yb + (long long)r * ldy) = out;
      }
    }
  }
}

// One warp per row; C <= 1280 (5 octets per lane), two-pass statistics in registers.
template <bool F16>
__global__ void layernorm_kernel(const __nv_bfloat16* __restrict__ x, long long ldx, long long M, int C,
                                 const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                 __nv_bfloat16* __restrict__ y, long long ldy) {
  pdl_wait();
  pdl_launch_dependents();
  const long long row = (long long)blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= M) return;
  const int oct = C / 8;
  float v[5][8];
  float s = 0.f;
  const __nv_bfloat16* xr = x + row * ldx;
#pragma unroll
  for (int k = 0; k < 5; ++k) {
    int o = lane + k * 32;
    if (o < oct) {
      uint4 u = __ldg(reinterpret_cast<const uint4*>(xr + o * 8));
      uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        float2 f = unpack16x2<F16>(w[i]);
        v[k][2 * i] = f.x;
        v[k][2 * i + 1] = f.y;
        s += f.x + f.y;
      }
    }
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) s += __shfl_xor_sync(0xffffffffu, s, d);
  const float mean = s / (float)C;
  float q = 0.f;
#pragma unroll
  for (int k = 0; k < 5; ++k) {
    int o = lane + k * 32;
    if (o < oct) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float d = v[k][i] - mean;
        q += d * d;
      }
    }
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) q += __shfl_xor_sync(0xffffffffu, q, d);
  const float rstd = rsqrtf(q / (float)C + eps);
  __nv_bfloat16* yr = y + row * ldy;
#pragma unroll
  for (int k = 0; k < 5; ++k) {
    int o = lane + k * 32;
    if (o < oct) {
      float r[8];
      float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + o * 8));
      float4 g1 = __ldg(reinterpret_cast<const float4*>(gamma + o * 8 + 4));
      float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + o * 8));
      float4 b1 = __ldg(reinterpret_cast<const float4*>(beta + o * 8 + 4));
      float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
      float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i) r[i] = (v[k][i] - mean) * rstd * gg[i] + bb[i];
      uint4 out;
      out.x = pack16x2<F16>(r[0], r[1]);
      out.y = pack16x2<F16>(r[2], r[3]);
      out.z = pack16x2<F16>(r[4], r[5]);
      out.w = pack16x2<F16>(r[6], r[7]);
      *reinterpret_cast<uint4*>(yr + o * 8) = out;
    }
  }
}

// ---------------------------------------------------------------------------------------------- one-pass GroupNorm
// GroupNorm(+SiLU) in ONE launch with ONE read of x: a thread-block cluster of k CTAs (k = 1, 2, 4, 8) owns one
// (sample, group) pair.  Each CTA streams its rows of the group's channel slab (cpg = C / 32 channels, 20..160 bytes
// per row) into shared memory while accumulating sum / sum of squares about the pivot, the k partial pairs are exchanged
// through distributed shared memory (gn_cluster_sum: fixed order -> bitwise reproducible and identical in all CTAs), an
// outlying pivot triggers a second, centred pass over the slab (exchanged the same way), and the slab is normalised out
// of shared memory.  Replaces gn_stats + gn_apply (two launches, two reads of x, a partial-statistics round trip through
// global memory); those remain as the fallback for slabs that do not fit 8 x 200 KB.
// Thread layout: thread = (row lane, VEC-element column word); blockDim = lanes * (cpg / VEC), so the column word - and
// with it gamma / beta - is fixed per thread and no index division happens inside the loops; every thread re-reads only
// the shared-memory words it wrote itself.
__device__ __forceinline__ uint32_t mapa_u32(uint32_t saddr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(saddr), "r"(rank));
  return r;
}
__device__ __forceinline__ void st_cluster_f32x2(uint32_t raddr, float a, float b) {
  asm volatile("st.shared::cluster.v2.f32 [%0], {%1, %2};" ::"r"(raddr), "f"(a), "f"(b) : "memory");
}

// (s, q) summed over the CTA's threads, then over the cluster's k CTAs in rank order through `table` (every CTA stores its
// pair into every peer's table, one cluster barrier): the same bits in every thread of every CTA.  Called by all threads.
// A table serves one call only, since a peer may still be reading it when this CTA reaches the next call.
__device__ __forceinline__ float2 gn_cluster_sum(float s, float q, float (*wred)[2], float2* table, int k, int rank,
                                                 bool wait_peers) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, d);
    q += __shfl_xor_sync(0xffffffffu, q, d);
  }
  const int warp = threadIdx.x >> 5, nwarps = (blockDim.x + 31) >> 5;
  if ((threadIdx.x & 31) == 0) {
    wred[warp][0] = s;
    wred[warp][1] = q;
  }
  __syncthreads();
  if (wait_peers && k > 1) asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");   // all peers have started
  if (threadIdx.x == 0) {
    float ts = 0.f, tq = 0.f;
    for (int w = 0; w < nwarps; ++w) {
      ts += wred[w][0];
      tq += wred[w][1];
    }
    if (k > 1) {
      const uint32_t slot = smem_u32(&table[rank]);
      for (int peer = 0; peer < k; ++peer) st_cluster_f32x2(mapa_u32(slot, (uint32_t)peer), ts, tq);
    } else {
      table[0] = make_float2(ts, tq);
    }
  }
  if (k > 1) cluster_sync_all();     // release / acquire at cluster scope: the peers' table stores are visible
  else __syncthreads();
  float2 t = make_float2(0.f, 0.f);
  for (int i = 0; i < k; ++i) {
    t.x += table[i].x;
    t.y += table[i].y;
  }
  return t;
}

template <bool F16, int VEC>   // VEC = 16-bit elements per load / store: 4 (cpg % 4 == 0) or 2
__global__ void __launch_bounds__(256)
gn_group_kernel(const __nv_bfloat16* __restrict__ x, long long ldx, int HW, int C, int rows_per_cta, int k, int lanes,
                const float* __restrict__ gamma, const float* __restrict__ beta, float eps, int silu_act,
                __nv_bfloat16* __restrict__ y, long long ldy) {
  extern __shared__ __align__(16) uint8_t gsm[];
  __shared__ float wred[8][2];
  __shared__ float2 table[2][8];    // per-CTA partials of the two passes, filled by the peers through DSMEM
  // Distributed shared memory may only be touched once every CTA of the cluster is known to be running: arrive here, wait
  // right before the first remote store (the loads and the local reduction in between hide the barrier latency).
  if (k > 1) asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  pdl_wait();
  pdl_launch_dependents();
  const int cpg = C / GN_GROUPS;
  const int vpr = cpg / VEC;                       // column words per row
  // `lanes` row lanes (lanes * vpr <= blockDim.x; blockDim is rounded up to whole warps, the surplus threads only take
  // part in the shuffles)
  const int rank = k > 1 ? (int)cluster_ctarank() : 0;
  const int bg = blockIdx.x / k;                   // (sample, group)
  const int b = bg / GN_GROUPS, g = bg - b * GN_GROUPS;
  const int v = threadIdx.x % vpr, rl = threadIdx.x / vpr;
  const int r0 = rank * rows_per_cta, r1 = min(HW, r0 + rows_per_cta);
  using word_t = typename std::conditional<VEC == 4, uint2, uint32_t>::type;
  word_t* slab = reinterpret_cast<word_t*>(gsm);
  const __nv_bfloat16* xb = x + ((long long)b * HW) * ldx + g * cpg + v * VEC;
  const float p = gn_pivot<F16>(x, ldx, b, HW, g * cpg);   // sums of x - p and (x - p)^2, see gn_pivot
  float s = 0.f, q = 0.f;
  if (rl < lanes) {
    for (int r = r0 + rl; r < r1; r += 4 * lanes) {
      word_t w[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int rr = r + j * lanes;
        if (rr < r1) w[j] = __ldg(reinterpret_cast<const word_t*>(xb + (long long)rr * ldx));
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int rr = r + j * lanes;
        if (rr < r1) {
          slab[(rr - r0) * vpr + v] = w[j];
          if constexpr (VEC == 4) {
            const float2 f0 = unpack16x2<F16>(w[j].x), f1 = unpack16x2<F16>(w[j].y);
            const float d0 = f0.x - p, d1 = f0.y - p, d2 = f1.x - p, d3 = f1.y - p;
            s += (d0 + d1) + (d2 + d3);
            q += (d0 * d0 + d1 * d1) + (d2 * d2 + d3 * d3);
          } else {
            const float2 f0 = unpack16x2<F16>(w[j]);
            const float d0 = f0.x - p, d1 = f0.y - p;
            s += d0 + d1;
            q += d0 * d0 + d1 * d1;
          }
        }
      }
    }
  }
  const float n = (float)HW * (float)cpg;
  float2 t = gn_cluster_sum(s, q, wred, table[0], k, rank, true);
  float d = t.x / n;    // mean - pivot
  float mean = p + d, var = t.y / n - d * d;
  // The cancellation error of var grows with ((p - mean) / std)^2.  Beyond 4 std (an outlying pivot element) sum again,
  // about the mean, over the slab words this thread stored.  Every CTA of the cluster holds the same t: the branch and
  // the second exchange are uniform across the cluster.
  if (d * d > 16.f * var) {
    float s2 = 0.f, q2 = 0.f;
    if (rl < lanes) {
      for (int r = r0 + rl; r < r1; r += lanes) {
        const word_t w = slab[(r - r0) * vpr + v];
        if constexpr (VEC == 4) {
          const float2 f0 = unpack16x2<F16>(w.x), f1 = unpack16x2<F16>(w.y);
          const float d0 = f0.x - mean, d1 = f0.y - mean, d2 = f1.x - mean, d3 = f1.y - mean;
          s2 += (d0 + d1) + (d2 + d3);
          q2 += (d0 * d0 + d1 * d1) + (d2 * d2 + d3 * d3);
        } else {
          const float2 f0 = unpack16x2<F16>(w);
          const float d0 = f0.x - mean, d1 = f0.y - mean;
          s2 += d0 + d1;
          q2 += d0 * d0 + d1 * d1;
        }
      }
    }
    t = gn_cluster_sum(s2, q2, wred, table[1], k, rank, false);
    d = t.x / n;
    mean += d;
    var = t.y / n - d * d;
  }
  const float rstd = rsqrtf(fmaxf(var, 0.f) + eps);
  if (rl >= lanes) return;
  float sc[VEC], sh[VEC];   // y = (x - mean) * sc + sh, as in gn_apply_kernel
#pragma unroll
  for (int i = 0; i < VEC; ++i) {
    const int c = g * cpg + v * VEC + i;
    sc[i] = __ldg(gamma + c) * rstd;
    sh[i] = __ldg(beta + c);
  }
  __nv_bfloat16* yb = y + ((long long)b * HW) * ldy + g * cpg + v * VEC;
  for (int r = r0 + rl; r < r1; r += lanes) {
    const word_t w = slab[(r - r0) * vpr + v];
    float o[VEC];
    if constexpr (VEC == 4) {
      const float2 f0 = unpack16x2<F16>(w.x), f1 = unpack16x2<F16>(w.y);
      o[0] = (f0.x - mean) * sc[0] + sh[0];
      o[1] = (f0.y - mean) * sc[1] + sh[1];
      o[2] = (f1.x - mean) * sc[2] + sh[2];
      o[3] = (f1.y - mean) * sc[3] + sh[3];
    } else {
      const float2 f0 = unpack16x2<F16>(w);
      o[0] = (f0.x - mean) * sc[0] + sh[0];
      o[1] = (f0.y - mean) * sc[1] + sh[1];
    }
    if (silu_act) {
#pragma unroll
      for (int i = 0; i < VEC; ++i) o[i] = silu(o[i]);
    }
    word_t out;
    if constexpr (VEC == 4) {
      out.x = pack16x2<F16>(o[0], o[1]);
      out.y = pack16x2<F16>(o[2], o[3]);
    } else {
      out = pack16x2<F16>(o[0], o[1]);
    }
    *reinterpret_cast<word_t*>(yb + (long long)r * ldy) = out;
  }
}


// ---------------------------------------------------------------------------------------------- backward (training)
// GroupNorm(+SiLU) backward for the ED-LoRA training step (trainer_edlora.py:237 reached through loss.backward()):
// gamma / beta are frozen, so only dx is produced.   z = xhat*gamma + beta, y = act(z), dz = dy * act'(z),
//   dx = rstd * (dz*gamma - mean_g(dz*gamma) - xhat * mean_g(dz*gamma*xhat))        (means over the group's HW*cpg)
__device__ __forceinline__ float silu_grad(float z) {
  const float sg = 1.0f / (1.0f + __expf(-z));
  return sg * (1.0f + z * (1.0f - sg));
}

// partial2[b][chunk][g][2] = (sum dz*gamma, sum dz*gamma*xhat)
__global__ void gn_bwd_reduce_kernel(const __nv_bfloat16* __restrict__ x, long long ldx,
                                     const __nv_bfloat16* __restrict__ dy, long long lddy, int HW, int C,
                                     const float* __restrict__ partial, const float* __restrict__ gamma,
                                     const float* __restrict__ beta, float eps, int silu_act, int rows_per_chunk,
                                     float* __restrict__ partial2) {
  extern __shared__ float red[];  // [blockDim][16]
  __shared__ float mean[GN_GROUPS], rstd[GN_GROUPS];
  pdl_wait();
  pdl_launch_dependents();
  const int b = blockIdx.y, chunk = blockIdx.x, nchunks = gridDim.x;
  const int cpg = C / GN_GROUPS;
  gn_merge_chunks(partial, nchunks, rows_per_chunk, b, HW, cpg, eps, mean, rstd);   // of gn_stats_kernel<false>
  __syncthreads();
  const int oct = C / 8;
  const int lanes = blockDim.x / oct;
  const int o = threadIdx.x % oct, rl = threadIdx.x / oct;
  float ga[8], be[8], mu[8], rs[8], a[8], bb[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int c = o * 8 + i, g = c / cpg;
    ga[i] = __ldg(gamma + c);
    be[i] = __ldg(beta + c);
    mu[i] = mean[g];
    rs[i] = rstd[g];
    a[i] = bb[i] = 0.f;
  }
  const int r0 = chunk * rows_per_chunk, r1 = min(HW, r0 + rows_per_chunk);
  const __nv_bfloat16* xb = x + ((long long)b * HW) * ldx + o * 8;
  const __nv_bfloat16* db = dy + ((long long)b * HW) * lddy + o * 8;
  for (int r = r0 + rl; r < r1; r += lanes) {
    const uint4 ux = __ldg(reinterpret_cast<const uint4*>(xb + (long long)r * ldx));
    const uint4 ud = __ldg(reinterpret_cast<const uint4*>(db + (long long)r * lddy));
    const uint32_t wx[4] = {ux.x, ux.y, ux.z, ux.w}, wd[4] = {ud.x, ud.y, ud.z, ud.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 fx = unpack_bf16x2(wx[i]), fd = unpack_bf16x2(wd[i]);
      const float xv[2] = {fx.x, fx.y}, dv[2] = {fd.x, fd.y};
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int k = 2 * i + h;
        const float xh = (xv[h] - mu[k]) * rs[k];
        float dz = dv[h];
        if (silu_act) dz *= silu_grad(xh * ga[k] + be[k]);
        const float t = dz * ga[k];
        a[k] += t;
        bb[k] += t * xh;
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    red[threadIdx.x * 16 + i] = a[i];
    red[threadIdx.x * 16 + 8 + i] = bb[i];
  }
  __syncthreads();
  if (threadIdx.x < GN_GROUPS) {  // fixed summation order
    const int g = threadIdx.x;
    float gs = 0.f, gq = 0.f;
    for (int c = g * cpg; c < (g + 1) * cpg; ++c) {
      for (int l = 0; l < lanes; ++l) {
        const float* t = red + (l * oct + (c >> 3)) * 16 + (c & 7);
        gs += t[0];
        gq += t[8];
      }
    }
    float* dst = partial2 + (((long long)b * nchunks + chunk) * GN_GROUPS + g) * 2;
    dst[0] = gs;
    dst[1] = gq;
  }
}

__global__ void gn_bwd_apply_kernel(const __nv_bfloat16* __restrict__ x, long long ldx,
                                    const __nv_bfloat16* __restrict__ dy, long long lddy, int HW, int C,
                                    const float* __restrict__ partial, const float* __restrict__ partial2,
                                    const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                    int silu_act, int rows_per_chunk, const __nv_bfloat16* __restrict__ add,
                                    long long ldadd, __nv_bfloat16* __restrict__ dx, long long lddx) {
  __shared__ float mean[GN_GROUPS], rstd[GN_GROUPS], ma[GN_GROUPS], mb[GN_GROUPS];
  pdl_wait();
  pdl_launch_dependents();
  const int b = blockIdx.y, nchunks = gridDim.x;
  const int cpg = C / GN_GROUPS;
  gn_merge_chunks(partial, nchunks, rows_per_chunk, b, HW, cpg, eps, mean, rstd);   // of gn_stats_kernel<false>
  if (threadIdx.x < GN_GROUPS * 4) {
    const int g = threadIdx.x >> 2, sub = threadIdx.x & 3;
    float s = 0.f, q = 0.f;
    for (int c = sub; c < nchunks; c += 4) {
      const float2 v = __ldg(reinterpret_cast<const float2*>(partial2 + (((long long)b * nchunks + c) * GN_GROUPS + g) * 2));
      s += v.x;
      q += v.y;
    }
#pragma unroll
    for (int d = 2; d > 0; d >>= 1) {
      s += __shfl_xor_sync(0xffffffffu, s, d);
      q += __shfl_xor_sync(0xffffffffu, q, d);
    }
    if (sub == 0) {
      const float n = (float)HW * (float)cpg;
      ma[g] = s / n;
      mb[g] = q / n;
    }
  }
  __syncthreads();
  const int oct = C / 8;
  const int lanes = blockDim.x / oct;
  const int o = threadIdx.x % oct, rl = threadIdx.x / oct;
  float ga[8], be[8], mu[8], rs[8], A[8], Bm[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int c = o * 8 + i, g = c / cpg;
    ga[i] = __ldg(gamma + c);
    be[i] = __ldg(beta + c);
    mu[i] = mean[g];
    rs[i] = rstd[g];
    A[i] = ma[g];
    Bm[i] = mb[g];
  }
  const int r0 = blockIdx.x * rows_per_chunk, r1 = min(HW, r0 + rows_per_chunk);
  const __nv_bfloat16* xb = x + ((long long)b * HW) * ldx + o * 8;
  const __nv_bfloat16* db = dy + ((long long)b * HW) * lddy + o * 8;
  const __nv_bfloat16* ab = add ? add + ((long long)b * HW) * ldadd + o * 8 : nullptr;
  __nv_bfloat16* ob = dx + ((long long)b * HW) * lddx + o * 8;
  for (int r = r0 + rl; r < r1; r += lanes) {
    const uint4 ux = __ldg(reinterpret_cast<const uint4*>(xb + (long long)r * ldx));
    const uint4 ud = __ldg(reinterpret_cast<const uint4*>(db + (long long)r * lddy));
    uint4 ua = make_uint4(0, 0, 0, 0);
    if (ab) ua = __ldg(reinterpret_cast<const uint4*>(ab + (long long)r * ldadd));
    const uint32_t wx[4] = {ux.x, ux.y, ux.z, ux.w}, wd[4] = {ud.x, ud.y, ud.z, ud.w}, wa[4] = {ua.x, ua.y, ua.z, ua.w};
    float v[8];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 fx = unpack_bf16x2(wx[i]), fd = unpack_bf16x2(wd[i]), fa = unpack_bf16x2(wa[i]);
      const float xv[2] = {fx.x, fx.y}, dv[2] = {fd.x, fd.y}, av[2] = {fa.x, fa.y};
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int k = 2 * i + h;
        const float xh = (xv[h] - mu[k]) * rs[k];
        float dz = dv[h];
        if (silu_act) dz *= silu_grad(xh * ga[k] + be[k]);
        v[k] = rs[k] * (dz * ga[k] - A[k] - xh * Bm[k]) + av[h];
      }
    }
    uint4 out;
    out.x = pack_bf16x2(v[0], v[1]);
    out.y = pack_bf16x2(v[2], v[3]);
    out.z = pack_bf16x2(v[4], v[5]);
    out.w = pack_bf16x2(v[6], v[7]);
    *reinterpret_cast<uint4*>(ob + (long long)r * lddx) = out;
  }
}

// LayerNorm backward, one warp per row (C <= 1280); statistics recomputed from x in registers.
__global__ void layernorm_bwd_kernel(const __nv_bfloat16* __restrict__ x, long long ldx,
                                     const __nv_bfloat16* __restrict__ dy, long long lddy, long long M, int C,
                                     const float* __restrict__ gamma, float eps, const __nv_bfloat16* __restrict__ add,
                                     long long ldadd, __nv_bfloat16* __restrict__ dx, long long lddx) {
  pdl_wait();
  pdl_launch_dependents();
  const long long row = (long long)blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= M) return;
  const int oct = C / 8;
  float v[5][8], g[5][8];
  float s = 0.f;
  const __nv_bfloat16* xr = x + row * ldx;
  const __nv_bfloat16* dr = dy + row * lddy;
#pragma unroll
  for (int k = 0; k < 5; ++k) {
    const int o = lane + k * 32;
    if (o < oct) {
      const uint4 u = __ldg(reinterpret_cast<const uint4*>(xr + o * 8));
      const uint4 d = __ldg(reinterpret_cast<const uint4*>(dr + o * 8));
      const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + o * 8));
      const float4 g1 = __ldg(reinterpret_cast<const float4*>(gamma + o * 8 + 4));
      const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
      const uint32_t w[4] = {u.x, u.y, u.z, u.w}, wd[4] = {d.x, d.y, d.z, d.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 f = unpack_bf16x2(w[i]), fd = unpack_bf16x2(wd[i]);
        v[k][2 * i] = f.x;
        v[k][2 * i + 1] = f.y;
        g[k][2 * i] = fd.x * gg[2 * i];
        g[k][2 * i + 1] = fd.y * gg[2 * i + 1];
        s += f.x + f.y;
      }
    }
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) s += __shfl_xor_sync(0xffffffffu, s, d);
  const float mean = s / (float)C;
  float q = 0.f;
#pragma unroll
  for (int k = 0; k < 5; ++k) {
    if (lane + k * 32 < oct) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float d = v[k][i] - mean;
        q += d * d;
      }
    }
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) q += __shfl_xor_sync(0xffffffffu, q, d);
  const float rstd = rsqrtf(q / (float)C + eps);
  float sa = 0.f, sb = 0.f;
#pragma unroll
  for (int k = 0; k < 5; ++k) {
    if (lane + k * 32 < oct) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        v[k][i] = (v[k][i] - mean) * rstd;   // xhat
        sa += g[k][i];
        sb += g[k][i] * v[k][i];
      }
    }
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    sa += __shfl_xor_sync(0xffffffffu, sa, d);
    sb += __shfl_xor_sync(0xffffffffu, sb, d);
  }
  sa /= (float)C;
  sb /= (float)C;
  __nv_bfloat16* outr = dx + row * lddx;
  const __nv_bfloat16* ar = add ? add + row * ldadd : nullptr;
#pragma unroll
  for (int k = 0; k < 5; ++k) {
    const int o = lane + k * 32;
    if (o < oct) {
      float a8[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      if (ar) {
        const uint4 ua = __ldg(reinterpret_cast<const uint4*>(ar + o * 8));
        const uint32_t wa[4] = {ua.x, ua.y, ua.z, ua.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 f = unpack_bf16x2(wa[i]);
          a8[2 * i] = f.x;
          a8[2 * i + 1] = f.y;
        }
      }
      float r[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) r[i] = rstd * (g[k][i] - sa - v[k][i] * sb) + a8[i];
      uint4 out;
      out.x = pack_bf16x2(r[0], r[1]);
      out.y = pack_bf16x2(r[2], r[3]);
      out.z = pack_bf16x2(r[4], r[5]);
      out.w = pack_bf16x2(r[6], r[7]);
      *reinterpret_cast<uint4*>(outr + o * 8) = out;
    }
  }
}

static int gn_block_threads(int C) {
  int oct = C / 8;
  int k = 320 / oct;
  if (k < 1) k = 1;
  return oct * k;
}

}  // namespace mos

using namespace mos;

static int g_gn_two_pass = -1;     // -1: read MOS_GN_TWOPASS on first use
extern "C" int mos_debug_set_gn_twopass(int32_t on) {   // A/B switch for tools/gn_debug.py
  g_gn_two_pass = on ? 1 : 0;
  return MOS_OK;
}

// GroupNorm(32) + optional SiLU:  y[b, r, c] = act((x - mean_bg) * rstd_bg * gamma_c + beta_c)
// x: bf16 [B, HW, ldx] (first C channels), y: bf16 [B, HW, ldy]; partial: fp32 workspace [B, nchunks, 32, 2] of the
// fallback, nchunks chosen to fit partial_capacity_floats (at least B * 64).
extern "C" int mos_groupnorm_fwd(const void* x, int64_t ldx, int32_t B, int32_t HW, int32_t C, const float* gamma,
                                 const float* beta, float eps, int32_t silu_act, float* partial,
                                 int32_t partial_capacity_floats, void* y, int64_t ldy, int32_t act_dtype,
                                 void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  MOS_CHECK_ARG(x && y && gamma && beta && partial, "mos_groupnorm_fwd: NULL pointer");
  MOS_CHECK_DTYPE(act_dtype, "mos_groupnorm_fwd");
  const bool f16 = act_dtype == MOS_DT_F16;
  MOS_CHECK_ARG(C % 32 == 0 && C % 8 == 0 && C <= 2560 && ldx % 8 == 0 && ldy % 8 == 0 && ldx >= C && ldy >= C,
                "mos_groupnorm_fwd: bad C=%d ldx=%lld ldy=%lld", C, (long long)ldx, (long long)ldy);
  const int threads = gn_block_threads(C);
  // ---- one-pass path: a cluster of k CTAs per (sample, group) keeps the group's channel slab in shared memory
  if (g_gn_two_pass < 0) {
    const char* e = getenv("MOS_GN_TWOPASS");
    g_gn_two_pass = (e && e[0] == '1') ? 1 : 0;
  }
  if (!g_gn_two_pass) {
    const int cpg = C / GN_GROUPS;
    const int vec = (cpg % 4 == 0 && ldx % 4 == 0 && ldy % 4 == 0) ? 4 : 2;
    const long long slab = (long long)HW * cpg * 2;
    int k = 1;
    static int min_ctas = 0;
    if (min_ctas == 0) {
      int dev = 0, sms = 0;
      MOS_CHECK_CUDA(cudaGetDevice(&dev));
      MOS_CHECK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
      const char* e = getenv("MOS_GN_MIN_CTAS");      // clusters are widened until the grid has at least this many CTAs
      min_ctas = e ? atoi(e) : 2 * sms;              // two CTAs per SM
      if (min_ctas < 1) min_ctas = 2 * sms;
    }
    while (k < 8 && HW / (2 * k) >= 16 && (slab / k > 48 * 1024 || (long long)B * GN_GROUPS * k < min_ctas)) k *= 2;
    const int rows_per_cta = (int)ceil_div(HW, k);
    const size_t smem = (size_t)rows_per_cta * cpg * 2;
    if (smem <= 200 * 1024 && cpg % 2 == 0 && ldx % 2 == 0 && ldy % 2 == 0) {
      const int vpr = cpg / vec;
      const int lanes = 256 / vpr;
      const int threads = ((lanes * vpr + 31) / 32) * 32;
      static bool configured = false;
      if (!configured) {
        MOS_CHECK_CUDA(cudaFuncSetAttribute(gn_group_kernel<false, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        MOS_CHECK_CUDA(cudaFuncSetAttribute(gn_group_kernel<false, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        MOS_CHECK_CUDA(cudaFuncSetAttribute(gn_group_kernel<true, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        MOS_CHECK_CUDA(cudaFuncSetAttribute(gn_group_kernel<true, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        configured = true;
      }
      cudaLaunchConfig_t cfg;
      memset(&cfg, 0, sizeof(cfg));
      cfg.gridDim = dim3((unsigned)(B * GN_GROUPS * k));
      cfg.blockDim = dim3((unsigned)threads);
      cfg.dynamicSmemBytes = smem;
      cfg.stream = stream;
      cudaLaunchAttribute attr[2];
      attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
      attr[0].val.programmaticStreamSerializationAllowed = 1;
      attr[1].id = cudaLaunchAttributeClusterDimension;
      attr[1].val.clusterDim.x = (unsigned)k;
      attr[1].val.clusterDim.y = 1;
      attr[1].val.clusterDim.z = 1;
      cfg.attrs = attr;
      cfg.numAttrs = k > 1 ? 2 : 1;
      const __nv_bfloat16* xp = reinterpret_cast<const __nv_bfloat16*>(x);
      __nv_bfloat16* yp = reinterpret_cast<__nv_bfloat16*>(y);
      auto kern = f16 ? (vec == 4 ? gn_group_kernel<true, 4> : gn_group_kernel<true, 2>)
                      : (vec == 4 ? gn_group_kernel<false, 4> : gn_group_kernel<false, 2>);
      MOS_CHECK_CUDA(cudaLaunchKernelEx(&cfg, kern, xp, (long long)ldx, (int)HW, (int)C, rows_per_cta, k, lanes, gamma, beta, eps,
                                        (int)silu_act, yp, (long long)ldy));
      return MOS_OK;
    }
  }
  // ---- two-launch fallback (very large maps)
  // aim for ~4 blocks per SM overall
  int nchunks = (int)ceil_div(2368, B);     // up to ~16 blocks per SM in flight: latency-bound kernels want parallelism
  int min_rows = 4 * (threads / (C / 8));
  if (nchunks > (int)ceil_div(HW, min_rows)) nchunks = (int)ceil_div(HW, min_rows);
  {
    const long long cap = (long long)partial_capacity_floats / ((long long)B * GN_GROUPS * 2);
    if (nchunks > cap) nchunks = (int)cap;
  }
  if (nchunks < 1) nchunks = 1;
  int rows_per_chunk = (int)ceil_div(HW, nchunks);
  nchunks = (int)ceil_div(HW, rows_per_chunk);
  MOS_CHECK_ARG((long long)B * nchunks * GN_GROUPS * 2 <= partial_capacity_floats,
                "mos_groupnorm_fwd: partial workspace too small (need %lld floats)",
                (long long)B * nchunks * GN_GROUPS * 2);
  MOS_CHECK_CUDA(launch_pdl(f16 ? gn_stats_kernel<true> : gn_stats_kernel<false>, dim3(nchunks, B), dim3(threads),
                            threads * 16 * sizeof(float), stream, reinterpret_cast<const __nv_bfloat16*>(x), (long long)ldx,
                            (int)HW, (int)C, rows_per_chunk, partial));
  MOS_CHECK_CUDA(launch_pdl(f16 ? gn_apply_kernel<true> : gn_apply_kernel<false>, dim3(nchunks, B), dim3(threads), 0, stream,
                            reinterpret_cast<const __nv_bfloat16*>(x), (long long)ldx, (int)HW, (int)C,
                            (const float*)partial, nchunks, gamma, beta, eps, (int)silu_act, rows_per_chunk,
                            reinterpret_cast<__nv_bfloat16*>(y), (long long)ldy));
  return MOS_OK;
}

extern "C" int mos_layernorm_fwd(const void* x, int64_t ldx, int64_t M, int32_t C, const float* gamma,
                                 const float* beta, float eps, void* y, int64_t ldy, int32_t act_dtype, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  MOS_CHECK_ARG(x && y && gamma && beta, "mos_layernorm_fwd: NULL pointer");
  MOS_CHECK_DTYPE(act_dtype, "mos_layernorm_fwd");
  MOS_CHECK_ARG(C % 8 == 0 && C <= 1280 && ldx % 8 == 0 && ldy % 8 == 0, "mos_layernorm_fwd: bad C=%d", C);
  const int warps = 8;
  MOS_CHECK_CUDA(launch_pdl(act_dtype == MOS_DT_F16 ? layernorm_kernel<true> : layernorm_kernel<false>,
                            dim3((unsigned)ceil_div(M, warps)), dim3(warps * 32), 0, stream,
                            reinterpret_cast<const __nv_bfloat16*>(x), (long long)ldx, (long long)M, (int)C, gamma, beta,
                            eps, reinterpret_cast<__nv_bfloat16*>(y), (long long)ldy));
  return MOS_OK;
}


// GroupNorm(+SiLU) backward (frozen affine):  dx = d/dx [ act(GN(x)) ] . dy  (+ add).  Statistics are recomputed from x.
// workspace: fp32, >= 2 * B * nchunks * 64 floats (the entry point picks nchunks to fit `workspace_floats`).
extern "C" int mos_groupnorm_bwd(const void* x, int64_t ldx, const void* dy, int64_t lddy, int32_t B, int32_t HW,
                                 int32_t C, const float* gamma, const float* beta, float eps, int32_t silu_act,
                                 float* workspace, int32_t workspace_floats, const void* add, int64_t ldadd, void* dx,
                                 int64_t lddx, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  MOS_CHECK_ARG(x && dy && dx && gamma && beta && workspace, "mos_groupnorm_bwd: NULL pointer");
  MOS_CHECK_ARG(C % 32 == 0 && C <= 2560 && ldx % 8 == 0 && lddy % 8 == 0 && lddx % 8 == 0 && ldx >= C && lddy >= C &&
                    lddx >= C && (!add || (ldadd % 8 == 0 && ldadd >= C)),
                "mos_groupnorm_bwd: bad C=%d / pitches", C);
  const int threads = gn_block_threads(C);
  int nchunks = (int)ceil_div(1184, B);
  const int min_rows = 4 * (threads / (C / 8));
  if (nchunks > (int)ceil_div(HW, min_rows)) nchunks = (int)ceil_div(HW, min_rows);
  {
    const long long cap = (long long)workspace_floats / ((long long)B * GN_GROUPS * 4);
    if (nchunks > cap) nchunks = (int)cap;
  }
  MOS_CHECK_ARG(nchunks >= 1, "mos_groupnorm_bwd: workspace too small (need >= %d floats)", B * GN_GROUPS * 4);
  const int rows_per_chunk = (int)ceil_div(HW, nchunks);
  nchunks = (int)ceil_div(HW, rows_per_chunk);
  float* p1 = workspace;
  float* p2 = workspace + (long long)B * nchunks * GN_GROUPS * 2;
  const __nv_bfloat16* xb = reinterpret_cast<const __nv_bfloat16*>(x);
  const __nv_bfloat16* db = reinterpret_cast<const __nv_bfloat16*>(dy);
  MOS_CHECK_CUDA(launch_pdl(gn_stats_kernel<false>, dim3(nchunks, B), dim3(threads), threads * 16 * sizeof(float), stream, xb,
                            (long long)ldx, (int)HW, (int)C, rows_per_chunk, p1));
  MOS_CHECK_CUDA(launch_pdl(gn_bwd_reduce_kernel, dim3(nchunks, B), dim3(threads), threads * 16 * sizeof(float), stream,
                            xb, (long long)ldx, db, (long long)lddy, (int)HW, (int)C, (const float*)p1, gamma, beta, eps,
                            (int)silu_act, rows_per_chunk, p2));
  MOS_CHECK_CUDA(launch_pdl(gn_bwd_apply_kernel, dim3(nchunks, B), dim3(threads), 0, stream, xb, (long long)ldx, db,
                            (long long)lddy, (int)HW, (int)C, (const float*)p1, (const float*)p2, gamma, beta, eps,
                            (int)silu_act, rows_per_chunk, reinterpret_cast<const __nv_bfloat16*>(add), (long long)ldadd,
                            reinterpret_cast<__nv_bfloat16*>(dx), (long long)lddx));
  return MOS_OK;
}

// LayerNorm backward (frozen affine): dx = d/dx LN(x) . dy (+ add); one warp per row.
extern "C" int mos_layernorm_bwd(const void* x, int64_t ldx, const void* dy, int64_t lddy, int64_t M, int32_t C,
                                 const float* gamma, float eps, const void* add, int64_t ldadd, void* dx, int64_t lddx,
                                 void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  MOS_CHECK_ARG(x && dy && dx && gamma, "mos_layernorm_bwd: NULL pointer");
  MOS_CHECK_ARG(C % 8 == 0 && C <= 1280 && ldx % 8 == 0 && lddy % 8 == 0 && lddx % 8 == 0 && (!add || ldadd % 8 == 0),
                "mos_layernorm_bwd: bad C=%d / pitches", C);
  const int warps = 8;
  MOS_CHECK_CUDA(launch_pdl(layernorm_bwd_kernel, dim3((unsigned)ceil_div(M, warps)), dim3(warps * 32), 0, stream,
                            reinterpret_cast<const __nv_bfloat16*>(x), (long long)ldx,
                            reinterpret_cast<const __nv_bfloat16*>(dy), (long long)lddy, (long long)M, (int)C, gamma, eps,
                            reinterpret_cast<const __nv_bfloat16*>(add), (long long)ldadd,
                            reinterpret_cast<__nv_bfloat16*>(dx), (long long)lddx));
  return MOS_OK;
}
