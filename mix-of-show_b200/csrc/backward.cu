// backward.cu — HBM-bound kernels of the ED-LoRA training step (EDLoRATrainer.forward, trainer_edlora.py:202-261, and the
// loss.backward() that follows it at train_edlora.py:120-123).  All base weights are frozen: only activation gradients
// and the rank-4 LoRA gradients exist.
//   geglu fwd / bwd (un-fused form: the pre-activation is kept for backward)
//   upsample2x bwd, stride-2 col2im (Downsample2D bwd), conv_out bwd
//   masked MSE loss + gradient (trainer_edlora.py:251-252), add_noise (DDPMScheduler.add_noise)
//   head-split transpose, attention delta (rowsum(dO * O)), LoRA gradients (dU, dD)
#include "common.h"
#include "tc.cuh"

namespace mos {

#define STREAM(s) reinterpret_cast<cudaStream_t>(s)
static inline unsigned nblk(long long total, int threads) { return (unsigned)((total + threads - 1) / threads); }

__device__ __forceinline__ void unpack8(const uint4& u, float* v) {
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 f = unpack_bf16x2(w[i]);
    v[2 * i] = f.x;
    v[2 * i + 1] = f.y;
  }
}
__device__ __forceinline__ uint4 pack8(const float* v) {
  uint4 u;
  u.x = pack_bf16x2(v[0], v[1]);
  u.y = pack_bf16x2(v[2], v[3]);
  u.z = pack_bf16x2(v[4], v[5]);
  u.w = pack_bf16x2(v[6], v[7]);
  return u;
}

// ------------------------------------------------------------------------------------------------ GEGLU
// z [M, 2H] in 160-column tiles [80 a | 80 gate] (the weight-row interleave of the fused GEMM), y [M, H]
__global__ void geglu_fwd_kernel(const __nv_bfloat16* __restrict__ z, long long ldz, long long M, int H,
                                 __nv_bfloat16* __restrict__ y, long long ldy) {
  pdl_wait();
  pdl_launch_dependents();
  const int oct = H / 8;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= M * oct) return;
  const int o = (int)(idx % oct);
  const long long m = idx / oct;
  const int tile = (o * 8) / 80, j = (o * 8) % 80;
  const __nv_bfloat16* zr = z + m * ldz + tile * 160 + j;
  float a[8], g[8], r[8];
  unpack8(__ldg(reinterpret_cast<const uint4*>(zr)), a);
  unpack8(__ldg(reinterpret_cast<const uint4*>(zr + 80)), g);
#pragma unroll
  for (int i = 0; i < 8; ++i) r[i] = a[i] * gelu_erf(g[i]);
  *reinterpret_cast<uint4*>(y + m * ldy + o * 8) = pack8(r);
}

__global__ void geglu_bwd_kernel(const __nv_bfloat16* __restrict__ z, long long ldz,
                                 const __nv_bfloat16* __restrict__ dy, long long lddy, long long M, int H,
                                 __nv_bfloat16* __restrict__ dz, long long lddz) {
  pdl_wait();
  pdl_launch_dependents();
  const int oct = H / 8;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= M * oct) return;
  const int o = (int)(idx % oct);
  const long long m = idx / oct;
  const int tile = (o * 8) / 80, j = (o * 8) % 80;
  const __nv_bfloat16* zr = z + m * ldz + tile * 160 + j;
  float a[8], g[8], d[8], da[8], dg[8];
  unpack8(__ldg(reinterpret_cast<const uint4*>(zr)), a);
  unpack8(__ldg(reinterpret_cast<const uint4*>(zr + 80)), g);
  unpack8(__ldg(reinterpret_cast<const uint4*>(dy + m * lddy + o * 8)), d);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float cdf = 0.5f * (1.0f + erff(g[i] * 0.70710678118654752f));
    const float pdf = 0.3989422804014327f * __expf(-0.5f * g[i] * g[i]);
    da[i] = d[i] * g[i] * cdf;
    dg[i] = d[i] * a[i] * (cdf + g[i] * pdf);
  }
  __nv_bfloat16* dr = dz + m * lddz + tile * 160 + j;
  *reinterpret_cast<uint4*>(dr) = pack8(da);
  *reinterpret_cast<uint4*>(dr + 80) = pack8(dg);
}

// ------------------------------------------------------------------------------------------------ resampling
// dx[b, h, w, :] = sum of the 2x2 block of dy  (backward of nearest x2)
__global__ void upsample2x_bwd_kernel(const __nv_bfloat16* __restrict__ dy, long long lddy, int B, int H, int W, int C,
                                      __nv_bfloat16* __restrict__ dx, long long lddx) {
  pdl_wait();
  pdl_launch_dependents();
  const int oct = C / 8;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)B * H * W * oct) return;
  const int o = (int)(idx % oct);
  const long long pix = idx / oct;
  const int w = (int)(pix % W), h = (int)((pix / W) % H), b = (int)(pix / ((long long)W * H));
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const long long src = ((long long)b * 2 * H + 2 * h + (t >> 1)) * 2 * W + 2 * w + (t & 1);
    float v[8];
    unpack8(__ldg(reinterpret_cast<const uint4*>(dy + src * lddy + o * 8)), v);
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] += v[i];
  }
  *reinterpret_cast<uint4*>(dx + pix * lddx + o * 8) = pack8(acc);
}

// dx[b, y, x, c] = sum over taps (kh, kw) with (y+1-kh, x+1-kw) even and in range of dcol[(b, oy, ox), tap*C + c]
__global__ void col2im_s2_kernel(const __nv_bfloat16* __restrict__ dcol, int B, int H, int W, int C,
                                 const __nv_bfloat16* __restrict__ add, long long ldadd,
                                 __nv_bfloat16* __restrict__ dx, long long lddx) {
  pdl_wait();
  pdl_launch_dependents();
  const int oct = C / 8, Ho = H / 2, Wo = W / 2;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)B * H * W * oct) return;
  const int o = (int)(idx % oct);
  const long long pix = idx / oct;
  const int x = (int)(pix % W), y = (int)((pix / W) % H), b = (int)(pix / ((long long)W * H));
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (add) unpack8(__ldg(reinterpret_cast<const uint4*>(add + pix * ldadd + o * 8)), acc);
  for (int kh = 0; kh < 3; ++kh) {
    const int ty = y + 1 - kh;
    if (ty < 0 || (ty & 1) || (ty >> 1) >= Ho) continue;
    for (int kw = 0; kw < 3; ++kw) {
      const int tx = x + 1 - kw;
      if (tx < 0 || (tx & 1) || (tx >> 1) >= Wo) continue;
      const long long op = ((long long)b * Ho + (ty >> 1)) * Wo + (tx >> 1);
      float v[8];
      unpack8(__ldg(reinterpret_cast<const uint4*>(dcol + op * 9 * C + (long long)(kh * 3 + kw) * C + o * 8)), v);
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] += v[i];
    }
  }
  *reinterpret_cast<uint4*>(dx + pix * lddx + o * 8) = pack8(acc);
}

// conv_out backward: dy fp32 NCHW [B, Cout<=4, H, W], w fp32 [Cout][9][C] -> dx bf16 [B*H*W, C]
__global__ void conv_out_bwd_kernel(const float* __restrict__ dy, int B, int H, int W, int C,
                                    const float* __restrict__ w, int Cout, __nv_bfloat16* __restrict__ dx) {
  pdl_wait();
  pdl_launch_dependents();
  const int oct = C / 8;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)B * H * W * oct) return;
  const int o = (int)(idx % oct);
  const long long pix = idx / oct;
  const int wq = (int)(pix % W), hq = (int)((pix / W) % H), b = (int)(pix / ((long long)W * H));
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int tap = 0; tap < 9; ++tap) {
    const int hh = hq - (tap / 3 - 1), ww = wq - (tap % 3 - 1);   // output pixel that read this input through `tap`
    if (hh < 0 || hh >= H || ww < 0 || ww >= W) continue;
    for (int oc = 0; oc < Cout; ++oc) {
      const float g = __ldg(dy + (((long long)b * Cout + oc) * H + hh) * W + ww);
      const float* wp = w + ((long long)oc * 9 + tap) * C + o * 8;
      const float4 w0 = __ldg(reinterpret_cast<const float4*>(wp));
      const float4 w1 = __ldg(reinterpret_cast<const float4*>(wp + 4));
      acc[0] += g * w0.x; acc[1] += g * w0.y; acc[2] += g * w0.z; acc[3] += g * w0.w;
      acc[4] += g * w1.x; acc[5] += g * w1.y; acc[6] += g * w1.z; acc[7] += g * w1.w;
    }
  }
  *reinterpret_cast<uint4*>(dx + pix * C + o * 8) = pack8(acc);
}

// ------------------------------------------------------------------------------------------------ loss
// per-sample sums: ws[b] = (sum_{c,h,w} (pred - target)^2 * mask[b, hw], sum_{hw} mask[b, hw])
__global__ void mse_sums_kernel(const float* __restrict__ pred, const float* __restrict__ target,
                                const float* __restrict__ mask, int Cc, int HW, float* __restrict__ ws) {
  __shared__ float sn[32], sd[32];
  pdl_wait();
  pdl_launch_dependents();
  const int b = blockIdx.x;
  float num = 0.f, den = 0.f;
  for (int i = threadIdx.x; i < HW; i += blockDim.x) {
    const float m = mask[(long long)b * HW + i];
    den += m;
    for (int c = 0; c < Cc; ++c) {
      const long long k = ((long long)b * Cc + c) * HW + i;
      const float d = pred[k] - target[k];
      num += d * d * m;
    }
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    num += __shfl_xor_sync(0xffffffffu, num, d);
    den += __shfl_xor_sync(0xffffffffu, den, d);
  }
  if ((threadIdx.x & 31) == 0) {
    sn[threadIdx.x >> 5] = num;
    sd[threadIdx.x >> 5] = den;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = 0.f, c = 0.f;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) {
      a += sn[i];
      c += sd[i];
    }
    ws[2 * b] = a;
    ws[2 * b + 1] = c;
  }
}

// dpred = grad_scale * 2 (pred - target) mask / (den_b * B);  loss[0] = mean_b num_b / den_b
__global__ void mse_grad_kernel(const float* __restrict__ pred, const float* __restrict__ target,
                                const float* __restrict__ mask, int B, int Cc, int HW, const float* __restrict__ ws,
                                float grad_scale, float* __restrict__ dpred, float* __restrict__ loss) {
  pdl_wait();
  pdl_launch_dependents();
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx == 0) {
    float l = 0.f;
    for (int b = 0; b < B; ++b) l += ws[2 * b] / ws[2 * b + 1];
    loss[0] = l / (float)B;
  }
  if (idx >= (long long)B * Cc * HW) return;
  const int i = (int)(idx % HW);
  const int b = (int)(idx / ((long long)Cc * HW));
  const float m = mask[(long long)b * HW + i];
  dpred[idx] = grad_scale * 2.0f * (pred[idx] - target[idx]) * m / (ws[2 * b + 1] * (float)B);
}

// noisy = sqrt(ac[t_b]) x0 + sqrt(1 - ac[t_b]) noise
__global__ void add_noise_kernel(const float* __restrict__ x0, const float* __restrict__ noise,
                                 const int* __restrict__ t, const float* __restrict__ alphas_cumprod, long long per,
                                 long long total, float* __restrict__ out) {
  pdl_wait();
  pdl_launch_dependents();
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const float ac = alphas_cumprod[t[idx / per]];
  out[idx] = sqrtf(ac) * x0[idx] + sqrtf(1.0f - ac) * noise[idx];
}

// ------------------------------------------------------------------------------------------------ attention glue
// dst[bh, j, r] = src[bh, r, j]   src [BH, R, DP] -> dst [BH, DV, R8] (r >= R left untouched: buffers are zero-initialised)
__global__ void heads_transpose_kernel(const __nv_bfloat16* __restrict__ src, int R, int DP, int DV, int R8,
                                       __nv_bfloat16* __restrict__ dst) {
  __shared__ __nv_bfloat16 tile[32][34];
  pdl_wait();
  pdl_launch_dependents();
  const int bh = blockIdx.z;
  const int r0 = blockIdx.x * 32, j0 = blockIdx.y * 32;
  const __nv_bfloat16* s = src + (long long)bh * R * DP;
  __nv_bfloat16* d = dst + (long long)bh * DV * R8;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int r = r0 + i, j = j0 + threadIdx.x;
    tile[i][threadIdx.x] = (r < R && j < DP) ? s[(long long)r * DP + j] : __float2bfloat16(0.f);
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int j = j0 + i, r = r0 + threadIdx.x;
    if (j < DV && r < R) d[(long long)j * R8 + r] = tile[threadIdx.x][i];
  }
}

// delta[bh, q] = sum_j dO[bh, q, j] * O[b*N + q, h*d + j]  (+ sum_c pcols[bh, q, c] * gcols[b, q, c] for the attn-reg path)
__global__ void attn_delta_kernel(const __nv_bfloat16* __restrict__ dO, int DP, const __nv_bfloat16* __restrict__ O,
                                  long long ldo, int heads, int d, int N, long long total,
                                  const float* __restrict__ pcols, const float* __restrict__ gcols,
                                  float* __restrict__ delta) {
  pdl_wait();
  pdl_launch_dependents();
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;   // bh * N + q
  if (idx >= total) return;
  const int q = (int)(idx % N);
  const int bh = (int)(idx / N);
  const int b = bh / heads, h = bh - b * heads;
  const __nv_bfloat16* dr = dO + idx * DP;
  const __nv_bfloat16* orow = O + ((long long)b * N + q) * ldo + h * d;
  float acc = 0.f;
  for (int c = 0; c < d / 8; ++c) {
    float a[8], g[8];
    unpack8(__ldg(reinterpret_cast<const uint4*>(dr + c * 8)), a);
    unpack8(__ldg(reinterpret_cast<const uint4*>(orow + c * 8)), g);
#pragma unroll
    for (int i = 0; i < 8; ++i) acc += a[i] * g[i];
  }
  if (pcols) {
    const float2 pc = *reinterpret_cast<const float2*>(pcols + idx * 2);
    const float2 gc = *reinterpret_cast<const float2*>(gcols + ((long long)b * N + q) * 2);
    acc += pc.x * gc.x + pc.y * gc.y;
  }
  delta[idx] = acc;
}

// ------------------------------------------------------------------------------------------------ LoRA gradients
// y = x W^T + alpha (x D^T) U^T  (edlora.py:244-246), dY given:
//   dU[n, r] = alpha sum_m dY[m, n] t[m, r],  t = x D^T ;   dD[r, k] = alpha sum_m s[m, r] x[m, k],  s = dY U
// Both gradients are skinny reductions over the M rows.  One block owns a slab of R rows (R chosen on the host so that
// at most 128 blocks exist):
//   step 1  t, s of every slab row -> smem (thread = (row, column part); D and U staged in smem, read as broadcasts)
//   step 2  thread (row group g of 4, lane) owns an 8-column chunk of x (-> dD) or dY (-> dU): one 128-bit load and 32
//           FMAs per row; the 4 row groups are summed in a fixed order through smem
// and writes its partial [4K + 4N]; lora_grad_reduce_kernel sums the <= 128 partials in a fixed order (bitwise
// reproducible).
// STAGE = false is the wide-layer variant (e.g. the GEGLU projection 1280 -> 10240, where D and U alone need 210 KB): D and
// U are read from global memory (L1 / L2 resident, 4 (K + N) floats) instead of being staged, and nothing else changes,
// so both variants give the same bits for any shape both accept.
constexpr int LG_THREADS = 256;
constexpr int LG_MAX_BLOCKS = 128;
constexpr long long LG_SMEM_MAX = 200 * 1024;

template <bool STAGE>
__global__ void __launch_bounds__(LG_THREADS)
lora_grad_partial_kernel(const __nv_bfloat16* __restrict__ x, long long ldx, const __nv_bfloat16* __restrict__ dy,
                         long long lddy, long long M, int K, int N, const float* __restrict__ down,
                         const float* __restrict__ up, int R, float* __restrict__ partial) {
  extern __shared__ float lg_smem[];
  float* ts = STAGE ? lg_smem + 4 * K + 4 * N : lg_smem;   // [R][8]: t[0..3], s[0..3]
  float* red = ts + (long long)R * 8;                      // [4 groups][32 values][64 lanes]
  const float* sD = down;              // [4][K]
  const float* sU = up;                // [N][4]
  pdl_wait();
  pdl_launch_dependents();
  const int tid = threadIdx.x;
  const long long m0 = (long long)blockIdx.x * R;
  const int rows = (int)min((long long)R, M - m0);
  if (STAGE) {
    float* stD = lg_smem;
    float* stU = stD + 4 * K;
    for (int i = tid * 4; i < 4 * K; i += LG_THREADS * 4)
      *reinterpret_cast<float4*>(stD + i) = __ldg(reinterpret_cast<const float4*>(down + i));
    for (int i = tid * 4; i < 4 * N; i += LG_THREADS * 4)
      *reinterpret_cast<float4*>(stU + i) = __ldg(reinterpret_cast<const float4*>(up + i));
    sD = stD;
    sU = stU;
    __syncthreads();
  }
  // ---- step 1: t = x D^T, s = dY U for every row of the slab.  Thread = (row, part): with R <= 128 rows the 256 threads
  // split every row's columns P = 256 / R ways (chunk c goes to part c mod P); partial dots are summed in a fixed order.
  const int P = R >= LG_THREADS ? 1 : LG_THREADS / R;
  float* tsp = P > 1 ? red : ts;       // [P][R][8] partial dots (aliases the step-2 reduction buffer; P * R * 8 <= 2048)
  for (int idx = tid; idx < R * P; idx += LG_THREADS) {
    const int r = idx % R, part = idx / R;
    float t[4] = {0.f, 0.f, 0.f, 0.f}, sv[4] = {0.f, 0.f, 0.f, 0.f};
    if (r < rows) {
      const __nv_bfloat16* xr = x + (m0 + r) * ldx;
#pragma unroll 8
      for (int k = part * 8; k < K; k += P * 8) {
        float v[8];
        unpack8(__ldg(reinterpret_cast<const uint4*>(xr + k)), v);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float4 d0 = *reinterpret_cast<const float4*>(sD + q * K + k);
          const float4 d1 = *reinterpret_cast<const float4*>(sD + q * K + k + 4);
          t[q] += v[0] * d0.x + v[1] * d0.y + v[2] * d0.z + v[3] * d0.w + v[4] * d1.x + v[5] * d1.y + v[6] * d1.z +
                  v[7] * d1.w;
        }
      }
      const __nv_bfloat16* dr = dy + (m0 + r) * lddy;
#pragma unroll 8
      for (int n = part * 8; n < N; n += P * 8) {
        float v[8];
        unpack8(__ldg(reinterpret_cast<const uint4*>(dr + n)), v);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float4 u = *reinterpret_cast<const float4*>(sU + (n + i) * 4);
          sv[0] += v[i] * u.x;
          sv[1] += v[i] * u.y;
          sv[2] += v[i] * u.z;
          sv[3] += v[i] * u.w;
        }
      }
    }
    float* o = tsp + ((long long)part * R + r) * 8;
    *reinterpret_cast<float4*>(o) = make_float4(t[0], t[1], t[2], t[3]);
    *reinterpret_cast<float4*>(o + 4) = make_float4(sv[0], sv[1], sv[2], sv[3]);
  }
  __syncthreads();
  if (P > 1) {
    for (int i = tid; i < R * 8; i += LG_THREADS) {
      float a = 0.f;
      for (int part = 0; part < P; ++part) a += tsp[(long long)part * R * 8 + i];
      ts[i] = a;
    }
    __syncthreads();
  }
  // ---- step 2: dD[q, k] = sum_r s[r, q] x[r, k];  dU[n, q] = sum_r t[r, q] dY[r, n]
  const int g = tid >> 6, ln = tid & 63;
  const int CK = K / 8, CH = CK + N / 8;
  const int rpg = R / 4;
  const int r_lo = g * rpg, r_hi = min(rows, (g + 1) * rpg);
  float* pblk = partial + (long long)blockIdx.x * 4 * (K + N);
  for (int c0 = 0; c0 < CH; c0 += 64) {
    const int c = c0 + ln;
    const bool active = c < CH;
    float acc[4][8];
#pragma unroll
    for (int q = 0; q < 4; ++q)
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[q][i] = 0.f;
    if (active) {
      const bool isx = c < CK;
      const __nv_bfloat16* base = isx ? x + m0 * ldx + c * 8 : dy + m0 * lddy + (c - CK) * 8;
      const long long ld = isx ? ldx : lddy;
      const float* w = ts + (isx ? 4 : 0);
#pragma unroll 8
      for (int r = r_lo; r < r_hi; ++r) {
        float v[8];
        unpack8(__ldg(reinterpret_cast<const uint4*>(base + r * ld)), v);
        const float4 wr = *reinterpret_cast<const float4*>(w + r * 8);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          acc[0][i] += wr.x * v[i];
          acc[1][i] += wr.y * v[i];
          acc[2][i] += wr.z * v[i];
          acc[3][i] += wr.w * v[i];
        }
      }
    }
#pragma unroll
    for (int q = 0; q < 4; ++q)
#pragma unroll
      for (int i = 0; i < 8; ++i) red[(g * 32 + q * 8 + i) * 64 + ln] = acc[q][i];
    __syncthreads();
    if (g == 0 && active) {
      float sum[4][8];
#pragma unroll
      for (int q = 0; q < 4; ++q)
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int j = q * 8 + i;
          sum[q][i] = ((red[j * 64 + ln] + red[(32 + j) * 64 + ln]) + red[(64 + j) * 64 + ln]) + red[(96 + j) * 64 + ln];
        }
      if (c < CK) {   // dD, layout [4][K]
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          float* d = pblk + (long long)q * K + c * 8;
          *reinterpret_cast<float4*>(d) = make_float4(sum[q][0], sum[q][1], sum[q][2], sum[q][3]);
          *reinterpret_cast<float4*>(d + 4) = make_float4(sum[q][4], sum[q][5], sum[q][6], sum[q][7]);
        }
      } else {        // dU, layout [N][4]
        float* d = pblk + 4LL * K + (long long)(c - CK) * 32;
#pragma unroll
        for (int i = 0; i < 8; ++i)
          *reinterpret_cast<float4*>(d + i * 4) = make_float4(sum[0][i], sum[1][i], sum[2][i], sum[3][i]);
      }
    }
    __syncthreads();
  }
}

// grad[i] (+)= alpha * sum_blk partial[blk][i];  i < n_down -> d_down, else d_up
__global__ void lora_grad_reduce_kernel(const float* __restrict__ partial, int nblk_, long long n_down, long long n,
                                        float alpha, int accumulate, float* __restrict__ d_down,
                                        float* __restrict__ d_up) {
  pdl_wait();
  pdl_launch_dependents();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float a = 0.f;
  for (int b = 0; b < nblk_; ++b) a += partial[(long long)b * n + i];
  float* g = i < n_down ? d_down + i : d_up + (i - n_down);
  *g = (accumulate ? *g : 0.f) + alpha * a;
}


// ------------------------------------------------------------------------------------------------ attention regulariser
// cal_attn_reg (trainer_edlora.py:281-313) on the two concept-token columns only.  Per resolution group:
//   cm[b, n, c] = mean over (layers of the group x heads) of pcols_l[(b, h), n, c]
//   y_c = cm_c / max(cm_c)  (max over the whole batch);  gt = nearest-resized mask
//   loss = w * ( full ? mean((y_1 - gt)^2) : mean_{gt==0} y_1   +   mean_{gt==0} y_0 )
// stats[8] per group = {max0, max1, T0, T1, nzero, loss, S0, S1}, S_c = sum_i g_i x_i (g = dloss/dy), T_c = the number of
// elements equal to max_c (torch's max() backward splits the gradient of the maximum evenly among them)
struct RegPtrs {
  const float* p[8];
};

__global__ void attnreg_mean_kernel(RegPtrs tab, int L, int heads, int B, int N, float* __restrict__ cm) {
  pdl_wait();
  pdl_launch_dependents();
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)B * N * 2) return;
  const int c = (int)(idx & 1);
  const long long bn = idx >> 1;
  const int n = (int)(bn % N), b = (int)(bn / N);
  float acc = 0.f;
  for (int l = 0; l < L; ++l)
    for (int h = 0; h < heads; ++h) acc += tab.p[l][(((long long)b * heads + h) * N + n) * 2 + c];
  cm[idx] = acc / (float)(L * heads);
}

__device__ __forceinline__ float reg_gt(const float* __restrict__ mask, int b, int n, int res, int MH, int MW) {
  const int y = n / res, x = n - y * res;
  const int sy = min((int)floorf((float)y * ((float)MH / (float)res)), MH - 1);
  const int sx = min((int)floorf((float)x * ((float)MW / (float)res)), MW - 1);
  return mask[((long long)b * MH + sy) * MW + sx];
}

__global__ void __launch_bounds__(1024)
attnreg_reduce_kernel(const float* __restrict__ cm, const float* __restrict__ mask, int B, int res, int MH, int MW,
                      int full_identity, float weight, float* __restrict__ stats) {
  __shared__ float sv[5][32];
  __shared__ float bc[8];
  pdl_wait();
  pdl_launch_dependents();
  const int N = res * res, total = B * N;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  // ---- phase 1: max per column, number of zero mask pixels
  float m0 = -INFINITY, m1 = -INFINITY, nz = 0.f;
  for (int i = threadIdx.x; i < total; i += blockDim.x) {
    m0 = fmaxf(m0, cm[2 * i]);
    m1 = fmaxf(m1, cm[2 * i + 1]);
    nz += (reg_gt(mask, i / N, i % N, res, MH, MW) == 0.f) ? 1.f : 0.f;
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, d));
    m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, d));
    nz += __shfl_xor_sync(0xffffffffu, nz, d);
  }
  if (lane == 0) { sv[0][warp] = m0; sv[1][warp] = m1; sv[2][warp] = nz; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float M0 = -INFINITY, M1 = -INFINITY, Z = 0.f;
    for (int w = 0; w < nw; ++w) {
      M0 = fmaxf(M0, sv[0][w]);
      M1 = fmaxf(M1, sv[1][w]);
      Z += sv[2][w];
    }
    bc[0] = M0; bc[1] = M1; bc[2] = Z;
    stats[0] = M0; stats[1] = M1;
    stats[4] = Z;
  }
  __syncthreads();
  const float M0 = bc[0], M1 = bc[1], Z = bc[2];
  // ---- phase 2: loss, S_c = sum_i g_i x_i and the tie counts T_c
  float ls = 0.f, s0 = 0.f, s1 = 0.f, t0 = 0.f, t1 = 0.f;
  for (int i = threadIdx.x; i < total; i += blockDim.x) {
    const float x0 = cm[2 * i], x1 = cm[2 * i + 1];
    const float gt = reg_gt(mask, i / N, i % N, res, MH, MW);
    const float y0 = x0 / M0, y1 = x1 / M1;
    const float zero = (gt == 0.f) ? 1.f : 0.f;
    float g1;
    if (full_identity) {
      ls += (y1 - gt) * (y1 - gt) / (float)total;
      g1 = 2.0f * (y1 - gt) / (float)total;
    } else {
      ls += zero * y1 / Z;
      g1 = zero / Z;
    }
    ls += zero * y0 / Z;
    s0 += (zero / Z) * x0;
    s1 += g1 * x1;
    t0 += (x0 == M0) ? 1.f : 0.f;
    t1 += (x1 == M1) ? 1.f : 0.f;
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    ls += __shfl_xor_sync(0xffffffffu, ls, d);
    s0 += __shfl_xor_sync(0xffffffffu, s0, d);
    s1 += __shfl_xor_sync(0xffffffffu, s1, d);
    t0 += __shfl_xor_sync(0xffffffffu, t0, d);
    t1 += __shfl_xor_sync(0xffffffffu, t1, d);
  }
  __syncthreads();
  if (lane == 0) { sv[0][warp] = ls; sv[1][warp] = s0; sv[2][warp] = s1; sv[3][warp] = t0; sv[4][warp] = t1; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = 0.f, b = 0.f, c = 0.f, u0 = 0.f, u1 = 0.f;
    for (int w = 0; w < nw; ++w) { a += sv[0][w]; b += sv[1][w]; c += sv[2][w]; u0 += sv[3][w]; u1 += sv[4][w]; }
    stats[2] = u0;
    stats[3] = u1;
    stats[5] = weight * a;   // NaN when Z == 0, as the reference's mean over an empty selection
    stats[6] = b;
    stats[7] = c;
  }
}

// gcols[b, n, c] = valid * w * (g_c / max_c - [x_c == max_c] S_c / (max_c^2 T_c)) / (heads * L)
__global__ void attnreg_grad_kernel(const float* __restrict__ cm, const float* __restrict__ mask, int B, int res,
                                    int MH, int MW, int full_identity, float weight, const float* __restrict__ stats_all,
                                    int ngroups, int group, int L, int heads, float grad_scale,
                                    float* __restrict__ gcols) {
  pdl_wait();
  pdl_launch_dependents();
  const int N = res * res, total = B * N;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  bool valid = true;
  for (int g = 0; g < ngroups; ++g) valid = valid && (stats_all[g * 8 + 4] > 0.f);
  const float* st = stats_all + group * 8;
  const float M0 = st[0], M1 = st[1], T0 = st[2], T1 = st[3], Z = st[4], S0 = st[6], S1 = st[7];
  const float gt = reg_gt(mask, i / N, i % N, res, MH, MW);
  const float zero = (gt == 0.f) ? 1.f : 0.f;
  const float x0 = cm[2 * i], x1 = cm[2 * i + 1];
  const float g1 = full_identity ? 2.0f * (x1 / M1 - gt) / (float)total : zero / Z;
  const float g0 = zero / Z;
  const float k = valid ? grad_scale * weight / (float)(heads * L) : 0.f;
  float d0 = g0 / M0 - (x0 == M0 ? S0 / (M0 * M0 * T0) : 0.f);
  float d1 = g1 / M1 - (x1 == M1 ? S1 / (M1 * M1 * T1) : 0.f);
  if (!valid) d0 = d1 = 0.f;   // avoid 0 * NaN
  gcols[2 * i] = k * d0;
  gcols[2 * i + 1] = k * d1;
}

// out[0] = mse + (valid ? sum_g loss_g : 0);  out[1] = sum_g loss_g (NaN when some resized mask has no zero, :257)
__global__ void attnreg_total_kernel(const float* __restrict__ mse, const float* __restrict__ stats_all, int ngroups,
                                     float* __restrict__ out) {
  pdl_wait();
  pdl_launch_dependents();
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  float a = 0.f;
  for (int g = 0; g < ngroups; ++g) a += stats_all[g * 8 + 5];
  out[1] = a;
  out[0] = mse[0] + (isnan(a) ? 0.f : a);
}

}  // namespace mos

using namespace mos;

extern "C" int mos_geglu_fwd(const void* z, int64_t ldz, int64_t M, int32_t H, void* y, int64_t ldy, void* stream) {
  MOS_CHECK_ARG(z && y && H % 80 == 0 && ldz % 8 == 0 && ldy % 8 == 0 && ldz >= 2 * H && ldy >= H,
                "mos_geglu_fwd: bad arguments (H=%d must be a multiple of 80)", H);
  MOS_CHECK_CUDA(launch_pdl(geglu_fwd_kernel, dim3(nblk(M * (H / 8), 256)), dim3(256), 0, STREAM(stream),
                            reinterpret_cast<const __nv_bfloat16*>(z), (long long)ldz, (long long)M, (int)H,
                            reinterpret_cast<__nv_bfloat16*>(y), (long long)ldy));
  return MOS_OK;
}

extern "C" int mos_geglu_bwd(const void* z, int64_t ldz, const void* dy, int64_t lddy, int64_t M, int32_t H, void* dz,
                             int64_t lddz, void* stream) {
  MOS_CHECK_ARG(z && dy && dz && H % 80 == 0 && ldz % 8 == 0 && lddy % 8 == 0 && lddz % 8 == 0 && ldz >= 2 * H &&
                    lddz >= 2 * H && lddy >= H, "mos_geglu_bwd: bad arguments (H=%d must be a multiple of 80)", H);
  MOS_CHECK_CUDA(launch_pdl(geglu_bwd_kernel, dim3(nblk(M * (H / 8), 256)), dim3(256), 0, STREAM(stream),
                            reinterpret_cast<const __nv_bfloat16*>(z), (long long)ldz,
                            reinterpret_cast<const __nv_bfloat16*>(dy), (long long)lddy, (long long)M, (int)H,
                            reinterpret_cast<__nv_bfloat16*>(dz), (long long)lddz));
  return MOS_OK;
}

extern "C" int mos_upsample2x_bwd(const void* dy, int64_t lddy, int32_t B, int32_t H, int32_t W, int32_t C, void* dx,
                                  int64_t lddx, void* stream) {
  MOS_CHECK_ARG(dy && dx && C % 8 == 0 && lddy % 8 == 0 && lddx % 8 == 0, "mos_upsample2x_bwd: bad arguments");
  MOS_CHECK_CUDA(launch_pdl(upsample2x_bwd_kernel, dim3(nblk((long long)B * H * W * (C / 8), 256)), dim3(256), 0,
                            STREAM(stream), reinterpret_cast<const __nv_bfloat16*>(dy), (long long)lddy, (int)B, (int)H,
                            (int)W, (int)C, reinterpret_cast<__nv_bfloat16*>(dx), (long long)lddx));
  return MOS_OK;
}

extern "C" int mos_col2im_s2(const void* dcol, int32_t B, int32_t H, int32_t W, int32_t C, const void* add,
                             int64_t ldadd, void* dx, int64_t lddx, void* stream) {
  MOS_CHECK_ARG(dcol && dx && C % 8 == 0 && lddx % 8 == 0 && H % 2 == 0 && W % 2 == 0 && (!add || ldadd % 8 == 0),
                "mos_col2im_s2: bad arguments");
  MOS_CHECK_CUDA(launch_pdl(col2im_s2_kernel, dim3(nblk((long long)B * H * W * (C / 8), 256)), dim3(256), 0,
                            STREAM(stream), reinterpret_cast<const __nv_bfloat16*>(dcol), (int)B, (int)H, (int)W, (int)C,
                            reinterpret_cast<const __nv_bfloat16*>(add), (long long)ldadd,
                            reinterpret_cast<__nv_bfloat16*>(dx), (long long)lddx));
  return MOS_OK;
}

extern "C" int mos_conv_out_bwd(const float* dy, int32_t B, int32_t H, int32_t W, int32_t C, const float* w,
                                int32_t Cout, void* dx, void* stream) {
  MOS_CHECK_ARG(dy && w && dx && C % 8 == 0 && Cout >= 1 && Cout <= 4, "mos_conv_out_bwd: bad arguments");
  MOS_CHECK_CUDA(launch_pdl(conv_out_bwd_kernel, dim3(nblk((long long)B * H * W * (C / 8), 256)), dim3(256), 0,
                            STREAM(stream), dy, (int)B, (int)H, (int)W, (int)C, w, (int)Cout,
                            reinterpret_cast<__nv_bfloat16*>(dx)));
  return MOS_OK;
}

extern "C" int mos_masked_mse(const float* pred, const float* target, const float* mask, int32_t B, int32_t Cc,
                              int32_t HW, float grad_scale, float* ws, float* loss, float* dpred, void* stream) {
  MOS_CHECK_ARG(pred && target && mask && ws && loss && dpred && B > 0, "mos_masked_mse: bad arguments");
  MOS_CHECK_CUDA(launch_pdl(mse_sums_kernel, dim3(B), dim3(256), 0, STREAM(stream), pred, target, mask, (int)Cc, (int)HW, ws));
  MOS_CHECK_CUDA(launch_pdl(mse_grad_kernel, dim3(nblk((long long)B * Cc * HW, 256)), dim3(256), 0, STREAM(stream), pred,
                            target, mask, (int)B, (int)Cc, (int)HW, (const float*)ws, grad_scale, dpred, loss));
  return MOS_OK;
}

extern "C" int mos_add_noise(const float* x0, const float* noise, const int32_t* timesteps,
                             const float* alphas_cumprod, int32_t B, int64_t per_sample, float* out, void* stream) {
  MOS_CHECK_ARG(x0 && noise && timesteps && alphas_cumprod && out && B > 0, "mos_add_noise: bad arguments");
  MOS_CHECK_CUDA(launch_pdl(add_noise_kernel, dim3(nblk(B * per_sample, 256)), dim3(256), 0, STREAM(stream), x0, noise,
                            reinterpret_cast<const int*>(timesteps), alphas_cumprod, (long long)per_sample,
                            (long long)B * per_sample, out));
  return MOS_OK;
}

extern "C" int mos_heads_transpose(const void* src, int32_t BH, int32_t R, int32_t DP, int32_t DV, int32_t R8, void* dst,
                                   void* stream) {
  MOS_CHECK_ARG(src && dst && DV <= DP && R8 >= R && R8 % 8 == 0, "mos_heads_transpose: bad arguments");
  dim3 grid(nblk(R, 32), nblk(DV, 32), BH);
  MOS_CHECK_CUDA(launch_pdl(heads_transpose_kernel, grid, dim3(32, 8), 0, STREAM(stream),
                            reinterpret_cast<const __nv_bfloat16*>(src), (int)R, (int)DP, (int)DV, (int)R8,
                            reinterpret_cast<__nv_bfloat16*>(dst)));
  return MOS_OK;
}

extern "C" int mos_attn_delta(const void* dO, int32_t DP, const void* O, int64_t ldo, int32_t batch, int32_t heads,
                              int32_t head_dim, int32_t N, const float* pcols, const float* gcols, float* delta,
                              void* stream) {
  MOS_CHECK_ARG(dO && O && delta && head_dim % 8 == 0 && DP % 8 == 0 && ldo % 8 == 0 && (!pcols == !gcols),
                "mos_attn_delta: bad arguments");
  const long long total = (long long)batch * heads * N;
  MOS_CHECK_CUDA(launch_pdl(attn_delta_kernel, dim3(nblk(total, 128)), dim3(128), 0, STREAM(stream),
                            reinterpret_cast<const __nv_bfloat16*>(dO), (int)DP, reinterpret_cast<const __nv_bfloat16*>(O),
                            (long long)ldo, (int)heads, (int)head_dim, (int)N, total, pcols, gcols, delta));
  return MOS_OK;
}

extern "C" int mos_lora_grad(const void* x, int64_t ldx, const void* dy, int64_t lddy, int64_t M, int32_t K, int32_t N,
                             const float* down, const float* up, float alpha, float* workspace,
                             int64_t workspace_floats, int32_t accumulate, float* d_down, float* d_up, void* stream) {
  MOS_CHECK_ARG(x && dy && down && up && workspace && d_down && d_up, "mos_lora_grad: NULL pointer");
  MOS_CHECK_ARG(K % 8 == 0 && N % 8 == 0 && ldx % 8 == 0 && lddy % 8 == 0 && M > 0, "mos_lora_grad: bad shape");
  // slab height: a multiple of 64 rows such that at most LG_MAX_BLOCKS blocks exist
  long long R = ceil_div(ceil_div(M, (long long)LG_MAX_BLOCKS), 16LL) * 16;   // 16 | R, and R | 256 or 256 | R below
  if (R > 1024) R = 1024;
  if (R < 256) { long long p2 = 16; while (p2 < R) p2 *= 2; R = p2; } else R = ceil_div(R, 256LL) * 256;
  const int nb = (int)ceil_div(M, R);
  MOS_CHECK_ARG((long long)nb * 4 * (K + N) <= workspace_floats, "mos_lora_grad: workspace too small (need %lld floats)",
                (long long)nb * 4 * (K + N));
  // D and U are staged in shared memory whenever they fit next to the slab's t / s rows and the reduction buffer; wider
  // layers read them from global memory (same arithmetic, same bits)
  const size_t smem_work = (size_t)(R * 8 + 4 * 32 * 64) * sizeof(float);
  const size_t smem_staged = smem_work + (size_t)(4LL * K + 4LL * N) * sizeof(float);
  const bool stage = smem_staged <= (size_t)LG_SMEM_MAX;
  static bool configured = false;
  if (!configured) {
    MOS_CHECK_CUDA(cudaFuncSetAttribute(lora_grad_partial_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        (int)LG_SMEM_MAX));
    MOS_CHECK_CUDA(cudaFuncSetAttribute(lora_grad_partial_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        (int)LG_SMEM_MAX));
    configured = true;
  }
  MOS_CHECK_CUDA(launch_pdl(stage ? lora_grad_partial_kernel<true> : lora_grad_partial_kernel<false>, dim3(nb),
                            dim3(LG_THREADS), stage ? smem_staged : smem_work, STREAM(stream),
                            reinterpret_cast<const __nv_bfloat16*>(x), (long long)ldx,
                            reinterpret_cast<const __nv_bfloat16*>(dy), (long long)lddy, (long long)M, (int)K, (int)N, down,
                            up, (int)R, workspace));
  const long long n = 4LL * (K + N);
  MOS_CHECK_CUDA(launch_pdl(lora_grad_reduce_kernel, dim3(nblk(n, 256)), dim3(256), 0, STREAM(stream),
                            (const float*)workspace, nb, 4LL * K, n, alpha, (int)accumulate, d_down, d_up));
  return MOS_OK;
}


extern "C" int mos_attn_reg_group(const float* const* pcols_host_ptrs, int32_t L, int32_t B, int32_t heads, int32_t res,
                                  const float* mask, int32_t MH, int32_t MW, int32_t full_identity, float weight,
                                  float* cm, float* stats, void* stream) {
  MOS_CHECK_ARG(pcols_host_ptrs && mask && cm && stats && L >= 1 && L <= 8 && B > 0 && res > 0,
                "mos_attn_reg_group: bad arguments (1 <= layers per group <= 8)");
  RegPtrs tab;
  for (int l = 0; l < 8; ++l) tab.p[l] = l < L ? pcols_host_ptrs[l] : nullptr;
  const int N = res * res;
  MOS_CHECK_CUDA(launch_pdl(attnreg_mean_kernel, dim3(nblk((long long)B * N * 2, 256)), dim3(256), 0, STREAM(stream), tab,
                            (int)L, (int)heads, (int)B, N, cm));
  MOS_CHECK_CUDA(launch_pdl(attnreg_reduce_kernel, dim3(1), dim3(1024), 0, STREAM(stream), (const float*)cm, mask, (int)B,
                            (int)res, (int)MH, (int)MW, (int)full_identity, weight, stats));
  return MOS_OK;
}

extern "C" int mos_attn_reg_grad(const float* cm, const float* mask, int32_t B, int32_t res, int32_t MH, int32_t MW,
                                 int32_t full_identity, float weight, const float* stats_all, int32_t ngroups,
                                 int32_t group, int32_t L, int32_t heads, float grad_scale, float* gcols,
                                 void* stream) {
  MOS_CHECK_ARG(cm && mask && stats_all && gcols && group >= 0 && group < ngroups, "mos_attn_reg_grad: bad arguments");
  MOS_CHECK_CUDA(launch_pdl(attnreg_grad_kernel, dim3(nblk((long long)B * res * res, 256)), dim3(256), 0, STREAM(stream),
                            cm, mask, (int)B, (int)res, (int)MH, (int)MW, (int)full_identity, weight, stats_all,
                            (int)ngroups, (int)group, (int)L, (int)heads, grad_scale, gcols));
  return MOS_OK;
}

extern "C" int mos_attn_reg_total(const float* mse, const float* stats_all, int32_t ngroups, float* out, void* stream) {
  MOS_CHECK_ARG(mse && stats_all && out && ngroups >= 1, "mos_attn_reg_total: bad arguments");
  MOS_CHECK_CUDA(launch_pdl(attnreg_total_kernel, dim3(1), dim3(32), 0, STREAM(stream), mse, stats_all, (int)ngroups, out));
  return MOS_OK;
}
