// elementwise.cu — K6 and the small edge kernels of the denoise step (all HBM/latency-bound glue):
//   timestep embedding + small-batch GEMV (time MLP, the 22 time_emb_proj in one launch)
//   conv_in (NCHW fp32 latents -> NHWC bf16), conv_out (NHWC bf16 -> NCHW fp32)
//   nearest 2x upsample, stride-2 im2col (Downsample2D), strided add (T2I-Adapter residuals)
//   CFG combine + DPM-Solver++(2M) update (pipeline_edlora.py:273-290), region combine (regional :54-83)
#include "common.h"
#include "tc.cuh"

namespace mos {

// ---------------------------------------------------------------------------------- timestep embedding
// out[b, :] = [cos(t_b * f_i) | sin(t_b * f_i)], f_i = exp(-ln(10000) * i / half)   (flip_sin_to_cos, shift 0)
__global__ void timestep_embed_kernel(const float* __restrict__ t, int dim, float* __restrict__ out) {
  pdl_wait();
  pdl_launch_dependents();
  const int b = blockIdx.x, half = dim / 2;
  for (int i = threadIdx.x; i < half; i += blockDim.x) {
    float f = expf(-9.210340371976184f * (float)i / (float)half);
    float a = t[b] * f;
    out[b * dim + i] = cosf(a);
    out[b * dim + half + i] = sinf(a);
  }
}

// out[b, n] = act_out( bias[n] + sum_k act_in(x[b, k]) * W[n, k] ),  nb <= 8 rows, one warp per output column
template <int NB>
__global__ void gemv_kernel(const float* __restrict__ x, int K, const __nv_bfloat16* __restrict__ W,
                            const float* __restrict__ bias, int N, int act_in, int act_out, float* __restrict__ out,
                            long long ldo) {
  pdl_wait();
  pdl_launch_dependents();
  const int n = blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (n >= N) return;
  float acc[NB];
#pragma unroll
  for (int b = 0; b < NB; ++b) acc[b] = 0.f;
  const __nv_bfloat16* wr = W + (long long)n * K;
  for (int k = lane * 8; k < K; k += 256) {
    uint4 u = __ldg(reinterpret_cast<const uint4*>(wr + k));
    uint32_t w[4] = {u.x, u.y, u.z, u.w};
    float wf[8];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float2 f = unpack_bf16x2(w[i]);
      wf[2 * i] = f.x;
      wf[2 * i + 1] = f.y;
    }
#pragma unroll
    for (int b = 0; b < NB; ++b) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float xv = __ldg(x + (long long)b * K + k + i);
        if (act_in) xv = silu(xv);
        acc[b] += xv * wf[i];
      }
    }
  }
#pragma unroll
  for (int b = 0; b < NB; ++b) {
    float v = acc[b];
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
    if (lane == 0) {
      v += bias ? bias[n] : 0.f;
      if (act_out) v = silu(v);
      out[(long long)b * ldo + n] = v;
    }
  }
}

// ---------------------------------------------------------------------------------- conv_in / conv_out
// x: NCHW fp32 [B, Cin(4), H, W]; w: fp32 [9*Cin][Cout] (tap-major, Cout contiguous); y: NHWC bf16 [B,H,W,ldy]
template <bool F16>
__global__ void conv_in_kernel(const float* __restrict__ x, int B, int Cin, int H, int W,
                               const float* __restrict__ w, const float* __restrict__ bias, int Cout,
                               __nv_bfloat16* __restrict__ y, long long ldy) {
  pdl_wait();
  pdl_launch_dependents();
  const int oct = Cout / 8;
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long total = (long long)B * H * W * oct;
  if (idx >= total) return;
  const int o = (int)(idx % oct);
  long long pix = idx / oct;
  const int wq = (int)(pix % W);
  const int hq = (int)((pix / W) % H);
  const int b = (int)(pix / ((long long)W * H));
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = __ldg(bias + o * 8 + i);
  for (int kh = 0; kh < 3; ++kh) {
    int hh = hq + kh - 1;
    if (hh < 0 || hh >= H) continue;
    for (int kw = 0; kw < 3; ++kw) {
      int ww = wq + kw - 1;
      if (ww < 0 || ww >= W) continue;
      for (int c = 0; c < Cin; ++c) {
        float xv = __ldg(x + (((long long)b * Cin + c) * H + hh) * W + ww);
        const float* wp = w + ((long long)((kh * 3 + kw) * Cin + c)) * Cout + o * 8;
        float4 w0 = __ldg(reinterpret_cast<const float4*>(wp));
        float4 w1 = __ldg(reinterpret_cast<const float4*>(wp + 4));
        acc[0] += xv * w0.x; acc[1] += xv * w0.y; acc[2] += xv * w0.z; acc[3] += xv * w0.w;
        acc[4] += xv * w1.x; acc[5] += xv * w1.y; acc[6] += xv * w1.z; acc[7] += xv * w1.w;
      }
    }
  }
  uint4 u;
  u.x = pack16x2<F16>(acc[0], acc[1]);
  u.y = pack16x2<F16>(acc[2], acc[3]);
  u.z = pack16x2<F16>(acc[4], acc[5]);
  u.w = pack16x2<F16>(acc[6], acc[7]);
  *reinterpret_cast<uint4*>(y + pix * ldy + o * 8) = u;
}

// x: NHWC bf16 [B,H,W,C] (contiguous, already GN+SiLU'd); w: fp32 [Cout(4)][9][C]; y: NCHW fp32 [B,Cout,H,W]
// one warp per output pixel
template <bool F16>
__global__ void conv_out_kernel(const __nv_bfloat16* __restrict__ x, int B, int H, int W, int C,
                                const float* __restrict__ w, const float* __restrict__ bias, int Cout,
                                float* __restrict__ y) {
  pdl_wait();
  pdl_launch_dependents();
  const long long pix = (long long)blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (pix >= (long long)B * H * W) return;
  const int wq = (int)(pix % W);
  const int hq = (int)((pix / W) % H);
  const int b = (int)(pix / ((long long)W * H));
  const int oct = C / 8;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int tap = 0; tap < 9; ++tap) {
    int hh = hq + tap / 3 - 1, ww = wq + tap % 3 - 1;
    if (hh < 0 || hh >= H || ww < 0 || ww >= W) continue;
    const __nv_bfloat16* xp = x + (((long long)b * H + hh) * W + ww) * C;
    for (int o = lane; o < oct; o += 32) {
      uint4 u = __ldg(reinterpret_cast<const uint4*>(xp + o * 8));
      uint32_t uw[4] = {u.x, u.y, u.z, u.w};
      float xv[8];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        float2 f = unpack16x2<F16>(uw[i]);
        xv[2 * i] = f.x;
        xv[2 * i + 1] = f.y;
      }
#pragma unroll
      for (int oc = 0; oc < 4; ++oc) {
        if (oc < Cout) {
          const float* wp = w + ((long long)oc * 9 + tap) * C + o * 8;
          float4 w0 = __ldg(reinterpret_cast<const float4*>(wp));
          float4 w1 = __ldg(reinterpret_cast<const float4*>(wp + 4));
          acc[oc] += xv[0] * w0.x + xv[1] * w0.y + xv[2] * w0.z + xv[3] * w0.w + xv[4] * w1.x + xv[5] * w1.y +
                     xv[6] * w1.z + xv[7] * w1.w;
        }
      }
    }
  }
#pragma unroll
  for (int oc = 0; oc < 4; ++oc) {
    float v = acc[oc];
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
    if (lane == 0 && oc < Cout) y[(((long long)b * Cout + oc) * H + hq) * W + wq] = v + bias[oc];
  }
}

// ---------------------------------------------------------------------------------- resampling helpers
// y[b, 2h+i, 2w+j, :] = x[b, h, w, :]   (F.interpolate nearest, scale 2)
__global__ void upsample2x_kernel(const __nv_bfloat16* __restrict__ x, long long ldx, int B, int H, int W, int C,
                                  __nv_bfloat16* __restrict__ y) {
  pdl_wait();
  pdl_launch_dependents();
  const int oct = C / 8;
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long total = (long long)B * 2 * H * 2 * W * oct;
  if (idx >= total) return;
  const int o = (int)(idx % oct);
  long long pix = idx / oct;
  const int wo = (int)(pix % (2 * W));
  const int ho = (int)((pix / (2 * W)) % (2 * H));
  const int b = (int)(pix / ((long long)4 * W * H));
  uint4 u = __ldg(reinterpret_cast<const uint4*>(x + (((long long)b * H + ho / 2) * W + wo / 2) * ldx + o * 8));
  *reinterpret_cast<uint4*>(y + pix * C + o * 8) = u;
}

// y[b, ho, wo, :] = x[b, sh(ho), sw(wo), :]: F.interpolate(size=(Ho, Wo), mode='nearest') with PyTorch's source index
// rule, src = min(floor(dst * (in / out)), in - 1) in fp32 (dst >> 1 when out = 2 in).  diffusers' Upsample2D takes this
// path (output_size) when a latent side is not a multiple of 2^(levels - 1): each level is ceil(in / 2) of the one above.
__device__ __forceinline__ int nearest_src(int dst, int in, int out) {
  if (out == 2 * in) return dst >> 1;
  return min((int)floorf(__fmul_rn((float)dst, __fdiv_rn((float)in, (float)out))), in - 1);
}

__global__ void upsample_nearest_kernel(const __nv_bfloat16* __restrict__ x, long long ldx, int B, int H, int W, int C,
                                        int Ho, int Wo, __nv_bfloat16* __restrict__ y) {
  pdl_wait();
  pdl_launch_dependents();
  const int oct = C / 8;
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long total = (long long)B * Ho * Wo * oct;
  if (idx >= total) return;
  const int o = (int)(idx % oct);
  long long pix = idx / oct;
  const int wo = (int)(pix % Wo);
  const int ho = (int)((pix / Wo) % Ho);
  const int b = (int)(pix / ((long long)Wo * Ho));
  const int hs = nearest_src(ho, H, Ho), ws = nearest_src(wo, W, Wo);
  uint4 u = __ldg(reinterpret_cast<const uint4*>(x + (((long long)b * H + hs) * W + ws) * ldx + o * 8));
  *reinterpret_cast<uint4*>(y + pix * C + o * 8) = u;
}

// col[(b,ho,wo), tap*C + c] = x[b, 2ho+kh-1, 2wo+kw-1, c] (zero outside): Downsample2D conv 3x3 / stride 2 / pad 1, which
// gives ceil(H / 2) x ceil(W / 2) outputs; pad 0 (the VAE's, even sides only) gives H / 2 x W / 2
__global__ void im2col_s2_kernel(const __nv_bfloat16* __restrict__ x, long long ldx, int B, int H, int W, int C, int pad,
                                 __nv_bfloat16* __restrict__ col) {
  pdl_wait();
  pdl_launch_dependents();
  const int oct = C / 8, Ho = (H + pad) / 2, Wo = (W + pad) / 2;
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long total = (long long)B * Ho * Wo * 9 * oct;
  if (idx >= total) return;
  const int o = (int)(idx % oct);
  long long t = idx / oct;
  const int tap = (int)(t % 9);
  long long pix = t / 9;
  const int wo = (int)(pix % Wo);
  const int ho = (int)((pix / Wo) % Ho);
  const int b = (int)(pix / ((long long)Wo * Ho));
  const int hh = 2 * ho + tap / 3 - pad, ww = 2 * wo + tap % 3 - pad;   // pad 1: UNet Downsample2D; 0: VAE (pad right / bottom)
  uint4 u = make_uint4(0, 0, 0, 0);
  if (hh >= 0 && hh < H && ww >= 0 && ww < W)
    u = __ldg(reinterpret_cast<const uint4*>(x + (((long long)b * H + hh) * W + ww) * ldx + o * 8));
  *reinterpret_cast<uint4*>(col + pix * 9 * C + (long long)tap * C + o * 8) = u;
}

// x[m, :C] += r[m, :C]   (bf16, row pitches ldx / ldr)
template <bool F16>
__global__ void add_rows_kernel(__nv_bfloat16* __restrict__ x, long long ldx, const __nv_bfloat16* __restrict__ r,
                                long long ldr, long long M, int C) {
  pdl_wait();
  pdl_launch_dependents();
  const int oct = C / 8;
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= M * oct) return;
  const int o = (int)(idx % oct);
  const long long m = idx / oct;
  uint4 a = *reinterpret_cast<const uint4*>(x + m * ldx + o * 8);
  uint4 b = __ldg(reinterpret_cast<const uint4*>(r + m * ldr + o * 8));
  uint32_t aw[4] = {a.x, a.y, a.z, a.w}, bw[4] = {b.x, b.y, b.z, b.w}, ow[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 fa = unpack16x2<F16>(aw[i]), fb = unpack16x2<F16>(bw[i]);
    ow[i] = pack16x2<F16>(fa.x + fb.x, fa.y + fb.y);
  }
  *reinterpret_cast<uint4*>(x + m * ldx + o * 8) = make_uint4(ow[0], ow[1], ow[2], ow[3]);
}

// ---------------------------------------------------------------------------------- CLIP text encoder glue
// x[m, :C] = token_embedding[ids[m]] + position_embedding[m % T]   (fp32 tables -> bf16 rows; transformers
// CLIPTextEmbeddings as called through text_encoder(...) at pipeline_edlora.py:133-145); columns C..ld-1 are zeroed
// (the hidden state lives in a buffer padded to the GEMM's 160-column tile).
__global__ void clip_embed_kernel(const int* __restrict__ ids, const float* __restrict__ tok, const float* __restrict__ pos,
                                  long long M, int T, int C, int vocab, __nv_bfloat16* __restrict__ x, long long ld) {
  pdl_wait();
  pdl_launch_dependents();
  const int oct = (int)(ld / 8);
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= M * oct) return;
  const int o = (int)(idx % oct);
  const long long m = idx / oct;
  uint32_t w[4] = {0u, 0u, 0u, 0u};
  if (o * 8 < C) {
    int id = ids[m];
    id = min(max(id, 0), vocab - 1);
    const float* tr = tok + (long long)id * C + o * 8;
    const float* pr = pos + (long long)(m % T) * C + o * 8;
#pragma unroll
    for (int i = 0; i < 4; ++i) w[i] = pack_bf16x2(__ldg(tr + 2 * i) + __ldg(pr + 2 * i), __ldg(tr + 2 * i + 1) + __ldg(pr + 2 * i + 1));
  }
  *reinterpret_cast<uint4*>(x + m * ld + o * 8) = make_uint4(w[0], w[1], w[2], w[3]);
}

// quick-GELU in place: x <- x * sigmoid(1.702 x)   (CLIP MLP activation, transformers QuickGELUActivation)
__global__ void quick_gelu_kernel(__nv_bfloat16* __restrict__ x, long long ld, long long M, int C) {
  pdl_wait();
  pdl_launch_dependents();
  const int oct = C / 8;
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= M * oct) return;
  const int o = (int)(idx % oct);
  const long long m = idx / oct;
  uint4 a = *reinterpret_cast<const uint4*>(x + m * ld + o * 8);
  uint32_t aw[4] = {a.x, a.y, a.z, a.w}, ow[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 f = unpack_bf16x2(aw[i]);
    ow[i] = pack_bf16x2(f.x / (1.0f + __expf(-1.702f * f.x)), f.y / (1.0f + __expf(-1.702f * f.y)));
  }
  *reinterpret_cast<uint4*>(x + m * ld + o * 8) = make_uint4(ow[0], ow[1], ow[2], ow[3]);
}

// out-of-place quick-GELU (training forward keeps the pre-activation) and its backward:
//   y = x s, s = sigmoid(1.702 x);   dx = dy (s + 1.702 x s (1 - s))
__global__ void quick_gelu_fwd_kernel(const __nv_bfloat16* __restrict__ x, long long ldx, long long M, int C,
                                      __nv_bfloat16* __restrict__ y, long long ldy) {
  pdl_wait();
  pdl_launch_dependents();
  const int oct = C / 8;
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= M * oct) return;
  const int o = (int)(idx % oct);
  const long long m = idx / oct;
  uint4 a = __ldg(reinterpret_cast<const uint4*>(x + m * ldx + o * 8));
  uint32_t aw[4] = {a.x, a.y, a.z, a.w}, ow[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 f = unpack_bf16x2(aw[i]);
    ow[i] = pack_bf16x2(f.x / (1.0f + __expf(-1.702f * f.x)), f.y / (1.0f + __expf(-1.702f * f.y)));
  }
  *reinterpret_cast<uint4*>(y + m * ldy + o * 8) = make_uint4(ow[0], ow[1], ow[2], ow[3]);
}
__device__ __forceinline__ float quick_gelu_grad(float x) {
  const float s = 1.0f / (1.0f + __expf(-1.702f * x));
  return s + 1.702f * x * s * (1.0f - s);
}
__global__ void quick_gelu_bwd_kernel(const __nv_bfloat16* __restrict__ x, long long ldx, const __nv_bfloat16* __restrict__ dy,
                                      long long lddy, long long M, int C, __nv_bfloat16* __restrict__ dx, long long lddx) {
  pdl_wait();
  pdl_launch_dependents();
  const int oct = C / 8;
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= M * oct) return;
  const int o = (int)(idx % oct);
  const long long m = idx / oct;
  uint4 a = __ldg(reinterpret_cast<const uint4*>(x + m * ldx + o * 8));
  uint4 g = __ldg(reinterpret_cast<const uint4*>(dy + m * lddy + o * 8));
  uint32_t aw[4] = {a.x, a.y, a.z, a.w}, gw[4] = {g.x, g.y, g.z, g.w}, ow[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 f = unpack_bf16x2(aw[i]), d = unpack_bf16x2(gw[i]);
    ow[i] = pack_bf16x2(d.x * quick_gelu_grad(f.x), d.y * quick_gelu_grad(f.y));
  }
  *reinterpret_cast<uint4*>(dx + m * lddx + o * 8) = make_uint4(ow[0], ow[1], ow[2], ow[3]);
}

// gradient of the token-embedding rows `rows[r]` (the new-concept tokens, trainer_edlora.py:86-88: only those rows keep
// their update, train_edlora.py:133-136): out[r, c] (+)= sum over the positions m with ids[m] == rows[r] of dx[m, c].
// One block per row, fixed summation order (ascending m) -> bitwise reproducible.
__global__ void clip_embed_bwd_kernel(const int* __restrict__ ids, const __nv_bfloat16* __restrict__ dx, long long ld,
                                      long long M, int C, const int* __restrict__ rows, int accumulate,
                                      float* __restrict__ out) {
  pdl_wait();
  pdl_launch_dependents();
  const int tok = __ldg(rows + blockIdx.x);
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float acc = accumulate ? out[(long long)blockIdx.x * C + c] : 0.f;
    for (long long m = 0; m < M; ++m)
      if (__ldg(ids + m) == tok) acc += __bfloat162float(dx[m * ld + c]);
    out[(long long)blockIdx.x * C + c] = acc;
  }
}

// ---------------------------------------------------------------------------------- VAE glue (AutoencoderKL)
// Row softmax of fp32 logits (single-head d = 512 attention of the VAE mid block, computed as two wgmma GEMMs around this
// kernel): out[r, c] = softmax_c(scale * S[r, c]) for c < cols, as 16-bit.  One warp per row, two passes over the row
// (it is L2 resident: the producing GEMM has just written it).
template <bool F16>
__global__ void softmax_rows_kernel(const float* __restrict__ S, long long lds, long long rows, int cols, float scale_log2,
                                    __nv_bfloat16* __restrict__ out, long long ldo) {
  pdl_wait();
  pdl_launch_dependents();
  const long long r = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= rows) return;
  const float* row = S + r * lds;
  const int cols4 = cols & ~3;            // float4 body; the last cols % 4 columns (odd token counts) one at a time
  float m = -INFINITY;
  for (int c = lane * 4; c < cols4; c += 128) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(row + c));
    m = fmaxf(fmaxf(m, fmaxf(v.x, v.y)), fmaxf(v.z, v.w));
  }
  if (cols4 + lane < cols) m = fmaxf(m, __ldg(row + cols4 + lane));
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, d));
  const float mm = m * scale_log2;
  float sum = 0.f;
  for (int c = lane * 4; c < cols4; c += 128) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(row + c));
    sum += exp2f(v.x * scale_log2 - mm) + exp2f(v.y * scale_log2 - mm) + exp2f(v.z * scale_log2 - mm) +
           exp2f(v.w * scale_log2 - mm);
  }
  if (cols4 + lane < cols) sum += exp2f(__ldg(row + cols4 + lane) * scale_log2 - mm);
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, d);
  const float inv = 1.0f / sum;
  __nv_bfloat16* orow = out + r * ldo;
  for (int c = lane * 4; c < cols4; c += 128) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(row + c));
    uint2 o;
    o.x = pack16x2<F16>(exp2f(v.x * scale_log2 - mm) * inv, exp2f(v.y * scale_log2 - mm) * inv);
    o.y = pack16x2<F16>(exp2f(v.z * scale_log2 - mm) * inv, exp2f(v.w * scale_log2 - mm) * inv);
    *reinterpret_cast<uint2*>(orow + c) = o;
  }
  if (cols4 + lane < cols) {
    const float e = exp2f(__ldg(row + cols4 + lane) * scale_log2 - mm) * inv;
    reinterpret_cast<unsigned short*>(orow)[cols4 + lane] = (unsigned short)(pack16x2<F16>(e, 0.f) & 0xffffu);
  }
}

// out[b, o, p] = bias[o] + sum_c W[o, c] x[b, c, p]   (fp32 NCHW, <= 8 channels: post_quant_conv of the VAE decoder)
__global__ void conv1x1_nchw_kernel(const float* __restrict__ x, int B, int Cin, long long HW, const float* __restrict__ w,
                                    const float* __restrict__ bias, int Cout, float* __restrict__ y) {
  pdl_wait();
  pdl_launch_dependents();
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)B * HW) return;
  const int b = (int)(idx / HW);
  const long long p = idx - (long long)b * HW;
  float xv[8];
  for (int c = 0; c < Cin; ++c) xv[c] = __ldg(x + ((long long)b * Cin + c) * HW + p);
  for (int o = 0; o < Cout; ++o) {
    float acc = __ldg(bias + o);
    for (int c = 0; c < Cin; ++c) acc += __ldg(w + o * Cin + c) * xv[c];
    y[((long long)b * Cout + o) * HW + p] = acc;
  }
}

// Encoder tail: h = 16-bit NHWC [B*HW, ldh] holding the 2L "moments" channels of encoder.conv_out; quant_conv (1x1, 2L x 2L)
// is applied here, then mean / logvar (clamped to [-30, 20]) are written as fp32 NCHW [B, L, HW] and, when a standard
// normal draw `noise` is given, latents = scaling * (mean + exp(0.5 logvar) * noise)   (trainer_edlora.py:203-204).
template <bool F16>
__global__ void vae_moments_kernel(const __nv_bfloat16* __restrict__ h, long long ldh, int B, long long HW, int L,
                                   const float* __restrict__ w, const float* __restrict__ bias, float* __restrict__ mean,
                                   float* __restrict__ logvar, const float* __restrict__ noise, float scaling,
                                   float* __restrict__ latents) {
  pdl_wait();
  pdl_launch_dependents();
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)B * HW) return;
  const int b = (int)(idx / HW);
  const long long p = idx - (long long)b * HW;
  float xv[8], mo[8];
  for (int c = 0; c < 2 * L; ++c) xv[c] = ld16<F16>(h + idx * ldh + c);
  for (int o = 0; o < 2 * L; ++o) {
    float acc = __ldg(bias + o);
    for (int c = 0; c < 2 * L; ++c) acc += __ldg(w + o * 2 * L + c) * xv[c];
    mo[o] = acc;
  }
  for (int c = 0; c < L; ++c) {
    const float mu = mo[c], lv = fminf(fmaxf(mo[L + c], -30.0f), 20.0f);
    const long long off = ((long long)b * L + c) * HW + p;
    mean[off] = mu;
    logvar[off] = lv;
    if (noise != nullptr) latents[off] = scaling * (mu + __expf(0.5f * lv) * __ldg(noise + off));
  }
}

// ---------------------------------------------------------------------------------- CFG + DPM-Solver++(2M)
// eps = cfg ? u + g (c - u) : e ;  x0 = (x - sigma_s eps) / alpha_s ;  x <- c_x x + c_m0 x0 + c_m1 x0_prev ;
// x0_prev <- x0 ; unet_in (both CFG halves) <- x
__global__ void cfg_dpm_step_kernel(const float* __restrict__ noise_pred, float* __restrict__ latents,
                                    float* __restrict__ x0_prev, float* __restrict__ unet_in, long long n, int cfg,
                                    float guidance, float c_x, float c_m0, float c_m1, float alpha_s,
                                    float sigma_s, float* __restrict__ t_out, int t_count, float t_next) {
  pdl_wait();
  pdl_launch_dependents();
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t_out != nullptr && i < t_count) t_out[i] = t_next;  // timestep of the next UNet call
  if (i >= n) return;
  float eps;
  if (cfg) {
    float u = noise_pred[i], c = noise_pred[n + i];
    eps = u + guidance * (c - u);
  } else {
    eps = noise_pred[i];
  }
  float x = latents[i];
  float x0 = (x - sigma_s * eps) / alpha_s;
  float xn = c_x * x + c_m0 * x0 + c_m1 * x0_prev[i];
  latents[i] = xn;
  x0_prev[i] = x0;
  if (unet_in) {
    unet_in[i] = xn;
    if (cfg) unet_in[n + i] = xn;
  }
}

// ---------------------------------------------------------------------------------- region combine
// out = (count == 0) ? global : sum_{r covers pixel} region_r / count   (regional :54-83, replace_ratio 1)
struct RegionBoxes {
  int n;
  int box[8][4];  // sh, sw, eh, ew in feature pixels (host computes the ceil/floor in float64)
};
template <bool F16>
__global__ void region_combine_kernel(const __nv_bfloat16* __restrict__ glob, const __nv_bfloat16* const* __restrict__ regs,
                                      RegionBoxes rb, int B, int FH, int FW, int C, long long ld,
                                      __nv_bfloat16* __restrict__ out) {
  pdl_wait();
  pdl_launch_dependents();
  const int oct = C / 8;
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long total = (long long)B * FH * FW * oct;
  if (idx >= total) return;
  const int o = (int)(idx % oct);
  const long long pix = idx / oct;
  const int w = (int)(pix % FW), h = (int)((pix / FW) % FH);
  int count = 0;
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
  for (int r = 0; r < rb.n; ++r) {
    if (h >= rb.box[r][0] && h < rb.box[r][2] && w >= rb.box[r][1] && w < rb.box[r][3]) {
      ++count;
      uint4 u = __ldg(reinterpret_cast<const uint4*>(regs[r] + pix * ld + o * 8));
      uint32_t uw[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        float2 f = unpack16x2<F16>(uw[i]);
        acc[2 * i] += f.x;
        acc[2 * i + 1] += f.y;
      }
    }
  }
  uint4 res;
  if (count == 0) {
    res = __ldg(reinterpret_cast<const uint4*>(glob + pix * ld + o * 8));
  } else {
    float inv = 1.0f / (float)count;
    res.x = pack16x2<F16>(acc[0] * inv, acc[1] * inv);
    res.y = pack16x2<F16>(acc[2] * inv, acc[3] * inv);
    res.z = pack16x2<F16>(acc[4] * inv, acc[5] * inv);
    res.w = pack16x2<F16>(acc[6] * inv, acc[7] * inv);
  }
  *reinterpret_cast<uint4*>(out + pix * ld + o * 8) = res;
}

}  // namespace mos

using namespace mos;
#define STREAM(s) reinterpret_cast<cudaStream_t>(s)
static inline unsigned nblk(long long total, int threads) { return (unsigned)((total + threads - 1) / threads); }

extern "C" int mos_timestep_embedding(const float* t, int32_t B, int32_t dim, float* out, void* stream) {
  MOS_CHECK_ARG(t && out && B > 0 && dim % 2 == 0, "mos_timestep_embedding: bad arguments");
  MOS_CHECK_CUDA(launch_pdl(timestep_embed_kernel, dim3(B), dim3(160), 0, STREAM(stream), t, dim, out));
  return MOS_OK;
}

extern "C" int mos_gemv_bf16(const float* x, int32_t nb, int32_t K, const void* W, const float* bias, int32_t N,
                             int32_t act_in, int32_t act_out, float* out, int64_t ldo, void* stream) {
  MOS_CHECK_ARG(x && W && out && nb >= 1 && nb <= 8 && K % 8 == 0 && N > 0, "mos_gemv_bf16: bad arguments (nb=%d K=%d)",
                nb, K);
  const int warps = 8;
  dim3 grid(nblk(N, warps)), block(warps * 32);
  const __nv_bfloat16* w = reinterpret_cast<const __nv_bfloat16*>(W);
#define GEMV_CASE(NB)                                                                                   \
  case NB:                                                                                              \
    rc_ = launch_pdl(gemv_kernel<NB>, grid, block, 0, STREAM(stream), x, (int)K, w, bias, (int)N, (int)act_in, \
                     (int)act_out, out, (long long)ldo);                                        \
    break;
  cudaError_t rc_ = cudaSuccess;
  switch (nb) {
    GEMV_CASE(1) GEMV_CASE(2) GEMV_CASE(3) GEMV_CASE(4) GEMV_CASE(5) GEMV_CASE(6) GEMV_CASE(7) GEMV_CASE(8)
  }
#undef GEMV_CASE
  MOS_CHECK_CUDA(rc_);
  return MOS_OK;
}

extern "C" int mos_conv_in(const float* x, int32_t B, int32_t Cin, int32_t H, int32_t W, const float* w,
                           const float* bias, int32_t Cout, void* y, int64_t ldy, int32_t act_dtype, void* stream) {
  MOS_CHECK_ARG(x && w && bias && y && Cout % 8 == 0 && ldy % 8 == 0, "mos_conv_in: bad arguments");
  MOS_CHECK_DTYPE(act_dtype, "mos_conv_in");
  long long total = (long long)B * H * W * (Cout / 8);
  MOS_CHECK_CUDA(launch_pdl(act_dtype ? conv_in_kernel<true> : conv_in_kernel<false>, dim3(nblk(total, 256)), dim3(256), 0,
                            STREAM(stream), x, B, Cin, H, W, w, bias, Cout, reinterpret_cast<__nv_bfloat16*>(y), ldy));
  return MOS_OK;
}

extern "C" int mos_conv_out(const void* x, int32_t B, int32_t H, int32_t W, int32_t C, const float* w,
                            const float* bias, int32_t Cout, float* y, int32_t act_dtype, void* stream) {
  MOS_CHECK_ARG(x && w && bias && y && C % 8 == 0 && Cout <= 4, "mos_conv_out: bad arguments");
  MOS_CHECK_DTYPE(act_dtype, "mos_conv_out");
  long long pix = (long long)B * H * W;
  MOS_CHECK_CUDA(launch_pdl(act_dtype ? conv_out_kernel<true> : conv_out_kernel<false>, dim3(nblk(pix, 8)), dim3(256), 0,
                            STREAM(stream), reinterpret_cast<const __nv_bfloat16*>(x), B, H, W, C, w, bias, Cout, y));
  return MOS_OK;
}

extern "C" int mos_upsample2x(const void* x, int64_t ldx, int32_t B, int32_t H, int32_t W, int32_t C, void* y, int32_t Ho,
                              int32_t Wo, void* stream) {
  MOS_CHECK_ARG(x && y && C % 8 == 0 && ldx % 8 == 0 && H > 0 && W > 0 && Ho > 0 && Wo > 0, "mos_upsample2x: bad arguments");
  if (Ho == 2 * H && Wo == 2 * W) {
    long long total = (long long)B * 4 * H * W * (C / 8);
    MOS_CHECK_CUDA(launch_pdl(upsample2x_kernel, dim3(nblk(total, 256)), dim3(256), 0, STREAM(stream), reinterpret_cast<const __nv_bfloat16*>(x), ldx, B, H,
                                                                    W, C, reinterpret_cast<__nv_bfloat16*>(y)));
    return MOS_OK;
  }
  long long total = (long long)B * Ho * Wo * (C / 8);
  MOS_CHECK_CUDA(launch_pdl(upsample_nearest_kernel, dim3(nblk(total, 256)), dim3(256), 0, STREAM(stream),
                            reinterpret_cast<const __nv_bfloat16*>(x), ldx, B, H, W, C, Ho, Wo,
                            reinterpret_cast<__nv_bfloat16*>(y)));
  return MOS_OK;
}

extern "C" int mos_im2col_s2(const void* x, int64_t ldx, int32_t B, int32_t H, int32_t W, int32_t C, int32_t pad, void* col,
                             void* stream) {
  MOS_CHECK_ARG(x && col && C % 8 == 0 && ldx % 8 == 0 && H > 0 && W > 0 && (pad == 1 || (pad == 0 && H % 2 == 0 && W % 2 == 0)),
                "mos_im2col_s2: bad arguments");
  long long total = (long long)B * ((H + pad) / 2) * ((W + pad) / 2) * 9 * (C / 8);
  MOS_CHECK_CUDA(launch_pdl(im2col_s2_kernel, dim3(nblk(total, 256)), dim3(256), 0, STREAM(stream), reinterpret_cast<const __nv_bfloat16*>(x), ldx, B, H,
                                                                 W, C, (int)pad, reinterpret_cast<__nv_bfloat16*>(col)));
  return MOS_OK;
}

extern "C" int mos_add_rows(void* x, int64_t ldx, const void* r, int64_t ldr, int64_t M, int32_t C, int32_t act_dtype,
                            void* stream) {
  MOS_CHECK_ARG(x && r && C % 8 == 0 && ldx % 8 == 0 && ldr % 8 == 0, "mos_add_rows: bad arguments");
  MOS_CHECK_DTYPE(act_dtype, "mos_add_rows");
  MOS_CHECK_CUDA(launch_pdl(act_dtype ? add_rows_kernel<true> : add_rows_kernel<false>, dim3(nblk(M * (C / 8), 256)), dim3(256), 0, STREAM(stream),
                            reinterpret_cast<__nv_bfloat16*>(x), (long long)ldx,
                            reinterpret_cast<const __nv_bfloat16*>(r), (long long)ldr, (long long)M, (int)C));
  return MOS_OK;
}

extern "C" int mos_clip_embed(const int32_t* ids, const float* token_embedding, const float* position_embedding, int64_t M,
                              int32_t T, int32_t C, int32_t vocab, void* x, int64_t ld, void* stream) {
  MOS_CHECK_ARG(ids && token_embedding && position_embedding && x && M > 0 && T > 0 && vocab > 0,
                "mos_clip_embed: bad arguments");
  MOS_CHECK_ARG(C % 8 == 0 && ld % 8 == 0 && ld >= C, "mos_clip_embed: C=%d ld=%lld must be multiples of 8, ld >= C", C,
                (long long)ld);
  MOS_CHECK_CUDA(launch_pdl(clip_embed_kernel, dim3(nblk(M * (ld / 8), 256)), dim3(256), 0, STREAM(stream),
                            reinterpret_cast<const int*>(ids), token_embedding, position_embedding, (long long)M, (int)T,
                            (int)C, (int)vocab, reinterpret_cast<__nv_bfloat16*>(x), (long long)ld));
  return MOS_OK;
}

extern "C" int mos_quick_gelu(void* x, int64_t ld, int64_t M, int32_t C, void* stream) {
  MOS_CHECK_ARG(x && M > 0 && C % 8 == 0 && ld % 8 == 0 && ld >= C, "mos_quick_gelu: bad arguments");
  MOS_CHECK_CUDA(launch_pdl(quick_gelu_kernel, dim3(nblk(M * (C / 8), 256)), dim3(256), 0, STREAM(stream),
                            reinterpret_cast<__nv_bfloat16*>(x), (long long)ld, (long long)M, (int)C));
  return MOS_OK;
}

extern "C" int mos_quick_gelu_fwd(const void* x, int64_t ldx, int64_t M, int32_t C, void* y, int64_t ldy, void* stream) {
  MOS_CHECK_ARG(x && y && M > 0 && C % 8 == 0 && ldx % 8 == 0 && ldy % 8 == 0 && ldx >= C && ldy >= C,
                "mos_quick_gelu_fwd: bad arguments");
  MOS_CHECK_CUDA(launch_pdl(quick_gelu_fwd_kernel, dim3(nblk(M * (C / 8), 256)), dim3(256), 0, STREAM(stream),
                            reinterpret_cast<const __nv_bfloat16*>(x), (long long)ldx, (long long)M, (int)C,
                            reinterpret_cast<__nv_bfloat16*>(y), (long long)ldy));
  return MOS_OK;
}

extern "C" int mos_quick_gelu_bwd(const void* x, int64_t ldx, const void* dy, int64_t lddy, int64_t M, int32_t C, void* dx,
                                  int64_t lddx, void* stream) {
  MOS_CHECK_ARG(x && dy && dx && M > 0 && C % 8 == 0 && ldx % 8 == 0 && lddy % 8 == 0 && lddx % 8 == 0,
                "mos_quick_gelu_bwd: bad arguments");
  MOS_CHECK_CUDA(launch_pdl(quick_gelu_bwd_kernel, dim3(nblk(M * (C / 8), 256)), dim3(256), 0, STREAM(stream),
                            reinterpret_cast<const __nv_bfloat16*>(x), (long long)ldx,
                            reinterpret_cast<const __nv_bfloat16*>(dy), (long long)lddy, (long long)M, (int)C,
                            reinterpret_cast<__nv_bfloat16*>(dx), (long long)lddx));
  return MOS_OK;
}

extern "C" int mos_clip_embed_bwd(const int32_t* ids, const void* dx, int64_t ld, int64_t M, int32_t C, const int32_t* rows,
                                  int32_t n_rows, int32_t accumulate, float* out, void* stream) {
  MOS_CHECK_ARG(ids && dx && rows && out && M > 0 && C > 0 && n_rows > 0 && ld >= C, "mos_clip_embed_bwd: bad arguments");
  MOS_CHECK_CUDA(launch_pdl(clip_embed_bwd_kernel, dim3((unsigned)n_rows), dim3(256), 0, STREAM(stream),
                            reinterpret_cast<const int*>(ids), reinterpret_cast<const __nv_bfloat16*>(dx), (long long)ld,
                            (long long)M, (int)C, reinterpret_cast<const int*>(rows), (int)accumulate, out));
  return MOS_OK;
}

extern "C" int mos_softmax_rows(const float* S, int64_t lds, int64_t rows, int32_t cols, float scale, void* out, int64_t ldo,
                                int32_t act_dtype, void* stream) {
  MOS_CHECK_ARG(S && out && rows > 0 && cols > 0 && lds % 4 == 0 && lds >= cols && ldo % 4 == 0 && ldo >= cols,
                "mos_softmax_rows: bad arguments (lds, ldo must be multiples of 4)");
  MOS_CHECK_DTYPE(act_dtype, "mos_softmax_rows");
  const int warps = 8;
  MOS_CHECK_CUDA(launch_pdl(act_dtype ? softmax_rows_kernel<true> : softmax_rows_kernel<false>, dim3(nblk(rows, warps)),
                            dim3(warps * 32), 0, STREAM(stream), S, (long long)lds, (long long)rows, (int)cols,
                            scale * 1.4426950408889634f, reinterpret_cast<__nv_bfloat16*>(out), (long long)ldo));
  return MOS_OK;
}

extern "C" int mos_conv1x1_nchw(const float* x, int32_t B, int32_t Cin, int64_t HW, const float* w, const float* bias,
                                int32_t Cout, float* y, void* stream) {
  MOS_CHECK_ARG(x && w && bias && y && B > 0 && HW > 0 && Cin >= 1 && Cin <= 8 && Cout >= 1 && Cout <= 8,
                "mos_conv1x1_nchw: bad arguments (at most 8 channels)");
  MOS_CHECK_CUDA(launch_pdl(conv1x1_nchw_kernel, dim3(nblk((long long)B * HW, 256)), dim3(256), 0, STREAM(stream), x, (int)B,
                            (int)Cin, (long long)HW, w, bias, (int)Cout, y));
  return MOS_OK;
}

extern "C" int mos_vae_moments(const void* h, int64_t ldh, int32_t B, int64_t HW, int32_t L, const float* w, const float* bias,
                               float* mean, float* logvar, const float* noise, float scaling, float* latents,
                               int32_t act_dtype, void* stream) {
  MOS_CHECK_ARG(h && w && bias && mean && logvar && B > 0 && HW > 0 && L >= 1 && L <= 4 && ldh >= 2 * L && (!noise == !latents),
                "mos_vae_moments: bad arguments");
  MOS_CHECK_DTYPE(act_dtype, "mos_vae_moments");
  MOS_CHECK_CUDA(launch_pdl(act_dtype ? vae_moments_kernel<true> : vae_moments_kernel<false>,
                            dim3(nblk((long long)B * HW, 256)), dim3(256), 0, STREAM(stream),
                            reinterpret_cast<const __nv_bfloat16*>(h), (long long)ldh, (int)B, (long long)HW, (int)L, w, bias,
                            mean, logvar, noise, scaling, latents));
  return MOS_OK;
}

extern "C" int mos_cfg_dpmpp_step(const float* noise_pred, float* latents, float* x0_prev, float* unet_in, int64_t n,
                                  int32_t cfg, float guidance, float c_x, float c_m0, float c_m1, float alpha_s,
                                  float sigma_s, float* t_out, int32_t t_count, float t_next, void* stream) {
  MOS_CHECK_ARG(noise_pred && latents && x0_prev && n > 0, "mos_cfg_dpmpp_step: bad arguments");
  MOS_CHECK_CUDA(launch_pdl(cfg_dpm_step_kernel, dim3(nblk(n, 256)), dim3(256), 0, STREAM(stream), noise_pred, latents, x0_prev, unet_in, n, cfg, guidance,
                                                                c_x, c_m0, c_m1, alpha_s, sigma_s, t_out, t_count, t_next));
  return MOS_OK;
}

extern "C" int mos_region_combine(const void* glob, const void* const* region_ptrs_dev, int32_t nregions,
                                  const int32_t* boxes_host, int32_t B, int32_t FH, int32_t FW, int32_t C, int64_t ld,
                                  void* out, int32_t act_dtype, void* stream) {
  MOS_CHECK_ARG(glob && out && region_ptrs_dev && boxes_host && nregions >= 0 && nregions <= 8 && C % 8 == 0,
                "mos_region_combine: bad arguments (at most 8 regions)");
  MOS_CHECK_DTYPE(act_dtype, "mos_region_combine");
  RegionBoxes rb;
  rb.n = nregions;
  for (int r = 0; r < nregions; ++r)
    for (int k = 0; k < 4; ++k) rb.box[r][k] = boxes_host[r * 4 + k];
  long long total = (long long)B * FH * FW * (C / 8);
  MOS_CHECK_CUDA(launch_pdl(act_dtype ? region_combine_kernel<true> : region_combine_kernel<false>, dim3(nblk(total, 256)),
                            dim3(256), 0, STREAM(stream),
      reinterpret_cast<const __nv_bfloat16*>(glob), reinterpret_cast<const __nv_bfloat16* const*>(region_ptrs_dev), rb,
      B, FH, FW, C, ld, reinterpret_cast<__nv_bfloat16*>(out)));
  return MOS_OK;
}
