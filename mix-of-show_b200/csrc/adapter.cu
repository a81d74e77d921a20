// adapter.cu — the layout and elementwise kernels of the T2I-Adapter (diffusers `T2IAdapter`, adapter_type 'full_adapter',
// run once per image at reference pipeline_regionally_t2iadapter.py:474-482).  Its convolutions are mos_gemm_bf16 launches
// (3x3 implicit conv, 1x1 plain GEMM, the resnet add as the residual epilogue); these kernels supply what lies between:
//   PixelUnshuffle(8) of the fp32 NCHW condition image into the 16-bit NHWC rows of conv_in's A operand,
//   ReLU in place between block1 and block2 of every AdapterResnetBlock,
//   AvgPool2d(2, 2) at the start of every level after the first.
#include "common.h"
#include "tc.cuh"

namespace mos {

// y[(b, h, w), c*64 + i*8 + j] = x[b, c, 8h + i, 8w + j]; one thread per (pixel, c, i): 8 contiguous floats -> one 16 B store
template <bool F16>
__global__ void pixel_unshuffle_kernel(const float* __restrict__ x, int B, int Cin, int H, int W,
                                       __nv_bfloat16* __restrict__ y, long long ldy) {
  pdl_wait();
  pdl_launch_dependents();
  const int Ho = H / 8, Wo = W / 8, rows = Cin * 8;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)B * Ho * Wo * rows) return;
  const int r = (int)(idx % rows);                    // r = c * 8 + i
  const long long pix = idx / rows;
  const int wo = (int)(pix % Wo);
  const int ho = (int)((pix / Wo) % Ho);
  const int b = (int)(pix / ((long long)Wo * Ho));
  const int c = r / 8, i = r % 8;
  const float* src = x + (((long long)b * Cin + c) * H + 8 * ho + i) * W + 8 * wo;
  const float4 v0 = __ldg(reinterpret_cast<const float4*>(src));
  const float4 v1 = __ldg(reinterpret_cast<const float4*>(src + 4));
  uint4 u;
  u.x = pack16x2<F16>(v0.x, v0.y);
  u.y = pack16x2<F16>(v0.z, v0.w);
  u.z = pack16x2<F16>(v1.x, v1.y);
  u.w = pack16x2<F16>(v1.z, v1.w);
  *reinterpret_cast<uint4*>(y + pix * ldy + r * 8) = u;
}

// x[m, :C] <- (x < 0 ? 0 : x): NaN passes through, as F.relu
template <bool F16>
__global__ void relu_rows_kernel(__nv_bfloat16* __restrict__ x, long long ld, long long M, int C) {
  pdl_wait();
  pdl_launch_dependents();
  const int oct = C / 8;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= M * oct) return;
  const int o = (int)(idx % oct);
  const long long m = idx / oct;
  uint4 a = *reinterpret_cast<const uint4*>(x + m * ld + o * 8);
  uint32_t aw[4] = {a.x, a.y, a.z, a.w}, ow[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float2 f = unpack16x2<F16>(aw[k]);
    ow[k] = pack16x2<F16>(f.x < 0.f ? 0.f : f.x, f.y < 0.f ? 0.f : f.y);
  }
  *reinterpret_cast<uint4*>(x + m * ld + o * 8) = make_uint4(ow[0], ow[1], ow[2], ow[3]);
}

// y[b, ho, wo, :] = 0.25 * (x[b, 2ho, 2wo] + x[b, 2ho, 2wo+1] + x[b, 2ho+1, 2wo] + x[b, 2ho+1, 2wo+1])  (fp32 sum, one
// rounding to 16 bits; H and W even, so AvgPool2d(2) with and without ceil_mode agree)
template <bool F16>
__global__ void avgpool2x_kernel(const __nv_bfloat16* __restrict__ x, long long ldx, int B, int H, int W, int C,
                                 __nv_bfloat16* __restrict__ y, long long ldy) {
  pdl_wait();
  pdl_launch_dependents();
  const int oct = C / 8, Ho = H / 2, Wo = W / 2;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)B * Ho * Wo * oct) return;
  const int o = (int)(idx % oct);
  const long long pix = idx / oct;
  const int wo = (int)(pix % Wo);
  const int ho = (int)((pix / Wo) % Ho);
  const int b = (int)(pix / ((long long)Wo * Ho));
  float acc[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) acc[k] = 0.f;
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const long long p = ((long long)b * H + 2 * ho + t / 2) * W + 2 * wo + t % 2;
    const uint4 u = __ldg(reinterpret_cast<const uint4*>(x + p * ldx + o * 8));
    const uint32_t uw[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 f = unpack16x2<F16>(uw[k]);
      acc[2 * k] += f.x;
      acc[2 * k + 1] += f.y;
    }
  }
  uint4 r;
  r.x = pack16x2<F16>(0.25f * acc[0], 0.25f * acc[1]);
  r.y = pack16x2<F16>(0.25f * acc[2], 0.25f * acc[3]);
  r.z = pack16x2<F16>(0.25f * acc[4], 0.25f * acc[5]);
  r.w = pack16x2<F16>(0.25f * acc[6], 0.25f * acc[7]);
  *reinterpret_cast<uint4*>(y + pix * ldy + o * 8) = r;
}

}  // namespace mos

using namespace mos;
#define STREAM(s) reinterpret_cast<cudaStream_t>(s)
static inline unsigned nblk(long long total, int threads) { return (unsigned)((total + threads - 1) / threads); }

extern "C" int mos_pixel_unshuffle(const float* x, int32_t B, int32_t Cin, int32_t H, int32_t W, void* y, int64_t ldy,
                                   int32_t act_dtype, void* stream) {
  MOS_CHECK_ARG(x && y && B > 0 && Cin > 0 && H > 0 && W > 0, "mos_pixel_unshuffle: bad arguments");
  MOS_CHECK_ARG(H % 8 == 0 && W % 8 == 0 && ldy % 8 == 0 && ldy >= 64LL * Cin,
                "mos_pixel_unshuffle: H=%d W=%d must be multiples of 8, ldy=%lld a multiple of 8 and >= 64 Cin", H, W,
                (long long)ldy);
  MOS_CHECK_DTYPE(act_dtype, "mos_pixel_unshuffle");
  const long long total = (long long)B * (H / 8) * (W / 8) * Cin * 8;
  MOS_CHECK_CUDA(launch_pdl(act_dtype ? pixel_unshuffle_kernel<true> : pixel_unshuffle_kernel<false>,
                            dim3(nblk(total, 256)), dim3(256), 0, STREAM(stream), x, (int)B, (int)Cin, (int)H, (int)W,
                            reinterpret_cast<__nv_bfloat16*>(y), (long long)ldy));
  return MOS_OK;
}

extern "C" int mos_relu_rows(void* x, int64_t ld, int64_t M, int32_t C, int32_t act_dtype, void* stream) {
  MOS_CHECK_ARG(x && M > 0 && C > 0 && C % 8 == 0 && ld % 8 == 0 && ld >= C,
                "mos_relu_rows: bad arguments (C=%d ld=%lld: multiples of 8, ld >= C)", C, (long long)ld);
  MOS_CHECK_DTYPE(act_dtype, "mos_relu_rows");
  MOS_CHECK_CUDA(launch_pdl(act_dtype ? relu_rows_kernel<true> : relu_rows_kernel<false>, dim3(nblk(M * (C / 8), 256)),
                            dim3(256), 0, STREAM(stream), reinterpret_cast<__nv_bfloat16*>(x), (long long)ld,
                            (long long)M, (int)C));
  return MOS_OK;
}

extern "C" int mos_avgpool2x(const void* x, int64_t ldx, int32_t B, int32_t H, int32_t W, int32_t C, void* y, int64_t ldy,
                             int32_t act_dtype, void* stream) {
  MOS_CHECK_ARG(x && y && B > 0 && H > 0 && W > 0 && C > 0, "mos_avgpool2x: bad arguments");
  MOS_CHECK_ARG(H % 2 == 0 && W % 2 == 0 && C % 8 == 0 && ldx % 8 == 0 && ldy % 8 == 0 && ldx >= C && ldy >= C,
                "mos_avgpool2x: H=%d W=%d must be even, C=%d ldx=%lld ldy=%lld multiples of 8 and >= C", H, W, C,
                (long long)ldx, (long long)ldy);
  MOS_CHECK_DTYPE(act_dtype, "mos_avgpool2x");
  const long long total = (long long)B * (H / 2) * (W / 2) * (C / 8);
  MOS_CHECK_CUDA(launch_pdl(act_dtype ? avgpool2x_kernel<true> : avgpool2x_kernel<false>, dim3(nblk(total, 256)), dim3(256),
                            0, STREAM(stream), reinterpret_cast<const __nv_bfloat16*>(x), (long long)ldx, (int)B, (int)H,
                            (int)W, (int)C, reinterpret_cast<__nv_bfloat16*>(y), (long long)ldy));
  return MOS_OK;
}
