// fusion.cu — K7/K8: kernels of gradient fusion (gradient_fusion.py) in Gram form.
//
// The reference solves, per layer,  min_W mean((X W^T - V)^2)  with V = X W_c^T recorded per concept c
// (gradient_fusion.py:38-96, 394-429, 700-740) by L-BFGS, streaming X and V (GBs) from host memory on every closure
// call.  Because V_c = X_c W_c^T exactly (bias removed, gradient_fusion.py:155-160), the objective only depends on the
// per-concept Gram matrices  G_c = X_c^T X_c:
//     f(W) = s * sum_c tr((W - W_c) G_c (W - W_c)^T),   s = 1 / (n * out)
//     grad = 2 s (W G - C),  G = sum_c G_c,  C = sum_c W_c G_c,   f = s (<W, W G - 2 C> + vv),  vv = sum_c <W_c, W_c G_c>
// so features are reduced to [in, in] fp32 on the fly (wgmma GEMM with fp32 accumulate output, see gemm.cu) and a
// closure is one [out, in] x [in, in] fp32 GEMM.  Kernels here: bf16 transpose (Gram operand), small-n Gram, fp32
// SGEMM, closure epilogue (grad + loss), deterministic vector primitives for the L-BFGS driver, batched LoRA merge.
#include <stdlib.h>

#include "common.h"
#include "tc.cuh"

namespace mos {

// ------------------------------------------------------------------ bf16 transpose: x [rows, ldx](C cols) -> out [C, ldo]
__global__ void transpose_bf16_kernel(const __nv_bfloat16* __restrict__ x, long long ldx, int rows, int C,
                                      __nv_bfloat16* __restrict__ out, long long ldo) {
  __shared__ __nv_bfloat16 tile[32][34];
  pdl_wait();
  pdl_launch_dependents();
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int r = r0 + i, c = c0 + threadIdx.x;
    tile[i][threadIdx.x] = (r < rows && c < C) ? x[(long long)r * ldx + c] : __float2bfloat16(0.f);
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, r = r0 + threadIdx.x;
    if (c < C && r < rows) out[(long long)c * ldo + r] = tile[threadIdx.x][i];
  }
}

// ------------------------------------------------------------------ small-n A^T B: G[i][j] (+)= sum_r X[r][i] Y[r][j]
__global__ void atb_small_kernel(const float* __restrict__ X, const float* __restrict__ Y, int n, int dx, int dy,
                                 float* __restrict__ G, int accumulate) {
  __shared__ float xi[16][17], xj[16][17];
  const int i0 = blockIdx.y * 16, j0 = blockIdx.x * 16;
  float acc = 0.f;
  for (int r0 = 0; r0 < n; r0 += 16) {
    const int r = r0 + threadIdx.y;
    xi[threadIdx.y][threadIdx.x] = (r < n && i0 + threadIdx.x < dx) ? X[(long long)r * dx + i0 + threadIdx.x] : 0.f;
    xj[threadIdx.y][threadIdx.x] = (r < n && j0 + threadIdx.x < dy) ? Y[(long long)r * dy + j0 + threadIdx.x] : 0.f;
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 16; ++k) acc += xi[k][threadIdx.y] * xj[k][threadIdx.x];
    __syncthreads();
  }
  const int i = i0 + threadIdx.y, j = j0 + threadIdx.x;
  if (i < dx && j < dy) G[(long long)i * dy + j] = (accumulate ? G[(long long)i * dy + j] : 0.f) + acc;
}

// ------------------------------------------------------------------ fp32 SGEMM  C = alpha * A[M,K] * B[K,N] + beta * C
// 64x64 tile, 256 threads, 4x4 micro-tile, K step 16 (CUDA cores: exact fp32 for the closure of the solver)
__global__ void __launch_bounds__(256)
sgemm_nn_kernel(const float* __restrict__ A, const float* __restrict__ B, float* __restrict__ C, int M, int N, int K,
                float alpha, float beta) {
  __shared__ float As[16][64 + 4], Bs[16][64 + 4];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int k0 = 0; k0 < K; k0 += 16) {
    for (int i = threadIdx.x; i < 64 * 16; i += 256) {
      const int m = i >> 4, k = i & 15;   // A tile [64][16]
      As[k][m] = (m0 + m < M && k0 + k < K) ? A[(long long)(m0 + m) * K + k0 + k] : 0.f;
      const int kk = i >> 6, n = i & 63;  // B tile [16][64]
      Bs[kk][n] = (k0 + kk < K && n0 + n < N) ? B[(long long)(k0 + kk) * N + n0 + n] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = As[k][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = Bs[k][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n < N) {
        float* c = C + (long long)m * N + n;
        *c = alpha * acc[i][j] + (beta != 0.f ? beta * *c : 0.f);
      }
    }
  }
}

// ------------------------------------------------------------------ closure GEMM in fp64: Y[M,N] = A[M,K] (fp32) * B[K,N] (fp64)
// The Gram form squares the condition number of the least-squares problem; the product D G must therefore be carried
// in fp64 for the solver to reach the residual the reference reaches with its direct fp32 MSE (measured: 2e-5 vs
// 6e-7 relative residual on an exactly solvable problem with an fp32 product).  <= 4.2 GFLOP per closure.
template <int TM, int TN>   // CTA tile TM x TN (TM / 16 x TN / 16 outputs per thread): 32 x 64, 64 x 64 or 64 x 128
__global__ void __launch_bounds__(256, (TN > 64 ? 1 : 2))
dgemm_mixed_kernel(const float* __restrict__ A, const double* __restrict__ B, double* __restrict__ C, int M, int N,
                   int K) {
  // every output element accumulates fma(a, b, acc) over k ascending, whatever the tiling: results do not depend on the tile.
  // Global loads of k-tile t + 1 are issued before the products of tile t (register prefetch, double-buffered smem); 32-deep
  // k-tiles keep the DFMA pipe fed across the L2 round trip; thread tx owns columns tx, tx + 16, ... (bank-conflict free).
  constexpr int DK = 32;
  constexpr int RI = TM / 16, RJ = TN / 16;
  constexpr int AL = TM * DK / 256;           // A elements per thread and k-tile
  constexpr int BL = TN * DK / 256;           // B elements per thread and k-tile
  extern __shared__ __align__(16) unsigned char dsm[];
  double(*As)[DK][TM + 2] = reinterpret_cast<double(*)[DK][TM + 2]>(dsm);
  double(*Bs)[DK][TN + 2] = reinterpret_cast<double(*)[DK][TN + 2]>(dsm + sizeof(double) * 2 * DK * (TM + 2));
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int m0 = blockIdx.y * TM, n0 = blockIdx.x * TN;
  double acc[RI][RJ];
#pragma unroll
  for (int i = 0; i < RI; ++i)
#pragma unroll
    for (int j = 0; j < RJ; ++j) acc[i][j] = 0.0;
  float ra[AL];
  double rb[BL];
  auto gload = [&](int k0) {
#pragma unroll
    for (int u = 0; u < AL; ++u) {
      const int i = threadIdx.x + u * 256;
      const int m = i / DK, k = i % DK;
      ra[u] = (m0 + m < M && k0 + k < K) ? __ldg(A + (long long)(m0 + m) * K + k0 + k) : 0.f;
    }
#pragma unroll
    for (int u = 0; u < BL; ++u) {
      const int i = threadIdx.x + u * 256;
      const int kk = i / TN, n = i % TN;
      rb[u] = (k0 + kk < K && n0 + n < N) ? __ldg(B + (long long)(k0 + kk) * N + n0 + n) : 0.0;
    }
  };
  auto sstore = [&](int buf) {
#pragma unroll
    for (int u = 0; u < AL; ++u) {
      const int i = threadIdx.x + u * 256;
      As[buf][i % DK][i / DK] = (double)ra[u];
    }
#pragma unroll
    for (int u = 0; u < BL; ++u) {
      const int i = threadIdx.x + u * 256;
      Bs[buf][i / TN][i % TN] = rb[u];
    }
  };
  gload(0);
  sstore(0);
  __syncthreads();
  int buf = 0;
  for (int k0 = 0; k0 < K; k0 += DK) {
    const bool more = k0 + DK < K;
    if (more) gload(k0 + DK);
#pragma unroll 8
    for (int k = 0; k < DK; ++k) {
      double a[RI], b[RJ];
#pragma unroll
      for (int i = 0; i < RI; ++i) a[i] = As[buf][k][ty * RI + i];
#pragma unroll
      for (int j = 0; j < RJ; ++j) b[j] = Bs[buf][k][tx + 16 * j];
#pragma unroll
      for (int i = 0; i < RI; ++i)
#pragma unroll
        for (int j = 0; j < RJ; ++j) acc[i][j] = fma(a[i], b[j], acc[i][j]);
    }
    if (more) sstore(buf ^ 1);
    __syncthreads();
    buf ^= 1;
  }
#pragma unroll
  for (int i = 0; i < RI; ++i) {
    const int m = m0 + ty * RI + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < RJ; ++j) {
      const int n = n0 + tx + 16 * j;
      if (n < N) C[(long long)m * N + n] = acc[i][j];
    }
  }
}

// ------------------------------------------------------------------ deterministic block reductions
// max that propagates NaN (fmaxf drops it): a NaN gradient must not pass the solver's convergence tests, as with torch's
// abs().max()
__device__ __forceinline__ float nan_max(float a, float b) { return (a > b || a != a) ? a : b; }
__device__ __forceinline__ float block_sum(float v, float* sh) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = 0.f;
  if (threadIdx.x < 32) {
    r = threadIdx.x < (blockDim.x >> 5) ? sh[threadIdx.x] : 0.f;
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) r += __shfl_xor_sync(0xffffffffu, r, d);
  }
  __syncthreads();
  return r;   // valid in thread 0
}
__device__ __forceinline__ float block_max(float v, float* sh) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v = nan_max(v, __shfl_xor_sync(0xffffffffu, v, d));
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = 0.f;
  if (threadIdx.x < 32) {
    r = threadIdx.x < (blockDim.x >> 5) ? sh[threadIdx.x] : 0.f;
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) r = nan_max(r, __shfl_xor_sync(0xffffffffu, r, d));
  }
  __syncthreads();
  return r;
}

constexpr int RED_BLOCKS = 256;   // fixed grid -> fixed summation order -> bitwise reproducible scalars

// closure epilogue: grad = 2 s (Y - C);  partial[b] = sum W .* (Y - 2 C), accumulated in fp64: near the optimum the
// loss is a 1e-7-relative difference of O(1) terms and the line search needs its sign right
__global__ void ls_grad_loss_kernel(const float* __restrict__ W, const double* __restrict__ Y,
                                    const double* __restrict__ Cm, long long n, double s, float* __restrict__ grad,
                                    double* __restrict__ partial) {
  __shared__ double shd[256];
  double acc = 0.0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const double y = Y[i], c = Cm[i], w = (double)W[i];
    grad[i] = (float)(2.0 * s * (y - c));
    acc += w * (y - 2.0 * c);
  }
  shd[threadIdx.x] = acc;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) shd[threadIdx.x] += shd[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) partial[blockIdx.x] = shd[0];
}
// loss[0] (double) = s * sum(partial) + f0
__global__ void ls_loss_finalize_kernel(const double* __restrict__ partial, int nb, double s, double f0,
                                        double* __restrict__ loss) {
  __shared__ double shd[256];
  double v = 0.0;
  for (int i = threadIdx.x; i < nb; i += blockDim.x) v += partial[i];
  shd[threadIdx.x] = v;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) shd[threadIdx.x] += shd[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) loss[0] = s * shd[0] + f0;
}
// out[0] = scale * sum(partial) + add   (add applied after the scaling: keeps a large constant from swamping the sum)
__global__ void reduce_partials_kernel(const float* __restrict__ partial, int nb, float scale, float add, int is_max,
                                       float* __restrict__ out) {
  __shared__ float sh[32];
  float v = 0.f;
  for (int i = threadIdx.x; i < nb; i += blockDim.x) v = is_max ? nan_max(v, partial[i]) : v + partial[i];
  const float t = is_max ? block_max(v, sh) : block_sum(v, sh);
  if (threadIdx.x == 0) out[0] = is_max ? t : scale * t + add;
}
__global__ void vec_dot_kernel(const float* __restrict__ a, const float* __restrict__ b, long long n,
                               float* __restrict__ partial) {
  __shared__ float sh[32];
  float acc = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    acc += a[i] * b[i];
  const float t = block_sum(acc, sh);
  if (threadIdx.x == 0) partial[blockIdx.x] = t;
}
__global__ void vec_asum_kernel(const float* __restrict__ a, long long n, float* __restrict__ partial) {
  __shared__ float sh[32];
  float acc = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    acc += fabsf(a[i]);
  const float t = block_sum(acc, sh);
  if (threadIdx.x == 0) partial[blockIdx.x] = t;
}
__global__ void vec_absmax_kernel(const float* __restrict__ a, long long n, float scale, float* __restrict__ partial) {
  __shared__ float sh[32];
  float acc = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    acc = nan_max(acc, fabsf(a[i] * scale));
  const float t = block_max(acc, sh);
  if (threadIdx.x == 0) partial[blockIdx.x] = t;
}
// y = alpha * x + beta * y   (beta = 0: plain scaled copy, y may be uninitialised)
__global__ void vec_axpby_kernel(float* __restrict__ y, const float* __restrict__ x, float alpha, float beta,
                                 long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    y[i] = alpha * x[i] + (beta != 0.f ? beta * y[i] : 0.f);
}

// ------------------------------------------------------------------ L-BFGS two-loop recursion without host round trips
// One launch per history pair and loop: v <- v + c * upd (c = the coefficient the PREVIOUS launch left in device memory), then
// the dot product of the updated v with the next history vector, reduced by the last-arriving block exactly like
// vec_dot_kernel + reduce_partials_kernel (same grid, same partial layout, same final tree), so the direction equals the
// host-driven recursion bit for bit.  mode 0: first loop (al_i = rho_i <s_i, q>, next coefficient -al_i); mode 1: second loop
// (be_i = rho_i <y_i, r>, next coefficient al_i - be_i); mode 2: final update, dot with g -> gtd.
struct LbfgsStep {
  float* v;               // q / r, updated in place
  const float* g;         // first step only: v = -g
  const float* upd;       // vector added with the incoming coefficient (NULL: none)
  const float* dotv;      // vector of the dot product
  long long n;
  double rho;             // rho_i of this step (modes 0, 1)
  float h_diag;           // applied after the update when scale != 0 (transition q -> r = H0 q)
  int first, scale, mode, idx;
  double* al;             // [k] device: al_i
  double* coef;           // [1] device: coefficient for the next launch
  float* partial;         // [RED_BLOCKS]
  unsigned* counter;      // [1], zero between launches
  float* gtd;             // mode 2: <g, d>
  // ring addressing (mos_lbfgs_direction_ring): the history lives in two rings of `slots` vectors; logical pair i sits in
  // physical slot (*head + i) % slots, rho / h_diag are read from device memory - the launch parameters of a direction are
  // then the same on every iteration with a full history, so the 2k + 1 launches can be replayed as one CUDA graph
  int ring, slots, upd_kind, upd_idx, dot_kind;   // kinds: 0 none, 1 = S ring, 2 = Y ring, 3 = g
  const float *ring_s, *ring_y;
  const int* head;
  const double* rho_dev;  // [slots], physical
  const float* hdiag_dev;
};
__global__ void __launch_bounds__(256) lbfgs_step_kernel(const LbfgsStep p) {
  __shared__ float sh[32];
  __shared__ int last;
  const float* upd = p.upd;
  const float* dotv = p.dotv;
  double rho = p.rho;
  float h_diag = p.h_diag;
  if (p.ring) {
    const int head = *p.head;
    auto slot = [&](int i) { return (head + i) % p.slots; };
    upd = p.upd_kind == 1 ? p.ring_s + (long long)slot(p.upd_idx) * p.n
          : p.upd_kind == 2 ? p.ring_y + (long long)slot(p.upd_idx) * p.n : nullptr;
    dotv = p.dot_kind == 1 ? p.ring_s + (long long)slot(p.idx) * p.n
           : p.dot_kind == 2 ? p.ring_y + (long long)slot(p.idx) * p.n : p.g;
    if (p.mode != 2) rho = p.rho_dev[slot(p.idx)];
    h_diag = *p.hdiag_dev;
  }
  const float c = (upd != nullptr) ? (float)(*p.coef) : 0.f;
  float acc = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < p.n; i += (long long)gridDim.x * blockDim.x) {
    float v = p.first ? -1.0f * p.g[i] : p.v[i];
    if (upd != nullptr) v = c * upd[i] + v;              // contracted to one fma, as vec_axpby_kernel's alpha * x + 1 * y
    if (p.scale) v = h_diag * v;
    p.v[i] = v;
    acc += dotv[i] * v;                                  // vec_dot_kernel's a[i] * b[i] with a = history vector
  }
  const float t = block_sum(acc, sh);
  if (threadIdx.x == 0) {
    p.partial[blockIdx.x] = t;
    __threadfence();
    last = (atomicAdd(p.counter, 1u) == gridDim.x - 1) ? 1 : 0;
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  float vsum = 0.f;
  for (int i = threadIdx.x; i < (int)gridDim.x; i += blockDim.x) vsum += __ldcg(p.partial + i);
  const float dot = block_sum(vsum, sh);
  if (threadIdx.x == 0) {
    const float d1 = 1.f * dot + 0.f;                    // reduce_partials_kernel: scale * t + add
    if (p.mode == 0) {
      const double al = (double)d1 * rho;
      p.al[p.idx] = al;
      *p.coef = -al;
    } else if (p.mode == 1) {
      const double be = (double)d1 * rho;
      *p.coef = p.al[p.idx] - be;
    } else {
      *p.gtd = d1;
    }
    *p.counter = 0u;
  }
}

// ------------------------------------------------------------------ batched LoRA merge: W_l += alpha * up_l @ down_l
// table[l] = {W ptr, down ptr, up ptr, out, in, rank}; W fp32 [out, in] (4-D 1x1 conv weights have the same layout)
__global__ void lora_merge_kernel(const long long* __restrict__ table, float alpha) {
  const long long* e = table + (long long)blockIdx.y * 6;
  float* W = reinterpret_cast<float*>(e[0]);
  const float* down = reinterpret_cast<const float*>(e[1]);
  const float* up = reinterpret_cast<const float*>(e[2]);
  const long long out = e[3], in = e[4];
  const int rank = (int)e[5];
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < out * in; i += (long long)gridDim.x * blockDim.x) {
    const long long o = i / in, c = i - o * in;
    float acc = 0.f;
    for (int r = 0; r < rank; ++r) acc += up[o * rank + r] * down[(long long)r * in + c];
    W[i] += alpha * acc;
  }
}

}  // namespace mos

using namespace mos;
#define STREAM(s) reinterpret_cast<cudaStream_t>(s)

extern "C" int mos_transpose_bf16(const void* x, int64_t ldx, int32_t rows, int32_t C, void* out, int64_t ldo,
                                  void* stream) {
  MOS_CHECK_ARG(x && out && rows > 0 && C > 0 && ldo >= rows, "mos_transpose_bf16: bad arguments");
  dim3 grid((unsigned)ceil_div(C, 32), (unsigned)ceil_div(rows, 32)), block(32, 8);
  MOS_CHECK_CUDA(launch_pdl(transpose_bf16_kernel, grid, block, 0, STREAM(stream),
                            reinterpret_cast<const __nv_bfloat16*>(x), (long long)ldx, (int)rows, (int)C,
                            reinterpret_cast<__nv_bfloat16*>(out), (long long)ldo));
  return MOS_OK;
}

extern "C" int mos_gram_small(const float* X, int32_t n, int32_t d, float* G, int32_t accumulate, void* stream) {
  MOS_CHECK_ARG(X && G && n > 0 && d > 0, "mos_gram_small: bad arguments");
  dim3 grid((unsigned)ceil_div(d, 16), (unsigned)ceil_div(d, 16)), block(16, 16);
  atb_small_kernel<<<grid, block, 0, STREAM(stream)>>>(X, X, n, d, d, G, accumulate);
  MOS_CHECK_LAUNCH();
  return MOS_OK;
}

// out [dx, dy] (+)= X^T Y for X [n, dx], Y [n, dy] fp32 (C = V^T K of update_quasi_newton's generic form)
extern "C" int mos_atb_small(const float* X, const float* Y, int32_t n, int32_t dx, int32_t dy, float* out,
                             int32_t accumulate, void* stream) {
  MOS_CHECK_ARG(X && Y && out && n > 0 && dx > 0 && dy > 0, "mos_atb_small: bad arguments");
  dim3 grid((unsigned)ceil_div(dy, 16), (unsigned)ceil_div(dx, 16)), block(16, 16);
  atb_small_kernel<<<grid, block, 0, STREAM(stream)>>>(X, Y, n, dx, dy, out, accumulate);
  MOS_CHECK_LAUNCH();
  return MOS_OK;
}

extern "C" int mos_sgemm_nn(const float* A, const float* B, float* C, int32_t M, int32_t N, int32_t K, float alpha,
                            float beta, void* stream) {
  MOS_CHECK_ARG(A && B && C && M > 0 && N > 0 && K > 0, "mos_sgemm_nn: bad arguments");
  dim3 grid((unsigned)ceil_div(N, 64), (unsigned)ceil_div(M, 64));
  sgemm_nn_kernel<<<grid, 256, 0, STREAM(stream)>>>(A, B, C, M, N, K, alpha, beta);
  MOS_CHECK_LAUNCH();
  return MOS_OK;
}

// grad (fp32) = 2 s (Y - C); loss[0] (fp64) = s * <W, Y - 2C> + f0; Y, C fp64.  scratch: >= 256 doubles.
extern "C" int mos_dgemm_mixed(const float* A, const double* B, double* C, int32_t M, int32_t N, int32_t K,
                               void* stream) {
  MOS_CHECK_ARG(A && B && C && M > 0 && N > 0 && K > 0, "mos_dgemm_mixed: bad arguments");
  constexpr int DK = 32;
  auto smem = [](int tm, int tn) { return sizeof(double) * 2 * DK * ((tm + 2) + (tn + 2)); };
  // one-time set-up, run once even when several host threads (mos_lbfgs_solve_batch) make their first call together:
  // a function-local static is initialised exactly once, and the other callers wait for it.  A failed
  // cudaFuncSetAttribute is kept with it: every later call then returns that error instead of retrying the set-up
  struct Setup {
    int tile;
    cudaError_t err;
  };
  static const Setup setup = [&] {
    const char* e = getenv("MOS_DGEMM_TILE");     // 0 = heuristic, 1 = 32 x 64, 2 = 64 x 64, 3 = 64 x 128 (benchmarking)
    Setup s{e ? atoi(e) : 0, cudaSuccess};
    cudaError_t r[3] = {
        cudaFuncSetAttribute(dgemm_mixed_kernel<32, 64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem(32, 64)),
        cudaFuncSetAttribute(dgemm_mixed_kernel<64, 64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem(64, 64)),
        cudaFuncSetAttribute(dgemm_mixed_kernel<64, 128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem(64, 128))};
    for (cudaError_t x : r)
      if (s.err == cudaSuccess) s.err = x;
    return s;
  }();
  MOS_CHECK_CUDA(setup.err);
  int tile = setup.tile;
  if (tile == 0) tile = 2;   // 64 x 64 by default
  if (tile == 1) {
    dim3 grid((unsigned)ceil_div(N, 64), (unsigned)ceil_div(M, 32));
    dgemm_mixed_kernel<32, 64><<<grid, 256, smem(32, 64), STREAM(stream)>>>(A, B, C, M, N, K);
  } else if (tile == 2) {
    dim3 grid((unsigned)ceil_div(N, 64), (unsigned)ceil_div(M, 64));
    dgemm_mixed_kernel<64, 64><<<grid, 256, smem(64, 64), STREAM(stream)>>>(A, B, C, M, N, K);
  } else {
    dim3 grid((unsigned)ceil_div(N, 128), (unsigned)ceil_div(M, 64));
    dgemm_mixed_kernel<64, 128><<<grid, 256, smem(64, 128), STREAM(stream)>>>(A, B, C, M, N, K);
  }
  MOS_CHECK_LAUNCH();
  return MOS_OK;
}

extern "C" int mos_ls_grad_loss(const float* W, const double* Y, const double* Cm, int64_t n, double s, double f0,
                                float* grad, double* loss, double* scratch, void* stream) {
  MOS_CHECK_ARG(W && Y && Cm && grad && loss && scratch && n > 0, "mos_ls_grad_loss: bad arguments");
  ls_grad_loss_kernel<<<RED_BLOCKS, 256, 0, STREAM(stream)>>>(W, Y, Cm, n, s, grad, scratch);
  MOS_CHECK_LAUNCH();
  ls_loss_finalize_kernel<<<1, 256, 0, STREAM(stream)>>>(scratch, RED_BLOCKS, s, f0, loss);
  MOS_CHECK_LAUNCH();
  return MOS_OK;
}

extern "C" int mos_vec_dot(const float* a, const float* b, int64_t n, float* out, float* scratch, void* stream) {
  MOS_CHECK_ARG(a && b && out && scratch && n > 0, "mos_vec_dot: bad arguments");
  vec_dot_kernel<<<RED_BLOCKS, 256, 0, STREAM(stream)>>>(a, b, n, scratch);
  MOS_CHECK_LAUNCH();
  reduce_partials_kernel<<<1, 256, 0, STREAM(stream)>>>(scratch, RED_BLOCKS, 1.f, 0.f, 0, out);
  MOS_CHECK_LAUNCH();
  return MOS_OK;
}

extern "C" int mos_vec_asum(const float* a, int64_t n, float* out, float* scratch, void* stream) {
  MOS_CHECK_ARG(a && out && scratch && n > 0, "mos_vec_asum: bad arguments");
  vec_asum_kernel<<<RED_BLOCKS, 256, 0, STREAM(stream)>>>(a, n, scratch);
  MOS_CHECK_LAUNCH();
  reduce_partials_kernel<<<1, 256, 0, STREAM(stream)>>>(scratch, RED_BLOCKS, 1.f, 0.f, 0, out);
  MOS_CHECK_LAUNCH();
  return MOS_OK;
}

extern "C" int mos_vec_absmax(const float* a, int64_t n, float scale, float* out, float* scratch, void* stream) {
  MOS_CHECK_ARG(a && out && scratch && n > 0, "mos_vec_absmax: bad arguments");
  vec_absmax_kernel<<<RED_BLOCKS, 256, 0, STREAM(stream)>>>(a, n, scale, scratch);
  MOS_CHECK_LAUNCH();
  reduce_partials_kernel<<<1, 256, 0, STREAM(stream)>>>(scratch, RED_BLOCKS, 1.f, 0.f, 1, out);
  MOS_CHECK_LAUNCH();
  return MOS_OK;
}

extern "C" int mos_vec_axpby(float* y, const float* x, float alpha, float beta, int64_t n, void* stream) {
  MOS_CHECK_ARG(y && x && n > 0, "mos_vec_axpby: bad arguments");
  long long blocks = ceil_div(n, 256 * 4);
  if (blocks > 1184) blocks = 1184;
  vec_axpby_kernel<<<(unsigned)blocks, 256, 0, STREAM(stream)>>>(y, x, alpha, beta, n);
  MOS_CHECK_LAUNCH();
  return MOS_OK;
}

// d = -H g by the two-loop recursion over k curvature pairs (S[i], Y[i] host arrays of device pointers, oldest first; rho[i] =
// 1 / <y_i, s_i> and h_diag host values) and gtd[0] = <g, d>; 2k + 1 launches, no host synchronisation.
// work: >= k + 1 doubles, partial: >= 257 floats (device scratch; partial[256] is the block counter and must be zero on entry -
// the launches leave it zero).
extern "C" int mos_lbfgs_direction(const void* const* S, const void* const* Y, const double* rho, int32_t k, const float* g,
                                   float h_diag, int64_t n, float* d, double* work, float* partial, float* gtd,
                                   void* stream) {
  MOS_CHECK_ARG(g && d && work && partial && gtd && n > 0 && k >= 0 && (k == 0 || (S && Y && rho)),
                "mos_lbfgs_direction: bad arguments");
  LbfgsStep p;
  memset(&p, 0, sizeof(p));
  p.v = d;
  p.g = g;
  p.n = n;
  p.al = work;
  p.coef = work + k;
  p.partial = partial;
  p.counter = reinterpret_cast<unsigned*>(partial + RED_BLOCKS);
  p.gtd = gtd;
  p.h_diag = h_diag;
  bool first = true;
  const float* pending = nullptr;      // vector whose update (with the coefficient in *coef) the next launch applies
  for (int i = k - 1; i >= 0; --i) {   // first loop: q -= al_i y_i
    p.first = first ? 1 : 0;
    p.upd = pending;
    p.scale = 0;
    p.dotv = reinterpret_cast<const float*>(S[i]);
    p.mode = 0;
    p.idx = i;
    p.rho = rho[i];
    lbfgs_step_kernel<<<RED_BLOCKS, 256, 0, STREAM(stream)>>>(p);
    MOS_CHECK_LAUNCH();
    first = false;
    pending = reinterpret_cast<const float*>(Y[i]);
  }
  bool scale = true;                   // r = h_diag * q, applied by the first launch after the first loop
  for (int i = 0; i < k; ++i) {        // second loop: r += (al_i - be_i) s_i
    p.first = first ? 1 : 0;
    p.upd = pending;
    p.scale = scale ? 1 : 0;
    p.dotv = reinterpret_cast<const float*>(Y[i]);
    p.mode = 1;
    p.idx = i;
    p.rho = rho[i];
    lbfgs_step_kernel<<<RED_BLOCKS, 256, 0, STREAM(stream)>>>(p);
    MOS_CHECK_LAUNCH();
    first = false;
    scale = false;
    pending = reinterpret_cast<const float*>(S[i]);
  }
  p.first = first ? 1 : 0;
  p.upd = pending;
  p.scale = scale ? 1 : 0;
  p.dotv = g;
  p.mode = 2;
  lbfgs_step_kernel<<<RED_BLOCKS, 256, 0, STREAM(stream)>>>(p);
  MOS_CHECK_LAUNCH();
  return MOS_OK;
}

// Same recursion with the history held in two rings (see LbfgsStep): logical pair i = physical slot (*head_dev + i) % slots of
// S_ring / Y_ring [slots, n]; rho_dev [slots] (physical) and hdiag_dev [1] in device memory.  The 2k + 1 launches carry no
// per-iteration host values, so a caller may capture them once in a CUDA graph and replay it while k stays the same.
extern "C" int mos_lbfgs_direction_ring(const float* S_ring, const float* Y_ring, int32_t slots, const int32_t* head_dev,
                                        const double* rho_dev, const float* hdiag_dev, int32_t k, const float* g, int64_t n,
                                        float* d, double* work, float* partial, float* gtd, void* stream) {
  MOS_CHECK_ARG(S_ring && Y_ring && head_dev && rho_dev && hdiag_dev && g && d && work && partial && gtd && n > 0 && k >= 0 &&
                    slots >= k && slots > 0, "mos_lbfgs_direction_ring: bad arguments");
  LbfgsStep p;
  memset(&p, 0, sizeof(p));
  p.v = d;
  p.g = g;
  p.n = n;
  p.al = work;
  p.coef = work + k;
  p.partial = partial;
  p.counter = reinterpret_cast<unsigned*>(partial + RED_BLOCKS);
  p.gtd = gtd;
  p.ring = 1;
  p.slots = slots;
  p.ring_s = S_ring;
  p.ring_y = Y_ring;
  p.head = head_dev;
  p.rho_dev = rho_dev;
  p.hdiag_dev = hdiag_dev;
  bool first = true;
  int pend_kind = 0, pend_idx = 0;
  for (int i = k - 1; i >= 0; --i) {
    p.first = first ? 1 : 0;
    p.upd_kind = pend_kind, p.upd_idx = pend_idx;
    p.scale = 0;
    p.dot_kind = 1;
    p.mode = 0;
    p.idx = i;
    lbfgs_step_kernel<<<RED_BLOCKS, 256, 0, STREAM(stream)>>>(p);
    MOS_CHECK_LAUNCH();
    first = false;
    pend_kind = 2, pend_idx = i;
  }
  bool scale = true;
  for (int i = 0; i < k; ++i) {
    p.first = first ? 1 : 0;
    p.upd_kind = pend_kind, p.upd_idx = pend_idx;
    p.scale = scale ? 1 : 0;
    p.dot_kind = 2;
    p.mode = 1;
    p.idx = i;
    lbfgs_step_kernel<<<RED_BLOCKS, 256, 0, STREAM(stream)>>>(p);
    MOS_CHECK_LAUNCH();
    first = false;
    scale = false;
    pend_kind = 1, pend_idx = i;
  }
  p.first = first ? 1 : 0;
  p.upd_kind = pend_kind, p.upd_idx = pend_idx;
  p.scale = scale ? 1 : 0;
  p.dot_kind = 3;
  p.mode = 2;
  p.idx = 0;
  lbfgs_step_kernel<<<RED_BLOCKS, 256, 0, STREAM(stream)>>>(p);
  MOS_CHECK_LAUNCH();
  return MOS_OK;
}

extern "C" int mos_lora_merge(const int64_t* table_dev, int32_t n_layers, float alpha, void* stream) {
  MOS_CHECK_ARG(table_dev && n_layers > 0, "mos_lora_merge: bad arguments");
  dim3 grid(132, (unsigned)n_layers);   // one block row per SM of an H100 (the kernel strides over the layer)
  lora_merge_kernel<<<grid, 256, 0, STREAM(stream)>>>(reinterpret_cast<const long long*>(table_dev), alpha);
  MOS_CHECK_LAUNCH();
  return MOS_OK;
}
