// attention_bwd.cu — flash-attention backward on wgmma (sm_90a) for d = 40 / 80 / 160 (training step,
// trainer_edlora.py:237 reached through loss.backward(); forward counterpart: attention.cu).
//
//   P = softmax(S), S = scale Q K^T ;  O = P V ;  given dO:
//   dV = P^T dO ;  dP = dO V^T ;  dS = P o (dP + G - delta) ;  dQ = scale dS K ;  dK = scale dS^T Q
//   delta[q] = rowsum(dO o O) (+ rowsum(P o G));  G = optional gradient on the probabilities themselves (attention
//   regulariser, trainer_edlora.py:263-313: two key columns per sample, identical over heads).
//
// Two kernels, both recompute P from the saved log-sum-exp (no atomics, no N x N tensor in HBM):
//   attn_bwd_dq_kernel   one CTA per 128-query tile, loops over key tiles:  S, dP (wgmma, registers) -> dS in registers
//                        -> dQ += dS K (wgmma with dS as the register A operand)
//   attn_bwd_dkv_kernel  one CTA per 128-key tile, loops over query tiles: S^T = K Q^T, dP^T = V dO^T -> P^T, dS^T in
//                        registers -> dV += P^T dO, dK += dS^T Q.  For d = 160 the dK / dV columns are split over two CTAs
//                        (gridDim.z) so that both accumulators fit the register file.
// Roles as in the forward kernel: two consumer warpgroups of 64 rows each, warp 8 = TMA producer.
// Operand layouts: rows [B*H, R, DP] and transposed [B*H, DV, R8] copies (mos_heads_transpose) so that every shared-memory
// operand is K-major SWIZZLE_128B.  Outputs are token-major [B*R, ld] bf16 (head h in columns h*d ..).
#include "common.h"
#include "tc.cuh"

namespace mos {

__device__ __forceinline__ float ex2_approx_b(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

template <int D>
struct BwdCfg {
  static constexpr int KSTEPS = (D + 15) / 16;
  static constexpr int DP = ((D + 63) / 64) * 64;
  static constexpr int QCH = DP / 64;
  static constexpr int DV = ((D + 15) / 16) * 16;
  static constexpr int BT = 64;                               // inner tile (keys for dQ, queries for dK / dV)
  static constexpr int STAGES = D <= 80 ? 2 : 1;
  // ---- dQ kernel
  static constexpr int A_Q_BYTES = QCH * 128 * 128;           // Q or dO tile [128, DP]
  static constexpr int A_K_BYTES = QCH * BT * 128;            // K or V tile [BT, DP]
  static constexpr int A_KT_BYTES = DV * 128;                 // K^T tile [DV, BT]
  static constexpr int A_STAGE = 2 * A_K_BYTES + A_KT_BYTES;
  static constexpr int A_SMEM = 2 * A_Q_BYTES + STAGES * A_STAGE + 1024;
  // ---- dK/dV kernel
  static constexpr int DVH = D <= 80 ? DV : DV / 2;           // output columns per CTA
  static constexpr int ZSPLIT = DV / DVH;
  static constexpr int B_K_BYTES = QCH * 128 * 128;           // K or V tile [128, DP]
  static constexpr int B_Q_BYTES = QCH * BT * 128;            // Q or dO tile [BT, DP]
  static constexpr int B_QT_BYTES = DV * 128;                 // Q^T or dO^T tile [DV, BT]
  static constexpr int B_STAGE = 2 * B_Q_BYTES + 2 * B_QT_BYTES;
  static constexpr int B_SMEM = 2 * B_K_BYTES + STAGES * B_STAGE + 1024;
  static_assert(A_SMEM <= 227 * 1024 - 2048 && B_SMEM <= 227 * 1024 - 2048, "smem budget");
};

constexpr int BWD_THREADS = 256 + 32;

struct BwdDev {
  int nq, nk, heads;
  float scale, scale_log2;
  const float* lse2;    // [BH, nq]  log2-domain log-sum-exp of scale*S
  const float* delta;   // [BH, nq]
  const float* gcols;   // optional [B, nq, 2]: gradient on the probabilities at key columns pos[b][0..1]
  const int* pos;       // optional [B, 2]
  int causal;           // self-attention with keys <= query only (CLIP text encoder)
  __nv_bfloat16* dq;    // token-major outputs
  long long lddq;
  __nv_bfloat16* dk;
  long long lddk;
  __nv_bfloat16* dv;
  long long lddv;
};

// S = A_rows B_rows^T over the head dimension: KSTEPS k16 steps over 64-column chunks of [rows, DP] tiles
template <int D, int ROWS_B>
__device__ __forceinline__ void bwd_rows_product(float (&s)[BwdCfg<D>::BT / 2], const uint8_t* sa, const uint8_t* sb) {
  using C = BwdCfg<D>;
  const uint64_t ad = make_desc_sw128(smem_u32(sa)), bd = make_desc_sw128(smem_u32(sb));
#pragma unroll
  for (int kk = 0; kk < C::KSTEPS; ++kk)
    wgmma_ss<C::BT, false>(s, ad + (kk >> 2) * (16384 >> 4) + 2 * (kk & 3),
                           bd + (kk >> 2) * ((ROWS_B * 128) >> 4) + 2 * (kk & 3), 1u);
}

// =================================================================================================== dQ
template <int D>
__global__ void __launch_bounds__(BWD_THREADS, 1)
attn_bwd_dq_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmdO,
                   const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                   const __grid_constant__ CUtensorMap tmKt, const BwdDev p) {
  using C = BwdCfg<D>;
  constexpr int BT = C::BT, NS = BT / 2, NO = C::DV / 2;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sdO = sQ + C::A_Q_BYTES;
  uint8_t* sStages = sdO + C::A_Q_BYTES;

  __shared__ uint64_t qdo_full, kv_full[C::STAGES], kv_empty[C::STAGES];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * 128;
  const int bh = blockIdx.y;
  const int T = (p.nk + BT - 1) / BT;

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmdO);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    tma_prefetch_desc(&tmKt);
    mbar_init(&qdo_full, 1);
    for (int s = 0; s < C::STAGES; ++s) {
      mbar_init(&kv_full[s], 1);
      mbar_init(&kv_empty[s], 8);
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();
  pdl_launch_dependents();

  if (warp == 8) {
    if (lane == 0) {
      mbar_expect_tx(&qdo_full, 2 * C::A_Q_BYTES);
#pragma unroll
      for (int c = 0; c < C::QCH; ++c) {
        tma_load_3d(sQ + c * 16384, &tmQ, &qdo_full, c * 64, q0, bh);
        tma_load_3d(sdO + c * 16384, &tmdO, &qdo_full, c * 64, q0, bh);
      }
      int st = 0;
      uint32_t ph = 0;
      for (int j = 0; j < T; ++j) {
        uint8_t* sK = sStages + st * C::A_STAGE;
        uint8_t* sV = sK + C::A_K_BYTES;
        uint8_t* sKt = sV + C::A_K_BYTES;
        mbar_wait_hint(&kv_empty[st], ph ^ 1);
        mbar_expect_tx(&kv_full[st], C::A_STAGE);
#pragma unroll
        for (int c = 0; c < C::QCH; ++c) {
          tma_load_3d(sK + c * (BT * 128), &tmK, &kv_full[st], c * 64, j * BT, bh);
          tma_load_3d(sV + c * (BT * 128), &tmV, &kv_full[st], c * 64, j * BT, bh);
        }
        tma_load_3d(sKt, &tmKt, &kv_full[st], j * BT, 0, bh);
        if (++st == C::STAGES) {
          st = 0;
          ph ^= 1;
        }
      }
    }
    return;
  }

  const int wg = warp >> 2;
  const int rA = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const int cq = 2 * (lane & 3);
  const int b = bh / p.heads, h = bh - b * p.heads;
  float lse[2], dl[2], g0[2] = {0.f, 0.f}, g1[2] = {0.f, 0.f};
  int pos0 = -1, pos1 = -1;
  if (p.gcols != nullptr) {
    pos0 = __ldg(p.pos + b * 2);
    pos1 = __ldg(p.pos + b * 2 + 1);
  }
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int q_idx = q0 + rA + 8 * hr;
    const bool row_ok = q_idx < p.nq;
    lse[hr] = row_ok ? __ldg(p.lse2 + (long long)bh * p.nq + q_idx) : INFINITY;
    dl[hr] = row_ok ? __ldg(p.delta + (long long)bh * p.nq + q_idx) : 0.f;
    if (p.gcols != nullptr && row_ok) {
      g0[hr] = __ldg(p.gcols + ((long long)b * p.nq + q_idx) * 2);
      g1[hr] = __ldg(p.gcols + ((long long)b * p.nq + q_idx) * 2 + 1);
    }
  }
  float dq[NO];
#pragma unroll
  for (int i = 0; i < NO; ++i) dq[i] = 0.f;
  mbar_wait(&qdo_full, 0);
  int st = 0;
  uint32_t ph = 0;
  for (int j = 0; j < T; ++j) {
    uint8_t* sK = sStages + st * C::A_STAGE;
    uint8_t* sV = sK + C::A_K_BYTES;
    uint8_t* sKt = sV + C::A_K_BYTES;
    mbar_wait(&kv_full[st], ph);
    float s[NS], dp[NS];
#pragma unroll
    for (int i = 0; i < NS; ++i) s[i] = dp[i] = 0.f;
    wgmma_fence_regs(s);
    wgmma_fence_regs(dp);
    wgmma_fence();
    bwd_rows_product<D, BT>(s, sQ + wg * (64 * 128), sK);
    bwd_rows_product<D, BT>(dp, sdO + wg * (64 * 128), sV);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(s);
    wgmma_fence_regs(dp);
    const int kv_valid = min(BT, p.nk - j * BT);
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const int q_idx = q0 + rA + 8 * hr;
#pragma unroll
      for (int i = 0; i < BT / 8; ++i)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = 8 * i + cq + e, key = j * BT + col;
          const int x = 4 * i + 2 * hr + e;
          float pr = ex2_approx_b(fmaf(s[x], p.scale_log2, -lse[hr]));
          pr = (col < kv_valid && (!p.causal || key <= q_idx)) ? pr : 0.f;
          float d = dp[x];
          if (p.gcols != nullptr) d += (key == pos0) ? g0[hr] : ((key == pos1) ? g1[hr] : 0.f);
          s[x] = pr * (d - dl[hr]) * p.scale;     // dS
        }
    }
    const int ksteps = (kv_valid + 15) >> 4;
    wgmma_fence_regs(dq);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < BT / 16; ++kk) {
      if (kk < ksteps) {
        uint32_t a[4];
        frag_to_a<false>(&s[8 * kk], a);
        wgmma_rs<C::DV, false>(dq, a, make_desc_sw128(smem_u32(sKt)) + 2 * kk, 1u);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(dq);
    __syncwarp();
    if (lane == 0) mbar_arrive(&kv_empty[st]);
    if (++st == C::STAGES) {
      st = 0;
      ph ^= 1;
    }
  }
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int q_idx = q0 + rA + 8 * hr;
    if (q_idx >= p.nq) continue;
    __nv_bfloat16* orow = p.dq + ((long long)b * p.nq + q_idx) * p.lddq + h * D;
#pragma unroll
    for (int i = 0; i < C::DV / 8; ++i) {
      const int col = 8 * i + cq;
      if (col < D) *reinterpret_cast<uint32_t*>(orow + col) = pack_bf16x2(dq[4 * i + 2 * hr], dq[4 * i + 2 * hr + 1]);
    }
  }
}

// =================================================================================================== dK, dV
template <int D>
__global__ void __launch_bounds__(BWD_THREADS, 1)
attn_bwd_dkv_kernel(const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                    const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmdO,
                    const __grid_constant__ CUtensorMap tmQt, const __grid_constant__ CUtensorMap tmdOt,
                    const BwdDev p) {
  using C = BwdCfg<D>;
  constexpr int BT = C::BT, NS = BT / 2, NO = C::DVH / 2;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sK = smem;
  uint8_t* sV = sK + C::B_K_BYTES;
  uint8_t* sStages = sV + C::B_K_BYTES;

  __shared__ uint64_t kv_full, q_full[C::STAGES], q_empty[C::STAGES];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int k0 = blockIdx.x * 128;
  const int bh = blockIdx.y;
  const int z = blockIdx.z;                  // output column block [z * DVH, z * DVH + DVH)
  const int T = (p.nq + BT - 1) / BT;

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmdO);
    tma_prefetch_desc(&tmQt);
    tma_prefetch_desc(&tmdOt);
    mbar_init(&kv_full, 1);
    for (int s = 0; s < C::STAGES; ++s) {
      mbar_init(&q_full[s], 1);
      mbar_init(&q_empty[s], 8);
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();
  pdl_launch_dependents();

  if (warp == 8) {
    if (lane == 0) {
      mbar_expect_tx(&kv_full, 2 * C::B_K_BYTES);
#pragma unroll
      for (int c = 0; c < C::QCH; ++c) {
        tma_load_3d(sK + c * 16384, &tmK, &kv_full, c * 64, k0, bh);
        tma_load_3d(sV + c * 16384, &tmV, &kv_full, c * 64, k0, bh);
      }
      int st = 0;
      uint32_t ph = 0;
      for (int i = 0; i < T; ++i) {
        uint8_t* sQ = sStages + st * C::B_STAGE;
        uint8_t* sdO = sQ + C::B_Q_BYTES;
        uint8_t* sQt = sdO + C::B_Q_BYTES;
        uint8_t* sdOt = sQt + C::B_QT_BYTES;
        mbar_wait_hint(&q_empty[st], ph ^ 1);
        mbar_expect_tx(&q_full[st], C::B_STAGE);
#pragma unroll
        for (int c = 0; c < C::QCH; ++c) {
          tma_load_3d(sQ + c * (BT * 128), &tmQ, &q_full[st], c * 64, i * BT, bh);
          tma_load_3d(sdO + c * (BT * 128), &tmdO, &q_full[st], c * 64, i * BT, bh);
        }
        tma_load_3d(sQt, &tmQt, &q_full[st], i * BT, 0, bh);
        tma_load_3d(sdOt, &tmdOt, &q_full[st], i * BT, 0, bh);
        if (++st == C::STAGES) {
          st = 0;
          ph ^= 1;
        }
      }
    }
    return;
  }

  const int wg = warp >> 2;
  const int rA = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // key rows rA, rA + 8 of the tile
  const int cq = 2 * (lane & 3);
  const int b = bh / p.heads, h = bh - b * p.heads;
  int gsel[2] = {0, 0};   // 1: this key is the first concept-token column, 2: the second
  if (p.gcols != nullptr) {
    const int pos0 = __ldg(p.pos + b * 2), pos1 = __ldg(p.pos + b * 2 + 1);
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const int key = k0 + rA + 8 * hr;
      gsel[hr] = key == pos0 ? 1 : (key == pos1 ? 2 : 0);
    }
  }
  float dk[NO], dv[NO];
#pragma unroll
  for (int i = 0; i < NO; ++i) dk[i] = dv[i] = 0.f;
  mbar_wait(&kv_full, 0);
  int st = 0;
  uint32_t ph = 0;
  for (int i = 0; i < T; ++i) {
    uint8_t* sQ = sStages + st * C::B_STAGE;
    uint8_t* sdO = sQ + C::B_Q_BYTES;
    uint8_t* sQt = sdO + C::B_Q_BYTES;
    uint8_t* sdOt = sQt + C::B_QT_BYTES;
    mbar_wait(&q_full[st], ph);
    float s[NS], dp[NS];
#pragma unroll
    for (int x = 0; x < NS; ++x) s[x] = dp[x] = 0.f;
    wgmma_fence_regs(s);
    wgmma_fence_regs(dp);
    wgmma_fence();
    bwd_rows_product<D, BT>(s, sK + wg * (64 * 128), sQ);
    bwd_rows_product<D, BT>(dp, sV + wg * (64 * 128), sdO);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(s);
    wgmma_fence_regs(dp);
    const int q_valid = min(BT, p.nq - i * BT);
    // per query column of this thread: lse, delta, probability gradient
#pragma unroll
    for (int c8 = 0; c8 < BT / 8; ++c8)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int col = 8 * c8 + cq + e, q = i * BT + col;
        const bool ok = col < q_valid;
        const float lq = ok ? __ldg(p.lse2 + (long long)bh * p.nq + q) : INFINITY;
        const float dq = ok ? __ldg(p.delta + (long long)bh * p.nq + q) : 0.f;
        float gq[2] = {0.f, 0.f};
        if (p.gcols != nullptr && ok) {
          gq[0] = __ldg(p.gcols + ((long long)b * p.nq + q) * 2);
          gq[1] = __ldg(p.gcols + ((long long)b * p.nq + q) * 2 + 1);
        }
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          const int key = k0 + rA + 8 * hr;
          const int x = 4 * c8 + 2 * hr + e;
          float pr = ex2_approx_b(fmaf(s[x], p.scale_log2, -lq));
          pr = (key < p.nk && (!p.causal || key <= q)) ? pr : 0.f;
          float d = dp[x];
          if (gsel[hr] != 0) d += gq[gsel[hr] - 1];
          s[x] = pr;                              // P^T
          dp[x] = pr * (d - dq) * p.scale;        // dS^T
        }
      }
    const int ksteps = (q_valid + 15) >> 4;
    const uint32_t zoff = (uint32_t)(z * C::DVH * 128);
    wgmma_fence_regs(dk);
    wgmma_fence_regs(dv);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < BT / 16; ++kk) {
      if (kk < ksteps) {
        uint32_t a[4];
        frag_to_a<false>(&s[8 * kk], a);
        wgmma_rs<C::DVH, false>(dv, a, make_desc_sw128(smem_u32(sdOt) + zoff) + 2 * kk, 1u);
        frag_to_a<false>(&dp[8 * kk], a);
        wgmma_rs<C::DVH, false>(dk, a, make_desc_sw128(smem_u32(sQt) + zoff) + 2 * kk, 1u);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(dk);
    wgmma_fence_regs(dv);
    __syncwarp();
    if (lane == 0) mbar_arrive(&q_empty[st]);
    if (++st == C::STAGES) {
      st = 0;
      ph ^= 1;
    }
  }
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int key = k0 + rA + 8 * hr;
    if (key >= p.nk) continue;
    __nv_bfloat16* krow = p.dk + ((long long)b * p.nk + key) * p.lddk + h * D + z * C::DVH;
    __nv_bfloat16* vrow = p.dv + ((long long)b * p.nk + key) * p.lddv + h * D + z * C::DVH;
#pragma unroll
    for (int c8 = 0; c8 < C::DVH / 8; ++c8) {
      const int col = 8 * c8 + cq;
      if (z * C::DVH + col < D) {
        *reinterpret_cast<uint32_t*>(krow + col) = pack_bf16x2(dk[4 * c8 + 2 * hr], dk[4 * c8 + 2 * hr + 1]);
        *reinterpret_cast<uint32_t*>(vrow + col) = pack_bf16x2(dv[4 * c8 + 2 * hr], dv[4 * c8 + 2 * hr + 1]);
      }
    }
  }
}

static int rows_tmap(CUtensorMap* tm, const void* base, int DP, int R, int BH, int box_rows) {
  uint64_t dims[3] = {(uint64_t)DP, (uint64_t)R, (uint64_t)BH};
  uint64_t str[2] = {(uint64_t)DP * 2, (uint64_t)R * DP * 2};
  uint32_t box[3] = {64, (uint32_t)box_rows, 1};
  return encode_tmap(tm, base, 2, 3, dims, str, box, 3);
}
static int trans_tmap(CUtensorMap* tm, const void* base, int DV, int R8, int BH) {
  uint64_t dims[3] = {(uint64_t)R8, (uint64_t)DV, (uint64_t)BH};
  uint64_t str[2] = {(uint64_t)R8 * 2, (uint64_t)DV * R8 * 2};
  uint32_t box[3] = {64, (uint32_t)DV, 1};
  return encode_tmap(tm, base, 2, 3, dims, str, box, 3);
}

template <int D>
static int launch_bwd(const void* Q, const void* K, const void* V, const void* dO, const void* Qt, const void* Kt,
                      const void* dOt, const BwdDev& p, int BH, int nq8, int nk8, cudaStream_t stream) {
  using C = BwdCfg<D>;
  CUtensorMap tQa, tdOa, tKa, tVa, tKt, tKb, tVb, tQb, tdOb, tQt, tdOt;
  int rc;
  if ((rc = rows_tmap(&tQa, Q, C::DP, p.nq, BH, 128))) return rc;
  if ((rc = rows_tmap(&tdOa, dO, C::DP, p.nq, BH, 128))) return rc;
  if ((rc = rows_tmap(&tKa, K, C::DP, p.nk, BH, C::BT))) return rc;
  if ((rc = rows_tmap(&tVa, V, C::DP, p.nk, BH, C::BT))) return rc;
  if ((rc = trans_tmap(&tKt, Kt, C::DV, nk8, BH))) return rc;
  if ((rc = rows_tmap(&tKb, K, C::DP, p.nk, BH, 128))) return rc;
  if ((rc = rows_tmap(&tVb, V, C::DP, p.nk, BH, 128))) return rc;
  if ((rc = rows_tmap(&tQb, Q, C::DP, p.nq, BH, C::BT))) return rc;
  if ((rc = rows_tmap(&tdOb, dO, C::DP, p.nq, BH, C::BT))) return rc;
  if ((rc = trans_tmap(&tQt, Qt, C::DV, nq8, BH))) return rc;
  if ((rc = trans_tmap(&tdOt, dOt, C::DV, nq8, BH))) return rc;
  static bool configured = false;
  if (!configured) {
    MOS_CHECK_CUDA(cudaFuncSetAttribute(attn_bwd_dq_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::A_SMEM));
    MOS_CHECK_CUDA(cudaFuncSetAttribute(attn_bwd_dkv_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::B_SMEM));
    configured = true;
  }
  MOS_CHECK_CUDA(launch_pdl(attn_bwd_dq_kernel<D>, dim3((unsigned)ceil_div(p.nq, 128), (unsigned)BH), dim3(BWD_THREADS),
                            (size_t)C::A_SMEM, stream, tQa, tdOa, tKa, tVa, tKt, p));
  MOS_CHECK_CUDA(launch_pdl(attn_bwd_dkv_kernel<D>, dim3((unsigned)ceil_div(p.nk, 128), (unsigned)BH, (unsigned)C::ZSPLIT),
                            dim3(BWD_THREADS), (size_t)C::B_SMEM, stream, tKb, tVb, tQb, tdOb, tQt, tdOt, p));
  return MOS_OK;
}

}  // namespace mos

using namespace mos;

extern "C" int mos_attention_bwd(const void* Q, const void* K, const void* V, const void* dO, const void* Qt,
                                 const void* Kt, const void* dOt, const float* lse2, const float* delta,
                                 const float* gcols, const int32_t* pos, void* dq, int64_t lddq, void* dk, int64_t lddk,
                                 void* dv, int64_t lddv, int32_t batch, int32_t heads, int32_t head_dim, int32_t nq,
                                 int32_t nk, int32_t nq8, int32_t nk8, float scale, int32_t causal, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  MOS_CHECK_ARG(Q && K && V && dO && Qt && Kt && dOt && lse2 && delta && dq && dk && dv, "mos_attention_bwd: NULL pointer");
  MOS_CHECK_ARG(batch > 0 && heads > 0 && nq > 0 && nk > 0 && nq8 >= nq && nk8 >= nk && nq8 % 8 == 0 && nk8 % 8 == 0,
                "mos_attention_bwd: bad shape");
  MOS_CHECK_ARG(lddq % 8 == 0 && lddk % 8 == 0 && lddv % 8 == 0 && (!gcols == !pos), "mos_attention_bwd: bad pitches");
  BwdDev p;
  p.nq = nq;
  p.nk = nk;
  p.heads = heads;
  p.scale = scale;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.lse2 = lse2;
  p.delta = delta;
  p.gcols = gcols;
  p.pos = reinterpret_cast<const int*>(pos);
  p.causal = causal ? 1 : 0;
  MOS_CHECK_ARG(!causal || nq == nk, "mos_attention_bwd: causal needs nq == nk");
  p.dq = reinterpret_cast<__nv_bfloat16*>(dq);
  p.lddq = lddq;
  p.dk = reinterpret_cast<__nv_bfloat16*>(dk);
  p.lddk = lddk;
  p.dv = reinterpret_cast<__nv_bfloat16*>(dv);
  p.lddv = lddv;
  const int BH = batch * heads;
  switch (head_dim) {
    case 40: return launch_bwd<40>(Q, K, V, dO, Qt, Kt, dOt, p, BH, nq8, nk8, stream);
    case 80: return launch_bwd<80>(Q, K, V, dO, Qt, Kt, dOt, p, BH, nq8, nk8, stream);
    case 160: return launch_bwd<160>(Q, K, V, dO, Qt, Kt, dOt, p, BH, nq8, nk8, stream);
    default: return set_err(MOS_EUNSUPPORTED, "mos_attention_bwd: head_dim %d not in {40, 80, 160}", head_dim);
  }
}
