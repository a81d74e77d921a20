// attention.cu — K2/K3: flash attention on wgmma (sm_90a) for the SD1.5 head sizes d = 40 / 80 / 160 (8 heads).
//
//   O = softmax(Q K^T * scale) V     per (batch, head);  self-attention (N x N) and cross-attention (N x 77)
//
// Replaces xformers.ops.memory_efficient_attention / attn.get_attention_scores + bmm at
// mixofshow/models/edlora.py:77-83,151-156 and pipeline_regionally_t2iadapter.py:111-116.
//
// One CTA = one 128-query tile of one (batch, head).  288 threads:
//   warps 0..7  two consumer warpgroups, 64 query rows each: S_j = Q K_j^T (wgmma, A and B from shared memory) into
//               registers, online softmax in registers (a row lives in the 4 lanes of a quad), P_j packed to 16 bits in
//               registers and fed back as the A operand of O += P_j V_j (wgmma, A from registers); O stays in registers
//   warp 8      TMA producer (Q once, K / V^T ring); the multi-tile kernel has a producer warpgroup, warps 8..11
// Two variants, chosen on the host from nk alone:
//   ONE (nk <= 128)  one KV tile; carries the probability maps (probs), the regulariser columns (pcols) and CAUSAL
//   multi (nk > 128) the KV tiles run as a software pipeline inside each consumer warpgroup (AttnPipe): the exponentials
//                    of tile j run while tile j-1's O += P V is on the tensor cores; a producer warpgroup instead of a
//                    warp; only lse2 among the optional outputs
// Layouts (written by the QKV GEMM epilogue): Q,K [B*H, rows, DP] (DP = d padded to 64, pad = 0),
// V^T [B*H, DV, nk8] (keys contiguous), so every shared-memory operand is K-major SWIZZLE_128B.
#include <stdlib.h>

#include "common.h"
#include "tc.cuh"

namespace mos {

// volatile: keeps the exponentials in program order with the wgmma issue and wait asm around them (a plain asm may be
// moved past the wait, out of the window where the tensor cores work under it)
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm volatile("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

struct AttnDev {
  int nq, nk, heads;
  float scale_log2;  // scale * log2(e)
  __nv_bfloat16* out;
  long long ldo;
  float* probs;  // optional [B*H, nq, nk] fp32 (single kv tile only)
  float* lse2;   // optional [B*H, nq]: log2-domain log-sum-exp of scale*S (saved for the backward kernels)
  float* pcols;  // optional [B*H, nq, 2]: probabilities at key columns pos[b][0..1] (single kv tile only)
  const int* pos;
};

// Two consumer warpgroups + the TMA producer.  Single tile: one producer warp.  Multi-tile: a producer warpgroup that
// hands registers to the consumers with setmaxnreg (more than 8 warps cap a thread at 168 registers at launch, since one
// SM sub-partition then holds 3 warps; at d = 80 the consumers need more for 128-key tiles without spilling).
template <bool ONE>
constexpr int attn_threads() { return ONE ? 256 + 32 : 256 + 128; }
constexpr int ATTN_PRODUCER_REGS = 40, ATTN_CONSUMER_REGS = 232;   // 128 * 40 + 256 * 232 = 384 * 168

// ONE: single-tile variant for cross-attention (nk <= 128): one 128-key tile, so that the probability maps /
// concept-token columns of the controller and regulariser paths come from a single kv tile.
template <int D, bool ONE = false>
struct AttnCfg {
  static constexpr int KSTEPS = (D + 15) / 16;
  static constexpr int DP = ((D + 63) / 64) * 64;
  static constexpr int QCH = DP / 64;
  static constexpr int DV = ((D + 15) / 16) * 16;
  static constexpr int BKV = ONE ? 128 : (D <= 80 ? 128 : 64);
  static constexpr int KVCH = BKV / 64;
  // multi: see AttnPipe
  static constexpr int STAGES = ONE ? 1 : 3;
  static constexpr int Q_BYTES = QCH * 128 * 128;
  static constexpr int K_BYTES = QCH * BKV * 128;
  static constexpr int V_BYTES = KVCH * DV * 128;
  static constexpr int STAGE_BYTES = K_BYTES + V_BYTES;
  static constexpr int SMEM_BYTES = Q_BYTES + STAGES * STAGE_BYTES + 1024;
  static_assert(SMEM_BYTES <= 227 * 1024, "smem budget");
};

__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// O += P V over the first NSTEP k16 steps of a KV tile: one straight-line wgmma chain.  pa holds the P fragments, packed
// before the fence (a register written between wgmma.fence and the wgmma that reads it makes ptxas inject a warpgroup
// arrive), and the chain length is a compile-time constant (a wgmma under a runtime guard makes ptxas serialise them all).
template <int NSTEP, int DV, bool F16, int NKK>
__device__ __forceinline__ void pv_chain(float (&o)[DV / 2], const uint32_t (&pa)[NKK][4], const uint8_t* sV) {
  wgmma_fence_regs(o);
  wgmma_fence();
#pragma unroll
  for (int kk = 0; kk < NSTEP; ++kk) {
    const uint64_t vd = make_desc_sw128(smem_u32(sV + (kk >> 2) * (DV * 128))) + 2 * (kk & 3);
    wgmma_rs<DV, F16>(o, pa[kk], vd, 1u);
  }
  wgmma_commit();
  wgmma_wait<0>();
  wgmma_fence_regs(o);
}
// ksteps (1..NSTEP) -> the chain of that length: every KV tile but a partial last one takes the NSTEP = BKV / 16 chain
template <int NSTEP, int DV, bool F16, int NKK>
__device__ __forceinline__ void pv_dispatch(int ksteps, float (&o)[DV / 2], const uint32_t (&pa)[NKK][4],
                                            const uint8_t* sV) {
  if (ksteps == NSTEP) {
    pv_chain<NSTEP, DV, F16>(o, pa, sV);
  } else if constexpr (NSTEP > 1) {
    pv_dispatch<NSTEP - 1, DV, F16>(ksteps, o, pa, sV);
  }
}

template <int R>
__device__ __forceinline__ void fence_regs_u32(uint32_t (&a)[R][4]) {
#pragma unroll
  for (int i = 0; i < R; ++i)
#pragma unroll
    for (int k = 0; k < 4; ++k) asm volatile("" : "+r"(a[i][k])::"memory");
}

// ---------------------------------------------------------------------------------------------- multi-tile consumer
// S = Q K^T of one KV tile, issued and committed, not waited for.  The first k-step overwrites the accumulator
// (scale-d = 0), so S needs no zeroing.
template <int D, bool F16>
__device__ __forceinline__ void issue_qk(float (&s)[AttnCfg<D>::BKV / 2], uint64_t qdesc, const uint8_t* sK) {
  using C = AttnCfg<D>;
  wgmma_fence_regs(s);
  wgmma_fence();
#pragma unroll
  for (int kk = 0; kk < C::KSTEPS; ++kk) {
    const uint64_t kd = make_desc_sw128(smem_u32(sK + (kk >> 2) * (C::BKV * 128)));
    wgmma_ss<C::BKV, F16>(s, qdesc + (kk >> 2) * (16384 >> 4) + 2 * (kk & 3), kd + 2 * (kk & 3), kk == 0 ? 0u : 1u);
  }
  wgmma_commit();
}

// Online softmax of one KV tile in the log2 domain, in two halves.  ptxas waits for every outstanding wgmma before a warp
// shuffle, so the row max (two quad shuffles per row) runs while no wgmma is in flight, and the exponentials, which
// need no shuffle, run under the tensor-core work issued between the two halves.
// row_max: m = max(m, c max_k S_k) and alpha = ex2(m_old - m_new), the factor O and l are rescaled by.  MASK (the
// partial last tile only): columns >= kv_valid -> -inf (P = 0); every tile has a valid column, so m stays finite.
template <int NS, bool MASK>
__device__ __forceinline__ void row_max(float (&s)[NS], float (&m)[2], float (&alpha)[2], float c, int cq,
                                        int kv_valid) {
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int i = 0; i < NS / 4; ++i) {
      float& x0 = s[4 * i + 2 * hr];
      float& x1 = s[4 * i + 2 * hr + 1];
      if constexpr (MASK) {
        if (8 * i + cq >= kv_valid) x0 = -INFINITY;
        if (8 * i + cq + 1 >= kv_valid) x1 = -INFINITY;
      }
      mx0 = fmaxf(mx0, x0);
      mx1 = fmaxf(mx1, x1);
    }
    const float m_new = fmaxf(m[hr], quad_max(fmaxf(mx0, mx1)) * c);
    alpha[hr] = ex2_approx(m[hr] - m_new);
    m[hr] = m_new;
  }
}
// S -> P = ex2(S c - m) in place, one FFMA per element; l = l alpha + this thread's row sums (the quad sum is taken
// once, in the epilogue)
template <int NS>
__device__ __forceinline__ void exp_rows(float (&s)[NS], const float (&m)[2], float (&l)[2], const float (&alpha)[2],
                                         float c) {
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const float nm = -m[hr];
    float rs0 = 0.f, rs1 = 0.f;
#pragma unroll
    for (int i = 0; i < NS / 4; ++i) {
      float& x0 = s[4 * i + 2 * hr];
      float& x1 = s[4 * i + 2 * hr + 1];
      x0 = ex2_approx(fmaf(x0, c, nm));
      x1 = ex2_approx(fmaf(x1, c, nm));
      rs0 += x0;
      rs1 += x1;
    }
    l[hr] = fmaf(l[hr], alpha[hr], rs0 + rs1);
  }
}

template <int NO>
__device__ __forceinline__ void rescale_o(float (&o)[NO], const float (&alpha)[2]) {
#pragma unroll
  for (int i = 0; i < NO / 4; ++i) {
    o[4 * i] *= alpha[0];
    o[4 * i + 1] *= alpha[0];
    o[4 * i + 2] *= alpha[1];
    o[4 * i + 3] *= alpha[1];
  }
}

__device__ __forceinline__ void release_stage(uint64_t* kv_empty, int lane) {
  __syncwarp();
  if (lane == 0) mbar_arrive(kv_empty);
}

// The KV tiles of one consumer warpgroup, software-pipelined (FlashAttention-3's intra-warpgroup overlap).  Step j
// starts with P_{j-1} packed in pa and nothing in flight:
//   issue S_j = Q K_j^T, wait | row max of S_j | issue O += P_{j-1} V_{j-1} | exponentials of S_j (MUFU) under it |
//   wait (PV_{j-1} done, its stage goes back to the producer) | rescale O, pack P_j
// While the exponentials run, the other warpgroup's Q K^T and P V keep the tensor cores busy.  Issuing S_{j+1} ahead of
// them as well would hold two S tiles: with 232 registers per consumer thread ptxas still spills that and serialises
// the wgmmas (C7512), so S_j is waited for before its row max.  K/V ring: 3 stages, so that tiles j+1 and j+2 load while
// tile j-1 is held for PV_{j-1}.  Full tiles carry no column mask; the last tile (possibly partial) does, and its PV
// chain has the compile-time length of its valid k-steps (V^T padding is never read).
template <int D, bool F16>
struct AttnPipe {
  using C = AttnCfg<D>;
  static constexpr int NS = C::BKV / 2, NO = C::DV / 2, NKK = C::BKV / 16;
  uint8_t* sKV;
  uint64_t* kv_full;
  uint64_t* kv_empty;
  uint64_t qdesc;
  float c;
  int cq, lane;
  int st;          // stage and kv_full phase of tile j
  uint32_t ph;
  float s[NS];
  float o[NO];
  float m[2], l[2];
  uint32_t pa[NKK][4];

  __device__ __forceinline__ static int prev(int s) { return s == 0 ? C::STAGES - 1 : s - 1; }

  // O += P V of the full tile in `stage`, issued and committed
  __device__ __forceinline__ void issue_pv(int stage) {
    const uint8_t* sV = sKV + stage * C::STAGE_BYTES + C::K_BYTES;
    wgmma_fence_regs(o);
    fence_regs_u32(pa);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < NKK; ++kk) {
      const uint64_t vd = make_desc_sw128(smem_u32(sV + (kk >> 2) * (C::DV * 128))) + 2 * (kk & 3);
      wgmma_rs<C::DV, F16>(o, pa[kk], vd, 1u);
    }
    wgmma_commit();
  }
  // tile j.  PREV: j > 0 (P_{j-1} in pa); MASK: the last tile, kv_valid keys
  template <bool PREV, bool MASK>
  __device__ __forceinline__ void step(int kv_valid) {
    mbar_wait(&kv_full[st], ph);
    issue_qk<D, F16>(s, qdesc, sKV + st * C::STAGE_BYTES);
    wgmma_wait<0>();
    wgmma_fence_regs(s);
    float alpha[2];
    row_max<NS, MASK>(s, m, alpha, c, cq, kv_valid);
    if constexpr (PREV) issue_pv(prev(st));
    exp_rows<NS>(s, m, l, alpha, c);
    if constexpr (PREV) {
      wgmma_wait<0>();
      wgmma_fence_regs(o);
      fence_regs_u32(pa);
      release_stage(&kv_empty[prev(st)], lane);
    }
    rescale_o(o, alpha);
#pragma unroll
    for (int kk = 0; kk < NKK; ++kk) frag_to_a<F16>(&s[8 * kk], pa[kk]);
    if (++st == C::STAGES) {
      st = 0;
      ph ^= 1;
    }
  }
  // O += P_{T-1} V_{T-1} (tile T-1 sits in the stage before st)
  __device__ __forceinline__ void finish(int kv_valid) {
    pv_dispatch<NKK, C::DV, F16>((kv_valid + 15) >> 4, o, pa, sKV + prev(st) * C::STAGE_BYTES + C::K_BYTES);
  }
};

template <int D, bool ONE, bool CAUSAL = false, bool F16 = false>
__global__ void __launch_bounds__(attn_threads<ONE>(), 1)
attn_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
            const __grid_constant__ CUtensorMap tmV, const AttnDev p) {
  using C = AttnCfg<D, ONE>;
  constexpr int NS = C::BKV / 2;    // S fragment registers per thread
  constexpr int NO = C::DV / 2;     // O fragment registers per thread
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sKV = sQ + C::Q_BYTES;

  __shared__ uint64_t q_full, kv_full[C::STAGES], kv_empty[C::STAGES];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * 128;
  const int bh = blockIdx.y;
  // ONE: the host launches it only for nk <= 128, so there is one KV tile; as a constant it lets the compiler see that
  // O is still zero while S is computed, instead of keeping (or spilling) its registers across that wgmma chain
  const int T = ONE ? 1 : (p.nk + C::BKV - 1) / C::BKV;

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    mbar_init(&q_full, 1);
    for (int s = 0; s < C::STAGES; ++s) {
      mbar_init(&kv_full[s], 1);
      mbar_init(&kv_empty[s], 8);     // one arrival per consumer warp
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();               // Q / K / V^T come from the previous kernel in the stream
  pdl_launch_dependents();

  if (warp >= 8) {
    // ================================================================= TMA producer
    if constexpr (!ONE) asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory");
    if (warp == 8 && lane == 0) {
      mbar_expect_tx(&q_full, C::Q_BYTES);
#pragma unroll
      for (int c = 0; c < C::QCH; ++c) tma_load_3d(sQ + c * 16384, &tmQ, &q_full, c * 64, q0, bh);
      int st = 0;
      uint32_t ph = 0;
      for (int j = 0; j < T; ++j) {
        mbar_wait_hint(&kv_empty[st], ph ^ 1);
        uint8_t* sK = sKV + st * (C::K_BYTES + C::V_BYTES);
        uint8_t* sV = sK + C::K_BYTES;
        mbar_expect_tx(&kv_full[st], C::K_BYTES + C::V_BYTES);
#pragma unroll
        for (int c = 0; c < C::QCH; ++c)
          tma_load_3d(sK + c * (C::BKV * 128), &tmK, &kv_full[st], c * 64, j * C::BKV, bh);
#pragma unroll
        for (int c = 0; c < C::KVCH; ++c)
          tma_load_3d(sV + c * (C::DV * 128), &tmV, &kv_full[st], j * C::BKV + c * 64, 0, bh);
        if (++st == C::STAGES) {
          st = 0;
          ph ^= 1;
        }
      }
    }
    return;
  }

  // =================================================================== consumers: rows rA, rA + 8 of the tile
  if constexpr (!ONE) asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n" ::: "memory");
  const int wg = warp >> 2;
  const int rA = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const int cq = 2 * (lane & 3);
  const int b = bh / p.heads, h = bh - b * p.heads;
  mbar_wait(&q_full, 0);
  const uint64_t qdesc = make_desc_sw128(smem_u32(sQ + wg * (64 * 128)));

  if constexpr (!ONE) {
    AttnPipe<D, F16> pp;
    pp.sKV = sKV;
    pp.kv_full = kv_full;
    pp.kv_empty = kv_empty;
    pp.qdesc = qdesc;
    pp.c = p.scale_log2;
    pp.cq = cq;
    pp.lane = lane;
    pp.st = 0;
    pp.ph = 0;
#pragma unroll
    for (int i = 0; i < NO; ++i) pp.o[i] = 0.f;
    pp.m[0] = pp.m[1] = -INFINITY;
    pp.l[0] = pp.l[1] = 0.f;
    // T >= 2: the host sends nk <= 128 to the single-tile kernel
    const int last_valid = p.nk - (T - 1) * C::BKV;
    pp.template step<false, false>(C::BKV);
    for (int j = 1; j < T - 1; ++j) pp.template step<true, false>(C::BKV);
    pp.template step<true, true>(last_valid);
    pp.finish(last_valid);
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const int q_idx = q0 + rA + 8 * hr;
      const float lt = quad_sum(pp.l[hr]);     // all lanes of the warp, before any of them leaves
      const float inv = 1.0f / lt;
      if (q_idx >= p.nq) continue;
      if (p.lse2 != nullptr && (lane & 3) == 0) p.lse2[(long long)bh * p.nq + q_idx] = pp.m[hr] + log2f(lt);
      __nv_bfloat16* orow = p.out + ((long long)b * p.nq + q_idx) * p.ldo + h * D;
#pragma unroll
      for (int i = 0; i < C::DV / 8; ++i) {
        const int col = 8 * i + cq;
        if (col < D)
          *reinterpret_cast<uint32_t*>(orow + col) =
              pack16x2<F16>(pp.o[4 * i + 2 * hr] * inv, pp.o[4 * i + 2 * hr + 1] * inv);
      }
    }
    return;
  } else {
    // ---- single KV tile: S, softmax (+ probs / pcols), O = P V
    const float c = p.scale_log2;
    const bool want_pc = p.pcols != nullptr;
    int pos0 = -1, pos1 = -1;
    if (want_pc) {
      const int bb = bh / p.heads;
      pos0 = __ldg(p.pos + bb * 2);
      pos1 = __ldg(p.pos + bb * 2 + 1);
    }
    float o[NO];
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f}, pc[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
    mbar_wait(&kv_full[0], 0);
    uint8_t* sK = sKV;
    uint8_t* sV = sK + C::K_BYTES;
    float s[NS];
#pragma unroll
    for (int i = 0; i < NS; ++i) s[i] = 0.f;
    wgmma_fence_regs(s);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < C::KSTEPS; ++kk) {
      const uint64_t kd = make_desc_sw128(smem_u32(sK + (kk >> 2) * (C::BKV * 128)));
      wgmma_ss<C::BKV, F16>(s, qdesc + (kk >> 2) * (16384 >> 4) + 2 * (kk & 3), kd + 2 * (kk & 3), 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(s);
    // ---- softmax (log2 domain); masked columns -> probability 0
    const int kv_valid = p.nk;
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const int q_idx = q0 + rA + 8 * hr;
      const int row_lim = CAUSAL ? max(0, min(kv_valid, q_idx + 1)) : kv_valid;
      float mx = -INFINITY;
#pragma unroll
      for (int i = 0; i < C::BKV / 8; ++i)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = 8 * i + cq + e;
          float& x = s[4 * i + 2 * hr + e];
          x = col < row_lim ? x * c : -INFINITY;
          mx = fmaxf(mx, x);
        }
      mx = quad_max(mx);
      const float m_use = mx == -INFINITY ? 0.f : mx;   // fully masked row: keep everything at 0
      m[hr] = mx;
      float rs = 0.f;
#pragma unroll
      for (int i = 0; i < C::BKV / 8; ++i)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float& x = s[4 * i + 2 * hr + e];
          x = ex2_approx(x - m_use);
          rs += x;
          if (want_pc) {
            const int kcol = 8 * i + cq + e;
            if (kcol == pos0) pc[hr][0] += x;
            if (kcol == pos1) pc[hr][1] += x;
          }
        }
      l[hr] = rs;
    }
    if (p.probs != nullptr) {
      // normalised probabilities for the attention controller (edlora.py:81-82)
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        const int q_idx = q0 + rA + 8 * hr;
        const float inv = 1.0f / quad_sum(l[hr]);
        if (q_idx < p.nq) {
          float* prow = p.probs + ((long long)bh * p.nq + q_idx) * p.nk;
#pragma unroll
          for (int i = 0; i < C::BKV / 8; ++i)
#pragma unroll
            for (int e = 0; e < 2; ++e)
              if (8 * i + cq + e < kv_valid) prow[8 * i + cq + e] = s[4 * i + 2 * hr + e] * inv;
        }
      }
    }
    // ---- O = P V (P from registers; k-steps past the last valid key are skipped: those columns of V^T may be padding).
    // O is zeroed only here, so its registers are not live across the S chain.
    const int ksteps = (kv_valid + 15) >> 4;
    uint32_t pa[C::BKV / 16][4];
#pragma unroll
    for (int kk = 0; kk < C::BKV / 16; ++kk) frag_to_a<F16>(&s[8 * kk], pa[kk]);
#pragma unroll
    for (int i = 0; i < NO; ++i) o[i] = 0.f;
    wgmma_fence_regs(o);
    pv_dispatch<C::BKV / 16, C::DV, F16>(ksteps, o, pa, sV);
    // ---- normalise and write the two rows
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const int q_idx = q0 + rA + 8 * hr;
      const float lt = quad_sum(l[hr]);
      const float inv = 1.0f / lt;
      if (want_pc) {
        const float p0 = quad_sum(pc[hr][0]), p1 = quad_sum(pc[hr][1]);
        if (q_idx < p.nq && (lane & 3) == 0)
          *reinterpret_cast<float2*>(p.pcols + ((long long)bh * p.nq + q_idx) * 2) = make_float2(p0 * inv, p1 * inv);
      }
      if (q_idx >= p.nq) continue;
      if (p.lse2 != nullptr && (lane & 3) == 0) p.lse2[(long long)bh * p.nq + q_idx] = m[hr] + log2f(lt);
      __nv_bfloat16* orow = p.out + ((long long)b * p.nq + q_idx) * p.ldo + h * D;
#pragma unroll
      for (int i = 0; i < C::DV / 8; ++i) {
        const int col = 8 * i + cq;
        if (col < D)
          *reinterpret_cast<uint32_t*>(orow + col) = pack16x2<F16>(o[4 * i + 2 * hr] * inv, o[4 * i + 2 * hr + 1] * inv);
      }
    }
  }
}

template <int D, bool ONE, bool CAUSAL = false, bool F16 = false>
static int launch_attn(const void* Q, const void* K, const void* Vt, void* out, int64_t ldo, float* probs, int BH,
                       int heads, int nq, int nk, int nk8, float scale, cudaStream_t stream, float* lse2 = nullptr,
                       float* pcols = nullptr, const int* pos = nullptr) {
  using C = AttnCfg<D, ONE>;
  CUtensorMap tmQ, tmK, tmV;
  {
    uint64_t dims[3] = {(uint64_t)C::DP, (uint64_t)nq, (uint64_t)BH};
    uint64_t str[2] = {(uint64_t)C::DP * 2, (uint64_t)nq * C::DP * 2};
    uint32_t box[3] = {64, 128, 1};
    int rc = encode_tmap(&tmQ, Q, 2, 3, dims, str, box, 3);
    if (rc) return rc;
  }
  {
    uint64_t dims[3] = {(uint64_t)C::DP, (uint64_t)nk, (uint64_t)BH};
    uint64_t str[2] = {(uint64_t)C::DP * 2, (uint64_t)nk * C::DP * 2};
    uint32_t box[3] = {64, (uint32_t)C::BKV, 1};
    int rc = encode_tmap(&tmK, K, 2, 3, dims, str, box, 3);
    if (rc) return rc;
  }
  {
    uint64_t dims[3] = {(uint64_t)nk8, (uint64_t)C::DV, (uint64_t)BH};
    uint64_t str[2] = {(uint64_t)nk8 * 2, (uint64_t)C::DV * nk8 * 2};
    uint32_t box[3] = {64, (uint32_t)C::DV, 1};
    int rc = encode_tmap(&tmV, Vt, 2, 3, dims, str, box, 3);
    if (rc) return rc;
  }
  AttnDev p;
  p.nq = nq;
  p.nk = nk;
  p.heads = heads;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.out = reinterpret_cast<__nv_bfloat16*>(out);
  p.ldo = ldo;
  p.probs = probs;
  p.lse2 = lse2;
  p.pcols = pcols;
  p.pos = pos;
  static bool configured = false;
  if (!configured) {
    MOS_CHECK_CUDA(cudaFuncSetAttribute(attn_kernel<D, ONE, CAUSAL, F16>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES));
    configured = true;
  }
  dim3 grid((unsigned)ceil_div(nq, 128), (unsigned)BH);
  MOS_CHECK_CUDA(launch_pdl(attn_kernel<D, ONE, CAUSAL, F16>, grid, dim3(attn_threads<ONE>()), (size_t)C::SMEM_BYTES, stream, tmQ, tmK, tmV, p));
  return MOS_OK;
}

}  // namespace mos

using namespace mos;

extern "C" int mos_attention_fwd(const void* Q, const void* K, const void* Vt, void* out, int64_t ldo, float* probs,
                                 int32_t batch, int32_t heads, int32_t head_dim, int32_t nq, int32_t nk,
                                 int32_t nk8, float scale, int32_t act_dtype, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  MOS_CHECK_ARG(Q && K && Vt && out, "mos_attention_fwd: NULL pointer");
  MOS_CHECK_ARG(batch > 0 && heads > 0 && nq > 0 && nk > 0, "mos_attention_fwd: bad shape");
  MOS_CHECK_ARG(nk8 >= nk && nk8 % 8 == 0, "mos_attention_fwd: nk8=%d must be >= nk=%d and a multiple of 8", nk8, nk);
  MOS_CHECK_ARG(ldo >= (int64_t)heads * head_dim && ldo % 8 == 0, "mos_attention_fwd: bad ldo");
  MOS_CHECK_DTYPE(act_dtype, "mos_attention_fwd");
  const int BH = batch * heads;
  if (probs) MOS_CHECK_ARG(nk <= 128, "mos_attention_fwd: probs output needs a single kv tile (nk <= 128)");
#define MOS_ATTN(D_, ONE_)                                                                                             \
  (act_dtype == MOS_DT_F16                                                                                             \
       ? launch_attn<D_, ONE_, false, true>(Q, K, Vt, out, ldo, probs, BH, heads, nq, nk, nk8, scale, stream)         \
       : launch_attn<D_, ONE_, false, false>(Q, K, Vt, out, ldo, probs, BH, heads, nq, nk, nk8, scale, stream))
  switch (head_dim) {
    case 40: return nk <= 128 ? MOS_ATTN(40, true) : MOS_ATTN(40, false);
    case 80: return nk <= 128 ? MOS_ATTN(80, true) : MOS_ATTN(80, false);
    case 160: return nk <= 128 ? MOS_ATTN(160, true) : MOS_ATTN(160, false);
    default: return set_err(MOS_EUNSUPPORTED, "mos_attention_fwd: head_dim %d not in {40, 80, 160}", head_dim);
  }
#undef MOS_ATTN
}


// Training forward: same kernel, additionally saves the log2-domain log-sum-exp [B*H, nq] for mos_attention_bwd and
// (cross-attention, nk <= 128) the per-head probabilities at the two concept-token columns pos[b][0..1] -> pcols
// [B*H, nq, 2] for the attention regulariser (trainer_edlora.py:263-313).
extern "C" int mos_attention_fwd_train(const void* Q, const void* K, const void* Vt, void* out, int64_t ldo, float* lse2,
                                       float* pcols, const int32_t* pos, int32_t batch, int32_t heads,
                                       int32_t head_dim, int32_t nq, int32_t nk, int32_t nk8, float scale,
                                       void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  MOS_CHECK_ARG(Q && K && Vt && out && lse2, "mos_attention_fwd_train: NULL pointer");
  MOS_CHECK_ARG(batch > 0 && heads > 0 && nq > 0 && nk > 0, "mos_attention_fwd_train: bad shape");
  MOS_CHECK_ARG(nk8 >= nk && nk8 % 8 == 0, "mos_attention_fwd_train: nk8 must be >= nk and a multiple of 8");
  MOS_CHECK_ARG(ldo >= (int64_t)heads * head_dim && ldo % 8 == 0, "mos_attention_fwd_train: bad ldo");
  MOS_CHECK_ARG(!pcols == !pos, "mos_attention_fwd_train: pcols and pos go together");
  if (pcols) MOS_CHECK_ARG(nk <= 128, "mos_attention_fwd_train: pcols needs a single kv tile (nk <= 128)");
  const int BH = batch * heads;
  const int* ip = reinterpret_cast<const int*>(pos);
  switch (head_dim) {
    case 40:
      if (nk <= 128)
        return launch_attn<40, true>(Q, K, Vt, out, ldo, nullptr, BH, heads, nq, nk, nk8, scale, stream, lse2, pcols, ip);
      return launch_attn<40, false>(Q, K, Vt, out, ldo, nullptr, BH, heads, nq, nk, nk8, scale, stream, lse2, pcols, ip);
    case 80:
      if (nk <= 128)
        return launch_attn<80, true>(Q, K, Vt, out, ldo, nullptr, BH, heads, nq, nk, nk8, scale, stream, lse2, pcols, ip);
      return launch_attn<80, false>(Q, K, Vt, out, ldo, nullptr, BH, heads, nq, nk, nk8, scale, stream, lse2, pcols, ip);
    case 160:
      if (nk <= 128)
        return launch_attn<160, true>(Q, K, Vt, out, ldo, nullptr, BH, heads, nq, nk, nk8, scale, stream, lse2, pcols, ip);
      return launch_attn<160, false>(Q, K, Vt, out, ldo, nullptr, BH, heads, nq, nk, nk8, scale, stream, lse2, pcols, ip);
    default: return set_err(MOS_EUNSUPPORTED, "mos_attention_fwd_train: head_dim %d not in {40, 80, 160}", head_dim);
  }
}

// Causal self-attention over one key tile (nq == nk <= 128): the CLIP text encoder's attention (77 tokens; 12 heads of 64
// dims run as head_dim 80 with zero-padded columns and scale = 64^-0.5).  Reference: transformers CLIPTextModel as called
// at mixofshow/pipelines/pipeline_edlora.py:133-145 and trainer_edlora.py:220-234.
extern "C" int mos_attention_fwd_causal(const void* Q, const void* K, const void* Vt, void* out, int64_t ldo, int32_t batch,
                                        int32_t heads, int32_t head_dim, int32_t n, int32_t n8, float scale,
                                        float* lse2, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  MOS_CHECK_ARG(Q && K && Vt && out, "mos_attention_fwd_causal: NULL pointer");
  MOS_CHECK_ARG(batch > 0 && heads > 0 && n > 0 && n <= 128, "mos_attention_fwd_causal: needs 0 < n <= 128 (one key tile)");
  MOS_CHECK_ARG(n8 >= n && n8 % 8 == 0, "mos_attention_fwd_causal: n8 must be >= n and a multiple of 8");
  MOS_CHECK_ARG(ldo >= (int64_t)heads * head_dim && ldo % 8 == 0, "mos_attention_fwd_causal: bad ldo");
  if (head_dim != 80) return set_err(MOS_EUNSUPPORTED, "mos_attention_fwd_causal: head_dim %d (only 80 is built)", head_dim);
  return launch_attn<80, true, true>(Q, K, Vt, out, ldo, nullptr, batch * heads, heads, n, n, n8, scale, stream, lse2);
}
