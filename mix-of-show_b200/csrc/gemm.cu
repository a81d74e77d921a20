// gemm.cu — K1/K4: warp-specialised wgmma GEMM and implicit-GEMM 3x3 convolution for sm_90a.
//
//   out[m,n] = epilogue( sum_k A[m,k] W[n,k] )        A, W 16-bit K-major; fp32 accumulation in registers
//
// Persistent kernel: one CTA per SM loops over 128 x 160 output tiles (160 divides every SD1.5 channel count).
// Roles (256 + 32 threads):
//   warps 0..7  two consumer warpgroups, 64 tile rows each: wgmma m64n160k16 (A and W from shared memory), then the fused
//               epilogue from the accumulator registers into the staging tile (16-bit row output)
//   warp 8      TMA producer   cp.async.bulk.tensor -> 128B-swizzled smem ring, mbarrier complete_tx; it runs ahead into
//               the next tile while the consumers are in their epilogue.  16-bit row output: after a tile's last k block
//               it loads the tile's residual into the staging tile, and once the consumers have filled the staging tile
//               it writes it out with TMA stores (rows past M / H / B are clipped by the tensor map bounds).  Head-split
//               output (Q/K rows, V^T) is written the same way, one tensor map per segment (tmO, tmR, tmS).
// LoRA fusion (edlora.py:244-246): the rank-padded down matrix [16, K] rides along as 16 extra W rows of the stage, and a
// second wgmma (m64n16k16) on the same A descriptor produces t = x * down^T; the epilogue adds t * (alpha*up)^T.
// Convolution: the A tile is a TW x TH x TB pixel patch of the NHWC activation fetched by a 4-D tensor map at
// the tap-shifted coordinate; TMA out-of-bounds zero fill implements the padding.
#include <stdlib.h>

#include "common.h"
#include "tc.cuh"

namespace mos {

constexpr int BM = 128;
constexpr int BN = 160;
constexpr int BK = 64;
constexpr int LORA_N = 16;
constexpr int MAX_STAGES = 8;
constexpr int A_STAGE_BYTES = BM * BK * 2;               // 16384
constexpr int B_STAGE_BYTES = BN * BK * 2;               // 20480
constexpr int CONSUMER_THREADS = 256;                    // two warpgroups
constexpr int NUM_THREADS = CONSUMER_THREADS + 32;       // + the TMA producer warp
constexpr int PRODUCER_WARP = CONSUMER_THREADS / 32;
constexpr int MAX_DYN_SMEM = 227 * 1024 - 6144;  // leave room for the static epilogue operands and barriers
constexpr int EPI_BATCHES = 5;   // batches one 128-row tile can span (plain: rows_per_batch >= 32; conv: TB <= 4)
// Staging tile of the 16-bit row output: 5 column boxes of [128 rows][w columns], w = 32 (row output, SWIZZLE_64B) or
// 16 (GEGLU's 80 output columns, SWIZZLE_32B), each box the smem image of one TMA store / residual load.
constexpr int EPI_BYTES = BM * BN * 2;                   // 40960
constexpr int EPI_BOXES = 5;
constexpr int EPI_LGW_ROWS = 5;                          // log2 of the box width: row output
constexpr int EPI_LGW_GEGLU = 4;                         // GEGLU (80 output columns per tile)

struct GemmDev {
  int M, N;
  int kb_total;        // number of 64-wide k blocks over the whole reduction (conv: 9 * C/64)
  int kb_per_split;
  int stages;
  int conv, H, W, B, kc_per_tap, TW, TH, TB, lgTW, lgTH, tiles_w, tiles_h;
  int geglu;
  int out_mode;
  int splits;
  int n_tiles, m_tiles, total_items, nbatch;
  float* partial;
  const float* bias;
  const float* bias_batch;
  long long rows_per_batch;
  long long bias_batch_ld;
  const __nv_bfloat16* residual;
  long long ldr;
  const float* lora_up;
  long long lora_seg;
  void* out;
  long long ldc;
  void* seg_ptr[3];
  int seg_kind[3];
  long long seg_rows_pad[3];
  int heads, head_dim, dpad, dv_pad;
  long long tokens_per_batch;
  int accum;           // MOS_OUT_F32: out += result (Gram accumulation)
  int epi_tma;         // 16-bit row output TMA can address: staged epilogue written by TMA stores (tensor map tmO)
  int res_tma;         // epi_tma and the residual is prefetched into the staging tile by TMA (tensor map tmR)
  int epi_lgw;         // log2 of the staging box width in columns (EPI_LGW_ROWS, EPI_LGW_GEGLU)
  int epi_heads;       // epi_tma for head-split output: copy-out staging layout, one tensor map per segment (tmO, tmR, tmS)
  int nseg;            // head-split segments (N / (heads * head_dim))
  int epi_copy;        // other 16-bit output (head-split, unaligned rows): staged epilogue, copied out by the consumers
  int epi_mode;        // EpiMode of the launch's tiles
  unsigned long long* tl;   // optional timeline buffer (mos_debug_set_timeline)
  int* counters;       // split-K with in-kernel finalize: one arrival counter per output tile (zero between launches)
  const uint8_t* pf;   // optional: bytes to pull into L2 for a LATER launch (the next layer's weights), see mos_gemm_args
  long long pf_bytes;
};

__device__ __forceinline__ void epi_bar() {  // consumer warps only
  asm volatile("bar.sync 1, %0;" ::"n"(CONSUMER_THREADS) : "memory");
}

// ---- optional in-kernel timeline (profiling aid): when a buffer is registered through mos_debug_set_timeline, the
// first 8 CTAs of every gemm launch record %globaltimer stamps (ns) at their phase boundaries, TL_SLOTS per CTA:
//   0 CTA start, 1 barriers initialised, 2 producer start, 3 first k block landed (consumer)
//   first tile:  4 accumulators ready, 6 epilogue operands in shared memory, 7 epi_ready passed, 8 staging tile
//                written (epi_full arrived), 9 epi_full observed by the producer, 10 stores issued, 5 tile written
//   second tile: 11 accumulators ready, 12 operands in shared memory, 13 epi_ready passed, 14 staging tile written,
//                15 tile written  The pointer travels in
// the kernel parameters (constant bank): a __device__ global would cost an L2 round trip at every stamp site.
constexpr int TL_SLOTS = 16;
#define stamp(slot)                                                       \
  do {                                                                    \
    if (p.tl != nullptr && blockIdx.x < 8) {                              \
      unsigned long long t_;                                              \
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_));              \
      p.tl[blockIdx.x * TL_SLOTS + (slot)] = t_;                          \
    }                                                                     \
  } while (0)

struct TileCoord {
  int n0, m0, cb0, ch0, cw0, split;
};
// work item ws -> its 128 x 160 tile and k split
__device__ __forceinline__ TileCoord item_coord(const GemmDev& p, int ws) {
  TileCoord t;
  t.split = ws % p.splits;
  const int tt = ws / p.splits;
  const int tn = tt % p.n_tiles;
  const int tm = tt / p.n_tiles;
  t.n0 = tn * BN;
  t.m0 = tm * BM;
  t.cb0 = t.ch0 = t.cw0 = 0;
  if (p.conv) {
    t.cw0 = (tm % p.tiles_w) * p.TW;
    t.ch0 = ((tm / p.tiles_w) % p.tiles_h) * p.TH;
    t.cb0 = (tm / (p.tiles_w * p.tiles_h)) * p.TB;
  }
  return t;
}
// row r of a tile -> global output row m (and validity)
__device__ __forceinline__ bool row_coord(const GemmDev& p, const TileCoord& t, int r, long long& m, int& b) {
  if (p.conv) {
    const int tw = r & (p.TW - 1), th = (r >> p.lgTW) & (p.TH - 1), tb = r >> (p.lgTW + p.lgTH);
    b = t.cb0 + tb;
    const int h = t.ch0 + th, w = t.cw0 + tw;
    m = ((long long)b * p.H + h) * p.W + w;
    return (b < p.B) && (h < p.H);
  }
  m = (long long)t.m0 + r;
  b = (int)(m / p.rows_per_batch);
  return m < p.M;
}

// Copy-out staging layout (head-split output, and row output whose destination TMA cannot address): 20 regions of 2 KB,
// one per 8-column group.  Row-major groups hold row r's 8 columns at r * 16: the smem image of an (8 columns, 128 rows)
// TMA box.  Transposed groups (V^T columns) hold two 1 KB halves of 64 rows; in a half, column c's 64 rows are a 128-byte
// line of 8 chunks of 8 rows at c % 8 * 128, chunk index XOR-ed with c % 8: the SWIZZLE_128B smem image of a (64 rows,
// 8 columns) TMA box.  Both the fragment writes and the 16-byte chunk reads of a warp touch distinct banks.
__device__ __forceinline__ uint32_t cp_off(int r, int c, bool tr) {
  const int k = c >> 3, cc = c & 7;
  return tr ? (k << 11) + ((r >> 6) << 10) + (cc << 7) + ((((r >> 3) ^ cc) & 7) << 4) + ((r & 7) << 1)
            : (k << 11) + (r << 4) + (cc << 1);
}
// head-split output: bit k is set when 8-column group k of the tile at column n0 belongs to a V^T segment
__device__ __forceinline__ uint32_t transposed_groups(const GemmDev& p, int n0) {
  if (p.out_mode != MOS_OUT_HEADS) return 0u;
  const int seg_len = p.heads * p.head_dim;
  int seg = n0 / seg_len, c = n0 - seg * seg_len;
  uint32_t mask = 0;
#pragma unroll 1
  for (int k = 0; k < BN / 8; ++k) {
    if (p.seg_kind[seg] == MOS_SEG_TRANSPOSED) mask |= 1u << k;
    if ((c += 8) == seg_len) {
      c = 0;
      ++seg;
    }
  }
  return mask;
}
// destination of the 16-bit output element (row m, tile column c) of the tile at t
__device__ __forceinline__ uint16_t* out_elem(const GemmDev& p, const TileCoord& t, long long m, int c) {
  if (p.out_mode != MOS_OUT_HEADS)
    return reinterpret_cast<uint16_t*>(p.out) + m * p.ldc + (p.geglu ? t.n0 / 2 : t.n0) + c;
  const int nc = t.n0 + c;
  const int seg_len = p.heads * p.head_dim;
  const long long bb = m / p.tokens_per_batch;
  const long long tok = m - bb * p.tokens_per_batch;
  const int seg = nc / seg_len;
  const int cc2 = nc - seg * seg_len;
  const int head = cc2 / p.head_dim;
  const int j = cc2 - head * p.head_dim;
  uint16_t* base = reinterpret_cast<uint16_t*>(p.seg_ptr[seg]);
  const long long bh = bb * p.heads + head;
  if (p.seg_kind[seg] == MOS_SEG_ROWS) return base + (bh * p.seg_rows_pad[seg] + tok) * p.dpad + j;
  return base + (bh * p.dv_pad + j) * p.seg_rows_pad[seg] + tok;
}

// bias (+ per-batch bias) of output column n for a row of batch b
__device__ __forceinline__ float col_bias(const GemmDev& p, int b, int n) {
  float v = p.bias ? __ldg(p.bias + n) : 0.f;
  if (p.bias_batch) v += __ldg(p.bias_batch + (long long)b * p.bias_batch_ld + n);
  return v;
}
// LoRA: the rank values t[4 seg .. 4 seg + 3] (segment seg = 0..3) of tile row rA + 8 hr.  The 16 values of a row lie in
// the LoRA accumulator fragment of the 4 lanes of a quad: t[8h + 2s + e] = lacc[4h + 2hr + e] of quad lane s.  The quad
// shares its row, so it is either wholly inside the output or wholly outside: the shuffles name only its 4 lanes.  Only
// compile-time indices into lacc (selects), so that nothing lives in local memory.
__device__ __forceinline__ float4 lora_ranks(const float (&lacc)[LORA_N / 2], int hr, int seg, int lane) {
  const unsigned quad = 0xFu << (lane & ~3);
  const bool hi = seg >= 2;
  const float v0 = hi ? (hr ? lacc[6] : lacc[4]) : (hr ? lacc[2] : lacc[0]);
  const float v1 = hi ? (hr ? lacc[7] : lacc[5]) : (hr ? lacc[3] : lacc[1]);
  const int s = 2 * (seg & 1);
  return make_float4(__shfl_sync(quad, v0, s, 4), __shfl_sync(quad, v1, s, 4), __shfl_sync(quad, v0, s + 1, 4),
                     __shfl_sync(quad, v1, s + 1, 4));
}
// acc[i0 + 2 hr] for the tile row rA + 8 hr: a select between two compile-time indices, so that the epilogue's row loop
// needs no unrolling and nothing lives in local memory
__device__ __forceinline__ float frag(const float (&acc)[BN / 2], int i0, int hr) { return hr ? acc[i0 + 2] : acc[i0]; }
// LoRA term of an output column: t[4 ranks of the column's segment] . (alpha * up)[column]
__device__ __forceinline__ float lora_term(float4 t, float4 u) { return t.x * u.x + t.y * u.y + t.z * u.z + t.w * u.w; }

// Output path of a tile's epilogue, fixed per launch by the host (GemmDev::epi_mode), except EPI_HEADS_T, which a
// head-split tile takes when one of its 8-column groups belongs to a V^T segment.
enum EpiMode {
  EPI_ROWS,              // 16-bit rows (also head-split Q/K rows) into the staging tile
  EPI_ROWS_RES_SMEM,     // + residual, prefetched into the staging tile by TMA
  EPI_ROWS_RES_GLOBAL,   // + residual, read from global memory (TMA cannot address it)
  EPI_HEADS_T,           // head-split, copy-out layout, V^T groups transposed
  EPI_GEGLU,             // a * gelu(gate) rows (80 of the tile's 160 columns)
  EPI_F32,               // fp32 rows to global (optionally accumulated)
  EPI_PARTIAL,           // split-K fp32 partial tile to the workspace
};

struct EpiArgs {
  uint8_t* epi;          // staging tile
  const float* s_bias;   // [EPI_BATCHES][BN]
  const float4* s_lup;   // [BN] (LoRA)
  int rA, cq, lane, b_lo;
};

// Staging layouts of 16-bit row output (byte offset of tile row r, column c = 8i + cq; the fragment of group i holds
// columns 8i + cq, 8i + cq + 1):
//  - column boxes (TMA-store row output): box c / w of [128 rows][w columns], w = 1 << EPI_LGW_ROWS (32) or
//    1 << EPI_LGW_GEGLU (16), rows of 2w bytes, the 16-byte chunk index XOR-ed with address bits [7, 7 + log2(w/8)) of
//    the row: the TMA SWIZZLE_64B / SWIZZLE_32B pattern.  A warp's store of one fragment column pair (8 rows x 16 bytes)
//    then touches 32 distinct banks.
//  - copy-out groups (cp_off): 2 KB per 8-column group.
// Either way the offset of group i is base[i % G] + (i / G) * (G * 2 KB), G = w / 8 groups per box, with the G bases
// worked out once per row.
template <int LGW>
__device__ __forceinline__ void staging_bases(uint32_t (&base)[(1 << LGW) / 8], bool box, int r, int cq) {
  constexpr int G = (1 << LGW) / 8;
  static_assert(G * 2048 == BM * (1 << LGW) * 2, "a box of G groups is G copy-out groups");
  const uint32_t bx = (r << (LGW + 1)) | (((r >> (6 - LGW)) & (G - 1)) << 4) | (cq << 1);
#pragma unroll
  for (int k = 0; k < G; ++k) base[k] = box ? bx ^ (k << 4) : cp_off(r, 8 * k + cq, false);
}

// Epilogue of one tile from the accumulator fragment: d[4i + 2hr + e] = (row rA + 8 hr, column 8i + cq + e).  Every
// index into acc / lacc is a compile-time constant.  The bias and LoRA terms of a column group are added by one piece of
// code shared by every path that takes them; the group's store is its path's own compile-time instantiation
// (epi_store<MODE>, no runtime tests inside), picked by warp-uniform branches.  These also keep each group's
// shared-memory operand reads next to the group's store: hoisted above all 20 stores, they would hold 40 registers.
struct EpiRow {
  uint32_t base[(1 << EPI_LGW_ROWS) / 8];   // staging_bases of the row
  uint32_t tbase0, tbase1;                 // V^T groups (EPI_HEADS_T): column cq + e, 2-byte stores (cp_off transposed)
  const __nv_bfloat16* res;                // EPI_ROWS_RES_GLOBAL: residual of column n0 + cq
  float* fout;                             // EPI_F32: output of column n0 + cq
};
template <int MODE, bool F16>
__device__ __forceinline__ void epi_store(const GemmDev& p, const EpiArgs& ea, const EpiRow& er, int i, float o0, float o1,
                                          uint32_t trmask) {
  constexpr int G = (1 << EPI_LGW_ROWS) / 8;
  uint8_t* dst = ea.epi + er.base[i % G] + (i / G) * (G << 11);
  if constexpr (MODE == EPI_F32) {
    float2* d2 = reinterpret_cast<float2*>(er.fout + 8 * i);
    float2 r2 = make_float2(o0, o1);
    if (p.accum) {
      const float2 old = *d2;
      r2.x += old.x;
      r2.y += old.y;
    }
    *d2 = r2;
    return;
  }
  if constexpr (MODE == EPI_ROWS_RES_SMEM || MODE == EPI_ROWS_RES_GLOBAL) {
    const float2 f = unpack16x2<F16>(MODE == EPI_ROWS_RES_SMEM ? *reinterpret_cast<const uint32_t*>(dst)
                                                               : *reinterpret_cast<const uint32_t*>(er.res + 8 * i));
    o0 += f.x;
    o1 += f.y;
  }
  const uint32_t v = pack16x2<F16>(o0, o1);
  if (MODE == EPI_HEADS_T && ((trmask >> i) & 1u)) {
    *reinterpret_cast<uint16_t*>(ea.epi + er.tbase0 + (i << 11)) = (uint16_t)(v & 0xFFFFu);
    *reinterpret_cast<uint16_t*>(ea.epi + er.tbase1 + (i << 11)) = (uint16_t)(v >> 16);
  } else {
    *reinterpret_cast<uint32_t*>(dst) = v;
  }
}

template <bool F16, bool LORA>
__device__ __forceinline__ void epilogue(const GemmDev& p, const TileCoord& t, const EpiArgs& ea,
                                         const float (&acc)[BN / 2],
                                         const float (&lacc)[LORA_N / 2], uint32_t trmask, int mode) {
  // LoRA segment of the tile's first column, and that column's offset inside it.  Segments and tiles start at
  // multiples of 16 columns, so a segment can only change at an even group.
  const int lseg = (int)p.lora_seg;
  const int lseg0 = LORA ? t.n0 / lseg : 0;
  const int lcol0 = t.n0 - lseg0 * lseg;
  // The two rows of the thread share one copy of the code (not unrolled): in the denoise step every GEMM launch follows
  // other kernels and runs its once-per-tile epilogue from a cold instruction cache, so the code's size costs time.
  // Rolled, the variants are 20-30 % smaller and the step's GEMM time drops from 5.0 to 4.65 ms (H100, 700 W).
#pragma unroll 1
  for (int hr = 0; hr < 2; ++hr) {
    const int r = ea.rA + 8 * hr;
    long long m;
    int b;
    if (!row_coord(p, t, r, m, b)) continue;
    const float* sb = ea.s_bias + (p.bias_batch ? b - ea.b_lo : 0) * BN + ea.cq;   // s_bias slot of the row
    const float4* su = ea.s_lup + ea.cq;
    if (mode == EPI_PARTIAL) {                      // (the host rejects LoRA together with split-K)
      if constexpr (!LORA) {
        float* dst = p.partial + ((long long)t.split * p.M + m) * p.N + t.n0 + ea.cq;
#pragma unroll
        for (int i = 0; i < BN / 8; ++i)
          *reinterpret_cast<float2*>(dst + 8 * i) = make_float2(frag(acc, 4 * i, hr), frag(acc, 4 * i + 1, hr));
      }
      continue;
    }
    if (mode == EPI_GEGLU) {
      // tile columns [0,80) = a, [80,160) = gate for the same 80 outputs (columns n0/2 + [0,80) of the output)
      constexpr int G = (1 << EPI_LGW_GEGLU) / 8;
      uint32_t base[G];
      staging_bases<EPI_LGW_GEGLU>(base, p.epi_tma && !p.epi_heads, r, ea.cq);
      float4 t0 = make_float4(0.f, 0.f, 0.f, 0.f);
      if constexpr (LORA) t0 = lora_ranks(lacc, hr, 0, ea.lane);
#pragma unroll
      for (int i = 0; i < BN / 16; ++i) {
        float o[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float a = frag(acc, 4 * i + e, hr) + sb[8 * i + e];
          float g = frag(acc, 4 * (i + BN / 16) + e, hr) + sb[8 * i + BN / 2 + e];
          if constexpr (LORA) {
            a += lora_term(t0, su[8 * i + e]);
            g += lora_term(t0, su[8 * i + BN / 2 + e]);
          }
          o[e] = a * gelu_erf(g);
        }
        *reinterpret_cast<uint32_t*>(ea.epi + base[i % G] + (i / G) * (G << 11)) = pack16x2<F16>(o[0], o[1]);
      }
      continue;
    }
    // every other path: acc + bias (+ LoRA term), then the path's store
    EpiRow er;
    staging_bases<EPI_LGW_ROWS>(er.base, p.epi_tma && !p.epi_heads, r, ea.cq);
    er.tbase0 = cp_off(r, ea.cq, true);
    er.tbase1 = cp_off(r, ea.cq + 1, true);
    er.res = p.residual + m * p.ldr + t.n0 + ea.cq;
    er.fout = reinterpret_cast<float*>(p.out) + m * p.ldc + t.n0 + ea.cq;
    int seg = lseg0, scol = lcol0;                  // LoRA segment of group i, and the group pair's column inside it
    float4 tt = make_float4(0.f, 0.f, 0.f, 0.f);
    if constexpr (LORA) tt = lora_ranks(lacc, hr, seg, ea.lane);
#pragma unroll
    for (int i = 0; i < BN / 8; ++i) {
      float o[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) o[e] = frag(acc, 4 * i + e, hr) + sb[8 * i + e];
      if constexpr (LORA) {
        if (i > 0 && i % 2 == 0 && (scol += 16) == lseg) {   // seg is uniform over the warp
          scol = 0;
          tt = lora_ranks(lacc, hr, ++seg, ea.lane);
        }
#pragma unroll
        for (int e = 0; e < 2; ++e) o[e] += lora_term(tt, su[8 * i + e]);
      }
      // (direct branches on the uniform mode, in the order of how often the denoise step takes the paths: a jump
      // table's indirect branch per group costs more than the compares)
      if (mode == EPI_ROWS) epi_store<EPI_ROWS, F16>(p, ea, er, i, o[0], o[1], trmask);
      else if (mode == EPI_ROWS_RES_SMEM) epi_store<EPI_ROWS_RES_SMEM, F16>(p, ea, er, i, o[0], o[1], trmask);
      else if (mode == EPI_HEADS_T) epi_store<EPI_HEADS_T, F16>(p, ea, er, i, o[0], o[1], trmask);
      else if (mode == EPI_ROWS_RES_GLOBAL) epi_store<EPI_ROWS_RES_GLOBAL, F16>(p, ea, er, i, o[0], o[1], trmask);
      else epi_store<EPI_F32, F16>(p, ea, er, i, o[0], o[1], trmask);
    }
  }
}

// F16: 16-bit type of A, of the row / head-split outputs and of the residual (fp16 or bf16).
// LORA: the fused LoRA branch is present (a template parameter, so that the k16 wgmma chain of a k block is straight-line
// code in both variants: a runtime branch between two wgmmas makes ptxas serialise them).
template <bool F16, bool LORA>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
            const __grid_constant__ CUtensorMap tmL, const __grid_constant__ CUtensorMap tmO,
            const __grid_constant__ CUtensorMap tmR, const __grid_constant__ CUtensorMap tmS, const GemmDev p) {
  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment is required by SWIZZLE_128B (an offset from smem_raw, so that the compiler keeps the pointer in
  // the shared address space: the epilogue's staging stores then cannot alias global memory)
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  constexpr int stage_bytes = A_STAGE_BYTES + (LORA ? BN + LORA_N : BN) * 128;
  uint8_t* epi = smem + p.stages * stage_bytes;            // staging tile (p.epi_tma), 1024-byte aligned

  __shared__ uint64_t full_bar[MAX_STAGES];
  __shared__ uint64_t empty_bar[MAX_STAGES];
  __shared__ uint64_t epi_ready;   // producer -> consumers: the staging tile is free (and holds the tile's residual)
  __shared__ uint64_t epi_full;    // consumers -> producer: the staging tile holds the finished output tile
  // the tile's epilogue operands, loaded before its first store: bias + per-batch bias of the batches the tile spans
  // (col_bias), and the LoRA up rows (alpha * up)
  __shared__ float s_bias[EPI_BATCHES][BN];
  __shared__ float4 s_lup[LORA ? BN : 1];

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  if (threadIdx.x == 0) stamp(0);

  if (warp == PRODUCER_WARP && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if (LORA) tma_prefetch_desc(&tmL);
    if (p.epi_tma) {
      tma_prefetch_desc(&tmO);
      if (p.res_tma || (p.epi_heads && p.nseg > 1)) tma_prefetch_desc(&tmR);
      if (p.epi_heads && p.nseg > 2) tma_prefetch_desc(&tmS);
    }
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(&full_bar[s], 1);                          // one arrive.expect_tx by the producer
      mbar_init(&empty_bar[s], CONSUMER_THREADS / 32);     // one arrival per consumer warp
    }
    mbar_init(&epi_ready, 1);
    mbar_init(&epi_full, CONSUMER_THREADS);
    fence_barrier_init();
  }
  __syncthreads();

  // Everything above touched no global memory written by the previous kernel in the stream.
  if (threadIdx.x == 0) stamp(1);
  if (p.pf != nullptr && warp == PRODUCER_WARP && lane == 1) {
    // L2 staging of a later launch's weights (static data: no dependency on the previous kernel, so ahead of the wait):
    // this CTA's 1/gridDim slice, in 16 KB bulk prefetches.
    constexpr long long CH = 16384;
    const long long per = ((p.pf_bytes + gridDim.x - 1) / gridDim.x + CH - 1) / CH * CH;
    const long long lo = (long long)blockIdx.x * per, hi = min(p.pf_bytes, lo + per);
    for (long long off = lo; off < hi; off += CH) {
      const uint32_t n = (uint32_t)min(CH, hi - off) & ~15u;
      if (n) asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p.pf + off), "r"(n) : "memory");
    }
  }
  pdl_wait();
  pdl_launch_dependents();

  if (warp == PRODUCER_WARP) {
    // ===================================================================== TMA producer
    if (lane == 0) {
      stamp(2);
      const int box_w = 1 << p.epi_lgw;
      // staging box j of the tile at t (output column c0 + j w); conv tiles are TW x TH x TB pixel boxes
      auto epi_box = [&](const TileCoord& t, int c0, int j, auto&& op) {
        if (p.conv) op(epi + (j << (p.epi_lgw + 8)), c0 + j * box_w, t.cw0, t.ch0, t.cb0);
        else op(epi + (j << (p.epi_lgw + 8)), c0 + j * box_w, t.m0, 0, 0);
      };
      // head-split output of the tile at t: one store per 8-column group (which lies inside one head) from the copy-out
      // staging layout.  Q/K: an (8 columns, 128 tokens) box, or (8, 64 tokens, 1 head, 2 batches) at 64 tokens per
      // batch; V^T: two (64 tokens, 8 columns) boxes.  The maps' extents are head_dim and tokens_per_batch, so that the
      // pad columns, pad rows and pad tokens of the destination are never written.
      auto heads_store = [&](const TileCoord& t) {
        const int T = (int)p.tokens_per_batch;
        const int seg_len = p.heads * p.head_dim;
        int seg = t.n0 / seg_len;
        int head = (t.n0 - seg * seg_len) / p.head_dim;
        int j = t.n0 - seg * seg_len - head * p.head_dim;
        const int b0 = t.m0 / T, tok0 = t.m0 - b0 * T;
        const int b1 = (t.m0 + 64) / T, tok1 = t.m0 + 64 - b1 * T;
        for (int k = 0; k < BN / 8; ++k) {
          const CUtensorMap* tm = seg == 0 ? &tmO : seg == 1 ? &tmR : &tmS;
          const uint8_t* s = epi + (k << 11);
          if (p.seg_kind[seg] == MOS_SEG_ROWS) {
            tma_store_4d(tm, s, j, tok0, head, b0);
          } else {
            tma_store_4d(tm, s, tok0, j, head, b0);
            tma_store_4d(tm, s + 1024, tok1, j, head, b1);
          }
          if ((j += 8) == p.head_dim) {
            j = 0;
            if (++head == p.heads) {
              head = 0;
              ++seg;
            }
          }
        }
      };
      // write out item i (tile t) once the consumers have staged it; returns when the staging tile may be reused
      auto epi_store = [&](const TileCoord& t, int i) {
        mbar_wait_hint(&epi_full, i & 1);
        if (i == 0) stamp(9);
        if (p.epi_heads) {
          heads_store(t);
        } else {
          const int c0 = p.geglu ? t.n0 / 2 : t.n0;
          for (int j = 0; j < EPI_BOXES; ++j)
            epi_box(t, c0, j, [&](const uint8_t* s, int x, int y, int z, int w) {
              if (p.conv) tma_store_4d(&tmO, s, x, y, z, w);
              else tma_store_2d(&tmO, s, x, y);
            });
        }
        bulk_commit();
        if (i == 0) stamp(10);
        bulk_wait_read_all();
        if (i == 0) stamp(5);
        if (i == 1) stamp(15);
      };
      int stage = 0;
      uint32_t phase = 0;
      int it = 0;
      TileCoord prev{};
      for (int ws = blockIdx.x; ws < p.total_items; ws += gridDim.x, ++it) {
        const TileCoord t = item_coord(p, ws);
        const int kb_begin = t.split * p.kb_per_split;
        const int kb_end = min(p.kb_total, kb_begin + p.kb_per_split);
        for (int kb = kb_begin; kb < kb_end; ++kb) {
          uint8_t* sa = smem + stage * stage_bytes;
          uint8_t* sb = sa + A_STAGE_BYTES;
          mbar_wait_hint(&empty_bar[stage], phase ^ 1);     // the wgmmas that read this slot have retired
          mbar_expect_tx(&full_bar[stage], (uint32_t)stage_bytes);
          if (p.conv) {
            const int tap = kb / p.kc_per_tap;
            const int kc = kb - tap * p.kc_per_tap;
            const int kh = tap / 3, kw = tap - kh * 3;
            tma_load_4d(sa, &tmA, &full_bar[stage], kc * BK, t.cw0 + kw - 1, t.ch0 + kh - 1, t.cb0);
          } else {
            tma_load_2d(sa, &tmA, &full_bar[stage], kb * BK, t.m0);
          }
          tma_load_2d(sb, &tmB, &full_bar[stage], kb * BK, t.n0);
          if (LORA) tma_load_2d(sb + B_STAGE_BYTES, &tmL, &full_bar[stage], kb * BK, 0);
          if (++stage == p.stages) {
            stage = 0;
            phase ^= 1;
          }
        }
        if (p.epi_tma) {
          // the previous item's output leaves the staging tile, then this item's residual lands in it.  The producer is
          // here once it has issued this item's last k block: in a CTA with one item that is early in the consumers'
          // mainloop; with several items, the previous item's write-out waits until here, and with it this residual.
          if (it > 0) epi_store(prev, it - 1);
          if (p.res_tma) {
            mbar_expect_tx(&epi_ready, (uint32_t)EPI_BYTES);   // out-of-bounds box elements count too (zero fill)
            for (int j = 0; j < EPI_BOXES; ++j)
              epi_box(t, t.n0, j, [&](uint8_t* s, int x, int y, int z, int w) {
                if (p.conv) tma_load_4d(s, &tmR, &epi_ready, x, y, z, w);
                else tma_load_2d(s, &tmR, &epi_ready, x, y);
              });
          } else {
            mbar_arrive(&epi_ready);
          }
          prev = t;
        }
      }
      if (p.epi_tma && it > 0) {
        epi_store(prev, it - 1);
        bulk_wait_all();                                   // the global writes complete before the CTA exits
      }
    }
  } else {
    // ===================================================================== consumers (warps 0..7)
    const int wg = warp >> 2;                              // warpgroup: tile rows [64 wg, 64 wg + 64)
    const int rA = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // the two tile rows this thread holds: rA, rA + 8
    const int cq = 2 * (lane & 3);                         // column offset inside every 8-column group
    const int et = threadIdx.x;                            // 0..255
    int stage = 0;
    uint32_t phase = 0;
    int it = 0;
    for (int ws = blockIdx.x; ws < p.total_items; ws += gridDim.x, ++it) {
      const TileCoord t = item_coord(p, ws);
      const int kb_begin = t.split * p.kb_per_split;
      const int kb_end = min(p.kb_total, kb_begin + p.kb_per_split);
      float acc[BN / 2];
      float lacc[LORA_N / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
#pragma unroll
      for (int i = 0; i < LORA_N / 2; ++i) lacc[i] = 0.f;
      // One k block stays in flight: k block kb is issued before the wgmmas of kb - 1 are waited for, and only then is
      // kb - 1's slot handed back to the producer.  The wgmma sequence on the accumulator is the same as with a full
      // drain per k block, so the result is bit-identical; only the issue overlaps.
      int prev = -1;                                       // stage of the k block still in flight
      for (int kb = kb_begin; kb < kb_end; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        if (it == 0 && kb == kb_begin && et == 0) stamp(3);
        uint8_t* sa = smem + stage * stage_bytes + wg * (64 * 128);   // this warpgroup's 64 A rows
        const uint64_t adesc = make_desc_sw128(smem_u32(sa));
        const uint64_t bdesc = make_desc_sw128(smem_u32(smem + stage * stage_bytes + A_STAGE_BYTES));
        const uint64_t ldesc = make_desc_sw128(smem_u32(smem + stage * stage_bytes + A_STAGE_BYTES + B_STAGE_BYTES));
        wgmma_fence_regs(acc);
        if constexpr (LORA) wgmma_fence_regs(lacc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) {
          wgmma_ss<BN, F16>(acc, adesc + 2 * k, bdesc + 2 * k, 1u);
          if constexpr (LORA) wgmma_ss<LORA_N, F16>(lacc, adesc + 2 * k, ldesc + 2 * k, 1u);
        }
        wgmma_commit();
        wgmma_wait<1>();                                   // k block kb - 1 has retired
        wgmma_fence_regs(acc);
        if constexpr (LORA) wgmma_fence_regs(lacc);
        if (prev >= 0) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty_bar[prev]);   // this warp's reads of kb - 1's slot are done
        }
        prev = stage;
        if (++stage == p.stages) {
          stage = 0;
          phase ^= 1;
        }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      if constexpr (LORA) wgmma_fence_regs(lacc);
      if (prev >= 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[prev]);
      }
      if (et == 0 && it < 2) stamp(it == 0 ? 4 : 11);
      int b_lo;                                            // batch of the tile's first row (s_bias slot 0)
      {
        long long m0;
        row_coord(p, t, 0, m0, b_lo);
      }
      if (p.splits == 1) {                                 // (split-K partial tiles take no epilogue operands)
        epi_bar();                // every consumer is done with the previous tile's operands and its copy-out reads
        for (int i = et; i < EPI_BATCHES * BN; i += CONSUMER_THREADS) {
          const int j = i / BN, c = i - j * BN;
          s_bias[j][c] = b_lo + j < p.nbatch ? col_bias(p, b_lo + j, t.n0 + c) : 0.f;
        }
        if constexpr (LORA)
          if (et < BN) s_lup[et] = __ldg(reinterpret_cast<const float4*>(p.lora_up) + t.n0 + et);
        epi_bar();
      }
      if (et == 0 && it < 2) stamp(it == 0 ? 6 : 12);
      // ---- epilogue from the accumulator fragment.  16-bit output (rows, GEGLU, head-split) goes to the staging tile;
      // only fp32 output and split-K partials go to global.  Each output path is its own straight-line code (the
      // launch's path is a kernel parameter; head-split tiles with V^T columns take their own), so that a tile runs
      // only the instructions of its path.
      const uint32_t trmask = transposed_groups(p, t.n0);
      if (p.epi_tma) mbar_wait(&epi_ready, it & 1);
      if (et == 0 && it < 2) stamp(it == 0 ? 7 : 13);
      const EpiArgs ea{epi, &s_bias[0][0], s_lup, rA, cq, lane, b_lo};
      epilogue<F16, LORA>(p, t, ea, acc, lacc, trmask, trmask != 0u ? (int)EPI_HEADS_T : p.epi_mode);
      if (et == 0 && it < 2) stamp(it == 0 ? 8 : 14);
      if (p.epi_tma) {
        fence_proxy_async_smem();                          // this thread's staging writes -> the TMA store's reads
        mbar_arrive(&epi_full);
      } else {
        if (p.epi_copy) {
          // ---- copy-out: 16-byte chunks of the staging tile (8 columns of a row, or 8 rows of a V^T column) to their
          // destination, one 16-byte store where the 8 elements are contiguous and aligned there.  The rest (V^T
          // tokens across a batch boundary at a token count that is not a multiple of 8, unaligned row output) is
          // written element by element from the same chunk.
          epi_bar();
          const int groups = (p.geglu ? BN / 2 : BN) / 8;
          for (int idx = et; idx < groups * BM; idx += CONSUMER_THREADS) {
            const int k = idx / BM, rs = idx % BM;
            const bool tr = (trmask >> k) & 1u;
            const int r0 = tr ? (rs & ~7) : rs;           // V^T: 8 rows of column 8k + rs % 8
            const int c0 = tr ? 8 * k + (rs & 7) : 8 * k;
            const uint8_t* src = epi + cp_off(r0, c0, tr);
            long long m0, m7;
            int bq;
            uint16_t* d0 = nullptr;
            bool vec = row_coord(p, t, r0, m0, bq);
            if (vec) {
              d0 = out_elem(p, t, m0, c0);
              vec = (reinterpret_cast<uintptr_t>(d0) & 15) == 0;
              if (tr) vec = vec && row_coord(p, t, r0 + 7, m7, bq) && out_elem(p, t, m7, c0) == d0 + 7;
            }
            if (vec) {
              *reinterpret_cast<uint4*>(d0) = *reinterpret_cast<const uint4*>(src);
            } else {
#pragma unroll 1
              for (int e = 0; e < 8; ++e) {
                long long me;
                if (row_coord(p, t, tr ? r0 + e : r0, me, bq))
                  *out_elem(p, t, me, tr ? c0 : c0 + e) = *reinterpret_cast<const uint16_t*>(src + 2 * e);
              }
            }
          }
        }
        if (et == 0 && it < 2) stamp(it == 0 ? 5 : 15);
      }
      if (!LORA && p.counters != nullptr) {
        // split-K, in-kernel finalize: publish this item's partial tile (bar.sync ordered every consumer thread's stores
        // before this thread; its gpu-scope fence is cumulative over them - the pattern of a cooperative grid sync)
        epi_bar();
        if (et == 0) {
          __threadfence();
          atomicAdd(p.counters + ws / p.splits, 1);
        }
      }
    }
    if (!LORA && p.counters != nullptr) {
      // ---- phase 2 (split-K only): the `splits` CTAs that hold the partials of one output tile each reduce 1/splits of
      // its rows, in the fixed order split 0..S-1 (bitwise reproducible), and apply bias / per-batch bias / residual.
      // Deadlock-free: the grid has at most one CTA per SM (all resident), and no CTA waits before ALL its own partials are
      // published.  The counter runs 0 -> S (arrivals) -> 2S (slices done) and is reset by the last slice.
      const int nthr = CONSUMER_THREADS;
      const int S = p.splits;
      const int rows_per = (BM + S - 1) / S;
      for (int ws = blockIdx.x; ws < p.total_items; ws += gridDim.x) {
        const TileCoord t = item_coord(p, ws);
        int* ctr = p.counters + ws / S;
        if (et == 0) {
          int seen;
          do {
            asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(seen) : "l"(ctr) : "memory");
          } while (seen < S);
        }
        epi_bar();
        const int rlo = t.split * rows_per, rhi = min(BM, rlo + rows_per);
        const int total = (rhi - rlo) * (BN / 4);
        const long long MN = (long long)p.M * p.N;
        // two output quads per thread and four splits per round: 8 independent 16-byte L2 loads in flight per thread (the
        // partials were written by other SMs: the reduction is L2-latency bound, not bandwidth bound)
        for (int i0 = et; i0 < total; i0 += 2 * nthr) {
          bool ok[2];
          long long m[2];
          int b[2], n[2];
          const float* src[2];
          float4 acc4[2];
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int i = i0 + e * nthr;
            const int rr = rlo + i / (BN / 4), c4 = i % (BN / 4);
            m[e] = 0;
            b[e] = 0;
            ok[e] = (i < total) && row_coord(p, t, rr, m[e], b[e]);
            n[e] = t.n0 + c4 * 4;
            src[e] = p.partial + m[e] * p.N + n[e];
            acc4[e] = make_float4(0.f, 0.f, 0.f, 0.f);
          }
          for (int sp = 0; sp < S; sp += 4) {
            float4 v[2][4];
#pragma unroll
            for (int u = 0; u < 4; ++u)
#pragma unroll
              for (int e = 0; e < 2; ++e)
                if (ok[e] && sp + u < S) v[e][u] = __ldcg(reinterpret_cast<const float4*>(src[e] + (sp + u) * MN));
#pragma unroll
            for (int u = 0; u < 4; ++u)
#pragma unroll
              for (int e = 0; e < 2; ++e)
                if (ok[e] && sp + u < S) {     // split order 0..S-1: the summation order of mos_splitk_finalize
                  acc4[e].x += v[e][u].x; acc4[e].y += v[e][u].y; acc4[e].z += v[e][u].z; acc4[e].w += v[e][u].w;
                }
          }
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            if (!ok[e]) continue;
            float4 a4 = acc4[e];
            if (p.bias) {
              const float4 bv = __ldg(reinterpret_cast<const float4*>(p.bias + n[e]));
              a4.x += bv.x; a4.y += bv.y; a4.z += bv.z; a4.w += bv.w;
            }
            if (p.bias_batch) {
              const float4 bv = __ldg(reinterpret_cast<const float4*>(p.bias_batch + (long long)b[e] * p.bias_batch_ld + n[e]));
              a4.x += bv.x; a4.y += bv.y; a4.z += bv.z; a4.w += bv.w;
            }
            if (p.residual) {
              const uint2 rv = *reinterpret_cast<const uint2*>(p.residual + m[e] * p.ldr + n[e]);
              const float2 r0 = unpack16x2<F16>(rv.x), r1 = unpack16x2<F16>(rv.y);
              a4.x += r0.x; a4.y += r0.y; a4.z += r1.x; a4.w += r1.y;
            }
            uint2 o;
            o.x = pack16x2<F16>(a4.x, a4.y);
            o.y = pack16x2<F16>(a4.z, a4.w);
            *reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(p.out) + m[e] * p.ldc + n[e]) = o;
          }
        }
        epi_bar();
        if (et == 0) {
          const int old = atomicAdd(ctr, 1);
          if (old == 2 * S - 1) atomicExch(ctr, 0);     // every slice of this tile is written: ready for the next launch
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------- split-K finalize
template <bool F16>
__global__ void splitk_finalize_kernel(const float* __restrict__ partial, int splits, long long M, long long N,
                                       const float* __restrict__ bias, const float* __restrict__ bias_batch,
                                       long long rows_per_batch, long long bias_batch_ld,
                                       const __nv_bfloat16* __restrict__ residual, long long ldr,
                                       __nv_bfloat16* __restrict__ out, long long ldc) {
  pdl_wait();
  pdl_launch_dependents();
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;  // one thread per 4 columns
  long long n4 = N / 4;
  if (idx >= M * n4) return;
  long long m = idx / n4;
  long long n = (idx - m * n4) * 4;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int s = 0; s < splits; ++s) {
    float4 v = __ldg(reinterpret_cast<const float4*>(partial + ((long long)s * M + m) * N + n));
    acc.x += v.x;
    acc.y += v.y;
    acc.z += v.z;
    acc.w += v.w;
  }
  if (bias) {
    float4 b = __ldg(reinterpret_cast<const float4*>(bias + n));
    acc.x += b.x; acc.y += b.y; acc.z += b.z; acc.w += b.w;
  }
  if (bias_batch) {
    float4 b = __ldg(reinterpret_cast<const float4*>(bias_batch + (m / rows_per_batch) * bias_batch_ld + n));
    acc.x += b.x; acc.y += b.y; acc.z += b.z; acc.w += b.w;
  }
  if (residual) {
    uint2 r = __ldg(reinterpret_cast<const uint2*>(residual + m * ldr + n));
    float2 a = unpack16x2<F16>(r.x), b = unpack16x2<F16>(r.y);
    acc.x += a.x; acc.y += a.y; acc.z += b.x; acc.w += b.y;
  }
  uint2 o;
  o.x = pack16x2<F16>(acc.x, acc.y);
  o.y = pack16x2<F16>(acc.z, acc.w);
  *reinterpret_cast<uint2*>(out + m * ldc + n) = o;
}

static unsigned long long* g_timeline_host = nullptr;
static bool is_aligned(const void* p, size_t a) { return (reinterpret_cast<uintptr_t>(p) % a) == 0; }
static int ilog2(int v) {
  int l = 0;
  while ((1 << l) < v) ++l;
  return l;
}

}  // namespace mos

using namespace mos;

extern "C" int mos_gemm_bf16(const mos_gemm_args* a, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  MOS_CHECK_ARG(a != nullptr, "mos_gemm_bf16: args is NULL");
  MOS_CHECK_ARG(a->A && a->W, "mos_gemm_bf16: A/W is NULL");
  MOS_CHECK_ARG(a->M > 0 && a->N > 0 && a->K > 0, "mos_gemm_bf16: bad shape M=%lld N=%lld K=%lld",
                (long long)a->M, (long long)a->N, (long long)a->K);
  MOS_CHECK_ARG(a->N % BN == 0, "mos_gemm_bf16: N=%lld must be a multiple of %d", (long long)a->N, BN);
  MOS_CHECK_ARG(a->K % BK == 0, "mos_gemm_bf16: K=%lld must be a multiple of %d", (long long)a->K, BK);
  MOS_CHECK_ARG(is_aligned(a->A, 16) && is_aligned(a->W, 16), "mos_gemm_bf16: A/W must be 16-byte aligned");
  MOS_CHECK_DTYPE(a->a_dtype, "mos_gemm_bf16 (a_dtype)");
  MOS_CHECK_DTYPE(a->w_dtype, "mos_gemm_bf16 (w_dtype)");
  MOS_CHECK_ARG(a->a_dtype == a->w_dtype,
                "mos_gemm_bf16: A and W must share the 16-bit type (wgmma takes one operand type for A and B)");
  const bool f16 = a->a_dtype == MOS_DT_F16;
  const int splits = a->splits > 0 ? a->splits : 1;
  const bool lora = a->lora_down != nullptr;
  if (splits > 1) {
    MOS_CHECK_ARG(a->partial != nullptr, "mos_gemm_bf16: split-K needs a partial workspace");
    if (a->tile_counters != nullptr)
      MOS_CHECK_ARG(a->out != nullptr && a->ldc >= a->N && a->ldc % 4 == 0 && a->N % 4 == 0,
                    "mos_gemm_bf16: in-kernel split-K finalize needs `out` (16-bit rows, ldc %% 4 == 0)");
    MOS_CHECK_ARG(!lora && !a->geglu && a->out_mode == MOS_OUT_BF16,
                  "mos_gemm_bf16: split-K cannot be combined with lora / geglu / head-split output");
  } else {
    MOS_CHECK_ARG(a->out_mode == MOS_OUT_HEADS || a->out != nullptr, "mos_gemm_bf16: out is NULL");
  }
  if (lora) {
    MOS_CHECK_ARG(a->lora_up != nullptr && a->lora_seg > 0 && a->lora_seg % 16 == 0 && !a->conv,
                  "mos_gemm_bf16: bad LoRA arguments");
    MOS_CHECK_ARG(a->N / a->lora_seg <= 4, "mos_gemm_bf16: at most 4 LoRA segments");
  }
  if (a->out_mode == MOS_OUT_HEADS) {
    MOS_CHECK_ARG(a->heads > 0 && a->head_dim % 8 == 0 && a->N % (a->heads * a->head_dim) == 0 &&
                      a->N / (a->heads * a->head_dim) <= 3 && a->tokens_per_batch > 0,
                  "mos_gemm_bf16: bad head-split arguments");
  }
  if (a->geglu) MOS_CHECK_ARG(a->out_mode == MOS_OUT_BF16, "mos_gemm_bf16: geglu needs bf16 row-major output");

  GemmDev p;
  memset(&p, 0, sizeof(p));
  CUtensorMap tmA, tmB, tmL, tmO, tmR, tmS;
  memset(&tmL, 0, sizeof(tmL));
  memset(&tmO, 0, sizeof(tmO));
  memset(&tmR, 0, sizeof(tmR));
  memset(&tmS, 0, sizeof(tmS));
  p.M = (int)a->M;
  p.N = (int)a->N;
  p.conv = a->conv;
  p.n_tiles = (int)(a->N / BN);
  int m_tiles;
  if (a->conv) {
    MOS_CHECK_ARG(a->B > 0 && a->H > 0 && a->Wd > 0 && a->C == a->K, "mos_gemm_bf16: bad conv geometry");
    MOS_CHECK_ARG((int64_t)a->B * a->H * a->Wd == a->M, "mos_gemm_bf16: conv M != B*H*W");
    int TW = 1;
    while (TW * 2 <= 128 && a->Wd % (TW * 2) == 0) TW *= 2;
    // choose TH (power of two) maximising the fraction of valid rows in the 128-row tile
    int best_th = 1;
    double best_eff = -1;
    for (int TH = 1; TH * TW <= 128; TH *= 2) {
      int TB = 128 / (TW * TH);
      if (TB > 4 && TH * 2 * TW <= 128) continue;   // the epilogue stages per-batch bias for <= 4 batches per tile
      double eff = ((double)a->H / (ceil_div(a->H, TH) * TH)) * ((double)a->B / (ceil_div(a->B, TB) * TB));
      if (eff > best_eff + 1e-9) {
        best_eff = eff;
        best_th = TH;
      }
    }
    p.TW = TW;
    p.TH = best_th;
    p.TB = 128 / (TW * best_th);
    p.lgTW = ilog2(p.TW);
    p.lgTH = ilog2(p.TH);
    p.H = a->H;
    p.W = a->Wd;
    p.B = a->B;
    p.tiles_w = a->Wd / TW;
    p.tiles_h = (int)ceil_div(a->H, p.TH);
    int tiles_b = (int)ceil_div(a->B, p.TB);
    m_tiles = p.tiles_w * p.tiles_h * tiles_b;
    p.kc_per_tap = (int)(a->K / BK);
    p.kb_total = 9 * p.kc_per_tap;
  } else {
    MOS_CHECK_ARG(a->lda >= a->K && a->lda % 8 == 0, "mos_gemm_bf16: lda=%lld invalid", (long long)a->lda);
    m_tiles = (int)ceil_div(a->M, BM);
    p.kb_total = (int)(a->K / BK);
  }
  p.m_tiles = m_tiles;
  // ---- tensor maps: A tile [128 rows, 64], W tile [160 rows, 64], LoRA down [16, 64]
  if (a->conv) {
    uint64_t dims[4] = {(uint64_t)a->C, (uint64_t)a->Wd, (uint64_t)a->H, (uint64_t)a->B};
    const uint64_t pitch = (uint64_t)(a->lda > 0 ? a->lda : a->C);
    MOS_CHECK_ARG(pitch >= (uint64_t)a->C && pitch % 8 == 0, "mos_gemm_bf16: conv pixel pitch %llu invalid",
                  (unsigned long long)pitch);
    uint64_t str[3] = {pitch * 2, (uint64_t)a->Wd * pitch * 2, (uint64_t)a->H * a->Wd * pitch * 2};
    uint32_t box[4] = {BK, (uint32_t)p.TW, (uint32_t)p.TH, (uint32_t)p.TB};
    int rc = encode_tmap(&tmA, a->A, 2, 4, dims, str, box, 3);
    if (rc) return rc;
    uint64_t wd[2] = {(uint64_t)a->K * 9, (uint64_t)a->N};
    uint64_t ws[1] = {(uint64_t)a->K * 9 * 2};
    uint32_t wb[2] = {BK, BN};
    rc = encode_tmap(&tmB, a->W, 2, 2, wd, ws, wb, 3);
    if (rc) return rc;
  } else {
    uint64_t dims[2] = {(uint64_t)a->K, (uint64_t)a->M};
    uint64_t str[1] = {(uint64_t)a->lda * 2};
    uint32_t box[2] = {BK, (uint32_t)BM};
    int rc = encode_tmap(&tmA, a->A, 2, 2, dims, str, box, 3);
    if (rc) return rc;
    uint64_t wd[2] = {(uint64_t)a->K, (uint64_t)a->N};
    uint64_t ws[1] = {(uint64_t)a->K * 2};
    uint32_t wb[2] = {BK, BN};
    rc = encode_tmap(&tmB, a->W, 2, 2, wd, ws, wb, 3);
    if (rc) return rc;
    if (lora) {
      uint64_t ld[2] = {(uint64_t)a->K, LORA_N};
      uint64_t ls[1] = {(uint64_t)a->K * 2};
      uint32_t lb[2] = {BK, LORA_N};
      rc = encode_tmap(&tmL, a->lora_down, 2, 2, ld, ls, lb, 3);
      if (rc) return rc;
    }
  }
  MOS_CHECK_ARG(splits <= p.kb_total, "mos_gemm_bf16: splits=%d > k blocks=%d", splits, p.kb_total);
  p.splits = splits;
  p.kb_per_split = (int)ceil_div(p.kb_total, splits);
  MOS_CHECK_ARG((long long)p.kb_per_split * (splits - 1) < p.kb_total, "mos_gemm_bf16: empty split");
  p.geglu = a->geglu;
  p.out_mode = a->out_mode;
  p.partial = a->partial;
  p.bias = a->bias;
  p.bias_batch = a->bias_batch;
  p.rows_per_batch = a->rows_per_batch > 0 ? a->rows_per_batch : 1;
  p.bias_batch_ld = a->bias_batch_ld > 0 ? a->bias_batch_ld : a->N;
  p.residual = reinterpret_cast<const __nv_bfloat16*>(a->residual);
  p.ldr = a->ldr;
  p.lora_up = a->lora_up;
  p.lora_seg = a->lora_seg > 0 ? a->lora_seg : a->N;
  p.out = a->out;
  p.ldc = a->ldc;
  for (int i = 0; i < 3; ++i) {
    p.seg_ptr[i] = a->seg_ptr[i];
    p.seg_kind[i] = a->seg_kind[i];
    p.seg_rows_pad[i] = a->seg_rows_pad[i];
  }
  p.heads = a->heads;
  p.head_dim = a->head_dim;
  p.dpad = a->dpad;
  p.dv_pad = a->dv_pad;
  p.tokens_per_batch = a->tokens_per_batch > 0 ? a->tokens_per_batch : 1;
  p.accum = a->accumulate;
  // Every 16-bit output goes through the staging tile.  Row output (with GEGLU and residual) that TMA can address (16-byte
  // aligned base, row pitch a multiple of 8 elements) is written by TMA stores, its residual prefetched by TMA when that
  // is addressable too: tensor maps with the tile's row geometry (plain [M, cols], conv [B, H, W, cols]), one box per
  // staging box.  Head-split output is written by TMA stores as well when every 64-row half of a tile lies inside one
  // batch and a 128-row tile inside one batch or two whole ones (tokens_per_batch 64 or a multiple of 128), and every
  // segment is addressable: one tensor map per segment, Q/K [batch, head, token, j] and V^T [batch, head, j, token] with
  // the extents head_dim and tokens_per_batch.  Other head-split output (the 77-token text K/V) and other row output are
  // copied out of the staging tile by the consumers.  MOS_GEMM_HEADS_COPY=1 sends all head-split output that way.
  static int heads_copy_env = -1;
  if (heads_copy_env < 0) {
    const char* hc = getenv("MOS_GEMM_HEADS_COPY");
    heads_copy_env = (hc && atoi(hc) != 0) ? 1 : 0;
  }
  const uint64_t cols = (uint64_t)(a->geglu ? a->N / 2 : a->N);
  auto tma_rows = [&](const void* base, long long ld) {
    return base != nullptr && ld >= (long long)cols && ld % 8 == 0 && is_aligned(base, 16);
  };
  const long long T = p.tokens_per_batch;
  const int nseg = a->out_mode == MOS_OUT_HEADS ? (int)(a->N / ((long long)a->heads * a->head_dim)) : 0;
  bool heads_tma = a->out_mode == MOS_OUT_HEADS && !heads_copy_env && (T == 64 || T % 128 == 0) && a->M % T == 0;
  for (int s = 0; s < nseg && heads_tma; ++s) {
    const bool tr = a->seg_kind[s] == MOS_SEG_TRANSPOSED;
    heads_tma = a->seg_ptr[s] != nullptr && is_aligned(a->seg_ptr[s], 16) && a->seg_rows_pad[s] >= T &&
                (tr ? a->dv_pad >= a->head_dim && a->seg_rows_pad[s] % 8 == 0
                    : a->dpad >= a->head_dim && a->dpad % 8 == 0);
  }
  if (a->geglu || a->out_mode == MOS_OUT_HEADS) p.residual = nullptr;   // neither takes a residual
  p.epi_heads = heads_tma ? 1 : 0;
  p.nseg = nseg;
  p.epi_tma = ((a->out_mode == MOS_OUT_BF16 && splits == 1 && tma_rows(a->out, a->ldc)) || heads_tma) ? 1 : 0;
  p.res_tma = (p.epi_tma && p.residual != nullptr && tma_rows(a->residual, a->ldr)) ? 1 : 0;
  p.epi_copy = (a->out_mode != MOS_OUT_F32 && splits == 1 && !p.epi_tma) ? 1 : 0;
  p.epi_mode = splits > 1                    ? EPI_PARTIAL
               : a->out_mode == MOS_OUT_F32  ? EPI_F32
               : a->geglu                    ? EPI_GEGLU
               : p.residual == nullptr       ? EPI_ROWS
               : p.res_tma                   ? EPI_ROWS_RES_SMEM
                                             : EPI_ROWS_RES_GLOBAL;
  if (heads_tma) {
    CUtensorMap* maps[3] = {&tmO, &tmR, &tmS};
    const uint64_t B = (uint64_t)(a->M / T), H = (uint64_t)a->heads, d = (uint64_t)a->head_dim;
    for (int s = 0; s < nseg; ++s) {
      const uint64_t rows = (uint64_t)a->seg_rows_pad[s];
      int rc;
      if (a->seg_kind[s] == MOS_SEG_TRANSPOSED) {
        const uint64_t pitch = rows * 2;
        uint64_t dims[4] = {(uint64_t)T, d, H, B};
        uint64_t str[3] = {pitch, (uint64_t)a->dv_pad * pitch, H * a->dv_pad * pitch};
        uint32_t box[4] = {64, 8, 1, 1};
        rc = encode_tmap(maps[s], a->seg_ptr[s], 2, 4, dims, str, box, 3);
      } else {
        const uint64_t pitch = (uint64_t)a->dpad * 2;
        const uint32_t bt = T == 64 ? 64 : 128;
        uint64_t dims[4] = {d, (uint64_t)T, H, B};
        uint64_t str[3] = {pitch, rows * pitch, H * rows * pitch};
        uint32_t box[4] = {8, bt, 1, BM / bt};
        rc = encode_tmap(maps[s], a->seg_ptr[s], 2, 4, dims, str, box, 0);
      }
      if (rc) return rc;
    }
  }
  if (p.epi_tma && !p.epi_heads) {
    p.epi_lgw = a->geglu ? EPI_LGW_GEGLU : EPI_LGW_ROWS;
    const uint32_t bw = 1u << p.epi_lgw;
    const int swz = a->geglu ? 1 : 2;        // SWIZZLE_32B / SWIZZLE_64B: rows of 2 bw bytes (epilogue)
    auto row_map = [&](CUtensorMap* tm, const void* base, long long ld) -> int {
      const uint64_t pitch = (uint64_t)ld * 2;
      if (a->conv) {
        uint64_t dims[4] = {cols, (uint64_t)a->Wd, (uint64_t)a->H, (uint64_t)a->B};
        uint64_t str[3] = {pitch, (uint64_t)a->Wd * pitch, (uint64_t)a->H * a->Wd * pitch};
        uint32_t box[4] = {bw, (uint32_t)p.TW, (uint32_t)p.TH, (uint32_t)p.TB};
        return encode_tmap(tm, base, 2, 4, dims, str, box, swz);
      }
      uint64_t dims[2] = {cols, (uint64_t)a->M};
      uint64_t str[1] = {pitch};
      uint32_t box[2] = {bw, (uint32_t)BM};
      return encode_tmap(tm, base, 2, 2, dims, str, box, swz);
    };
    int rc = row_map(&tmO, a->out, a->ldc);
    if (rc) return rc;
    if (p.res_tma) {
      rc = row_map(&tmR, a->residual, a->ldr);
      if (rc) return rc;
    }
  }
  p.tl = g_timeline_host;
  p.pf = nullptr;
  p.pf_bytes = 0;
  if (a->prefetch_ptr != nullptr && a->prefetch_bytes >= 16) {
    MOS_CHECK_ARG(is_aligned(a->prefetch_ptr, 16), "mos_gemm_bf16: prefetch_ptr must be 16-byte aligned");
    p.pf = reinterpret_cast<const uint8_t*>(a->prefetch_ptr);
    p.pf_bytes = a->prefetch_bytes;
  }
  p.counters = (splits > 1) ? a->tile_counters : nullptr;
  if (p.counters != nullptr) {
    MOS_CHECK_ARG((long long)p.n_tiles * m_tiles <= a->tile_counters_len,
                  "mos_gemm_bf16: tile_counters holds %d counters, the launch needs %lld", (int)a->tile_counters_len,
                  (long long)p.n_tiles * m_tiles);
  }
  if (a->bias_batch && !a->conv)
    MOS_CHECK_ARG(p.rows_per_batch >= 32, "mos_gemm_bf16: bias_batch needs rows_per_batch >= 32 in plain mode");
  p.total_items = p.n_tiles * m_tiles * splits;
  p.nbatch = a->conv ? a->B : (int)ceil_div(a->M, p.rows_per_batch);

  // MOS_GEMM_STAGES=n: default pipeline depth (otherwise as many stages as fit in shared memory)
  // MOS_GEMM_MAX_CTAS=n (profiling aid): cap the persistent grid at n CTAs, to see whether a k block gets faster when
  // fewer SMs share L2 (tools/gemm_shape_bench.py --max-ctas)
  static int num_sms = 0, stages_env = -1, max_ctas_env = -1;
  if (stages_env < 0) {
    const char* st = getenv("MOS_GEMM_STAGES");
    stages_env = st ? atoi(st) : 0;
    const char* mc = getenv("MOS_GEMM_MAX_CTAS");
    max_ctas_env = mc ? atoi(mc) : 0;
  }
  if (num_sms == 0) {
    int dev = 0;
    MOS_CHECK_CUDA(cudaGetDevice(&dev));
    MOS_CHECK_CUDA(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev));
  }
  const int stage_bytes = A_STAGE_BYTES + (lora ? BN + LORA_N : BN) * 128;
  int stages = a->stages > 0 ? a->stages : (stages_env > 0 ? stages_env : MAX_STAGES);
  if (stages > MAX_STAGES) stages = MAX_STAGES;
  const int epi_bytes = (p.epi_tma || p.epi_copy) ? EPI_BYTES : 0;
  while (stages * stage_bytes + epi_bytes + 1024 > MAX_DYN_SMEM) --stages;
  if (stages < 2) stages = 2;
  p.stages = stages;
  const int smem_bytes = stages * stage_bytes + epi_bytes + 1024;

  static bool configured = false;
  if (!configured) {
    configured = true;
    MOS_CHECK_CUDA(cudaFuncSetAttribute(gemm_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, MAX_DYN_SMEM));
    MOS_CHECK_CUDA(cudaFuncSetAttribute(gemm_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, MAX_DYN_SMEM));
    MOS_CHECK_CUDA(cudaFuncSetAttribute(gemm_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, MAX_DYN_SMEM));
    MOS_CHECK_CUDA(cudaFuncSetAttribute(gemm_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, MAX_DYN_SMEM));
  }
  // persistent: at most one CTA per SM; each CTA loops over its share of the (tile, split) work items
  const int max_ctas = max_ctas_env > 0 && max_ctas_env < num_sms ? max_ctas_env : num_sms;
  const int units = p.total_items < max_ctas ? p.total_items : max_ctas;
  auto kern = f16 ? (lora ? gemm_kernel<true, true> : gemm_kernel<true, false>)
                  : (lora ? gemm_kernel<false, true> : gemm_kernel<false, false>);
  MOS_CHECK_CUDA(launch_pdl(kern, dim3((unsigned)units), dim3(NUM_THREADS), (size_t)smem_bytes, stream, tmA, tmB, tmL, tmO, tmR, tmS, p));
  return MOS_OK;
}

extern "C" int mos_debug_set_timeline(void* buf) {
  mos::g_timeline_host = reinterpret_cast<unsigned long long*>(buf);
  return MOS_OK;
}

extern "C" int mos_splitk_finalize(const float* partial, int32_t splits, int64_t M, int64_t N, const float* bias,
                                   const float* bias_batch, int64_t rows_per_batch, int64_t bias_batch_ld,
                                   const void* residual, int64_t ldr, void* out, int64_t ldc, int32_t act_dtype,
                                   void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  MOS_CHECK_ARG(partial && out && splits >= 1 && M > 0 && N > 0 && N % 4 == 0, "mos_splitk_finalize: bad arguments");
  MOS_CHECK_DTYPE(act_dtype, "mos_splitk_finalize");
  long long total = M * (N / 4);
  int threads = 256;
  long long blocks = ceil_div(total, threads);
  MOS_CHECK_CUDA(launch_pdl(act_dtype == MOS_DT_F16 ? splitk_finalize_kernel<true> : splitk_finalize_kernel<false>,
                            dim3((unsigned)blocks), dim3(threads), 0, stream, partial,
                            (int)splits, (long long)M, (long long)N, bias, bias_batch,
                            (long long)(rows_per_batch > 0 ? rows_per_batch : 1),
                            (long long)(bias_batch_ld > 0 ? bias_batch_ld : N),
                            reinterpret_cast<const __nv_bfloat16*>(residual), (long long)ldr,
                            reinterpret_cast<__nv_bfloat16*>(out), (long long)ldc));
  return MOS_OK;
}
