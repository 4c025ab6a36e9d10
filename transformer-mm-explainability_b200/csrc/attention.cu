// Attention forward that stages A = softmax(QK^T) to HBM, and the attention backward that stages dA = dO V^T
// (the two tensors the reference captures with forward / backward hooks) and continues to dQ, dK, dV.
//
// Numerics: fp32-faithful products from THREE fp16 tensor-core passes (the scheme of gemm_wgmma.cu):
//   x = hi + lo' / 2048,  hi = fp16(x),  lo' = fp16((x - hi) * 2048);   a.b = hi.hi + (lo'.hi + hi.lo') / 2048
// with hi.hi in one fp32 accumulator and the two cross products in a second one that is folded in once.  fp16 x fp16
// products are exact in the fp32 accumulator.  Operand range: |x| <= 65504 and an absolute floor of 3e-11 - activations,
// probabilities and the (power-of-two normalised, see gscale) gradient stream sit well inside.
//
// Structure.  The fp32 operands (Q, K, V, dO) are split ONCE per call into fp16 hi / lo planes by a streaming pre-pass
// (split_planes_kernel; 8 bytes moved per element, ~1 % of the attention time), so that the attention kernels themselves
// contain no conversion work: operand tiles arrive in shared memory with cp.async already in MMA precision, fragments are
// fetched with ldmatrix (one instruction per 16x16 A fragment or per two 16x8 B fragments, transposing on the fly where
// the product needs the other orientation), and the inner loops are 3 mma.sync.m16n8k16 per fragment pair.  The earlier
// version split fp32 tiles at every fragment load: each K / V tile was re-split by every warp that touched it and by
// every query tile of the head (10x at ViT-L/14@336), which made the kernels ALU-bound at long sequences
// (profiles/launches_l14_r2_before.md: attention = 61 % of the ViT-L/14@336 step).
// The softmax keeps each score row in registers across max / exp / normalise (one shared-memory read and one write per
// element), stages A with coalesced 8-byte stores and leaves the probabilities in shared memory as fp16 planes for P.V.
//
// One CTA = one (batch, head, TQ-query tile), TQ/8 warps; the score rows of the tile live in shared memory, so any S up
// to ~700 (TQ = 64) / ~1024 (TQ = 32: DETR at 800x1066 has 850 keys) is handled without a second pass; longer rows (up
// to 16384 keys) run the two-pass kernels below (attention_fwd_long_kernel / attention_bwd_q_long_kernel).  wgmma is
// the wrong tool for CLIP ViT-B/32 (a head is 50x50x64, below one 128-row GEMM tile).  Deterministic (no atomics):
// dK / dV come from a second kernel that walks the query tiles for one key tile.
#include "mmx_common.cuh"
#include <math_constants.h>
#include <cuda_fp16.h>

namespace mmx {

// Ragged self-attention (packed rows): sample b owns rows offs[b] .. offs[b]+lens[b]-1 of Q/K/V/O and attends within
// them; the staged A / dA planes stay dense [B,H,T,ld] with rows and columns >= lens[b] zero-filled.
struct Ragged {
  const int* offs = nullptr;
  const int* lens = nullptr;
};

constexpr int TKEY = 64;  // keys per shared-memory tile
constexpr int KV_THREADS = 256;
constexpr float LO_SCALE = 2048.f, LO_INV = 1.f / 2048.f;
constexpr int MAX_PAIRS = 16;   // score-row elements per lane held in registers: 2 * 32 * 16 = 1024 keys (NP = 2: S <= 128)

// (x0, x1) -> packed fp16 pair hi (x0 in the low half: element k sits below element k+1) and the packed pair of the
// scaled residuals
__device__ __forceinline__ void split_f16(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  const __half2 h = __floats2half2_rn(x0, x1);
  const float2 hf = __half22float2(h);
  const __half2 l = __floats2half2_rn((x0 - hf.x) * LO_SCALE, (x1 - hf.y) * LO_SCALE);
  hi = *reinterpret_cast<const uint32_t*>(&h);
  lo = *reinterpret_cast<const uint32_t*>(&l);
}

// ---------------------------------------------------------------------------------------------------------------------
// pre-pass: fp32 [rows, cols] (row stride ldx) -> fp16 planes hi / lo [rows, ldp]; columns < scale_cols are multiplied by
// `mul` first (the reference scales q before the product, auxilary.py:173).  8 columns per thread.
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) split_planes_kernel(const float* __restrict__ X, int ldx, long long rows, int cols, float mul,
                                                           int scale_cols, __half* __restrict__ hi, __half* __restrict__ lo, int ldp) {
  const int cpr = cols / 8;
  const long long n = rows * cpr;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / cpr;
    const int c = (int)(i - r * cpr) * 8;
    const float4 a = *reinterpret_cast<const float4*>(X + r * ldx + c), b = *reinterpret_cast<const float4*>(X + r * ldx + c + 4);
    const float m = c < scale_cols ? mul : 1.f;
    uint4 h, l;
    split_f16(a.x * m, a.y * m, h.x, l.x);
    split_f16(a.z * m, a.w * m, h.y, l.y);
    split_f16(b.x * m, b.y * m, h.z, l.z);
    split_f16(b.z * m, b.w * m, h.w, l.w);
    *reinterpret_cast<uint4*>(hi + r * ldp + c) = h;
    *reinterpret_cast<uint4*>(lo + r * ldp + c) = l;
  }
}

static int split_planes(const float* X, int ldx, long long rows, int cols, float mul, int scale_cols, __half* hi, __half* lo,
                        int ldp, cudaStream_t st) {
  if (rows == 0 || cols == 0) return 0;
  const long long n = rows * (cols / 8);
  long long g = (n + 255) / 256;
  const long long cap = (long long)sm_count() * 16;
  split_planes_kernel<<<(int)(g > cap ? cap : g), 256, 0, st>>>(X, ldx, rows, cols, mul, scale_cols, hi, lo, ldp);
  MMX_LAUNCH_CHECK();
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------------
// MMA / ldmatrix helpers.  Fragment layout of m16n8k16 (g = lane / 4, t = lane % 4), every register = two consecutive-k
// fp16 values:  A (16x16, row)  a0 (g, 2t..2t+1)  a1 (g+8, 2t..)  a2 (g, 2t+8..)  a3 (g+8, 2t+8..)
//               B (16x8, col)   b0 (k = 2t..2t+1, n = g)  b1 (k = 2t+8.., n = g)
//               C (16x8)        c0 (g, 2t)  c1 (g, 2t+1)  c2 (g+8, 2t)  c3 (g+8, 2t+1)
// Shared-memory planes are [row][k] halves with a row stride of (cols + 8) halves: the eight 16-byte rows of every 8x8
// ldmatrix tile then fall into eight different 16-byte bank groups (stride bytes = 16 mod 32).
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mma_f16(float (&d)[4], const uint32_t (&a)[4], const uint32_t* b) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], const __half* p) {
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t (&r)[4], const __half* p) {
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}
__device__ __forceinline__ void ldsm_x2_t(uint32_t (&r)[2], const __half* p) {
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0,%1}, [%2];" : "=r"(r[0]), "=r"(r[1]) : "r"(a));
}
// per-lane row addresses of the 8x8 tiles (lane l supplies row l & 7 of tile l >> 3)
//   A fragment of a [row][k] plane at (m0, k0):          tiles (m, k), (m+8, k), (m, k+8), (m+8, k+8)
__device__ __forceinline__ const __half* addr_a(const __half* base, int ld, int m0, int k0, int lane) {
  return base + (m0 + (lane & 7) + ((lane >> 3) & 1) * 8) * ld + k0 + ((lane >> 4) & 1) * 8;
}
//   two B fragments (n0, n0+8) of a [n][k] plane at k0:  tiles (n, k), (n, k+8), (n+8, k), (n+8, k+8)
__device__ __forceinline__ const __half* addr_b2(const __half* base, int ld, int n0, int k0, int lane) {
  return base + (n0 + (lane & 7) + ((lane >> 4) & 1) * 8) * ld + k0 + ((lane >> 3) & 1) * 8;
}
//   two B fragments (n0, n0+8) of a [k][n] plane at k0, transposed on load:  tiles (k, n), (k+8, n), (k, n+8), (k+8, n+8)
__device__ __forceinline__ const __half* addr_bt2(const __half* base, int ld, int k0, int n0, int lane) {
  return base + (k0 + (lane & 7) + ((lane >> 3) & 1) * 8) * ld + n0 + ((lane >> 4) & 1) * 8;
}
//   A fragment of a TRANSPOSED operand stored [k][m], transposed on load:  tiles (k, m), (k, m+8), (k+8, m), (k+8, m+8)
__device__ __forceinline__ const __half* addr_at(const __half* base, int ld, int k0, int m0, int lane) {
  return base + (k0 + (lane & 7) + ((lane >> 4) & 1) * 8) * ld + m0 + ((lane >> 3) & 1) * 8;
}
// 3-pass product on one fragment pair
__device__ __forceinline__ void mma3(float (&main)[4], float (&cross)[4], const uint32_t (&ahi)[4], const uint32_t (&alo)[4],
                                     const uint32_t* bhi, const uint32_t* blo) {
  mma_f16(cross, alo, bhi);
  mma_f16(cross, ahi, blo);
  mma_f16(main, ahi, bhi);
}

// A score row holds round_up(S,16) + 4 floats: the row stride is then = 16 (mod 32) bytes, so the eight rows of an ldmatrix
// tile of the P planes fall into eight different 16-byte bank groups.  After the softmax the same bytes hold the fp16 planes
// of the probabilities: hi at halves [0, S16), lo at halves [S16 + 8, 2 S16 + 8) (16-byte aligned, ends with the row).
__host__ __device__ inline int score_ld(int S) { return round_up(S, 16) + 4; }
__host__ __device__ inline int plane_lo_off(int S) { return round_up(S, 16) + 8; }

// profiling aid (mmx_gemm_trace): clock64 at the phase boundaries of block (0,0,0)
__device__ long long* g_attn_trace = nullptr;
#define ATT_TRACE(slot)                                                                                   \
  do {                                                                                                    \
    if (g_attn_trace != nullptr && (blockIdx.x | blockIdx.y | blockIdx.z) == 0 && threadIdx.x == 0)       \
      g_attn_trace[slot] = clock64();                                                                     \
  } while (0)

template <int HD>
struct AttnSmem {
  static constexpr int LDH = HD + 8;   // halves per row of an operand plane
  static constexpr int STAGE = 2 * TKEY * LDH;   // halves per K / V tile stage: hi plane then lo plane
  // score rows (fp32, later the P planes in place) + Q (or dO) planes + NS stages of K / V tile planes
  static size_t bytes(int S, int TQ, int NS = 2) {
    return sizeof(float) * (size_t)TQ * score_ld(S) + sizeof(__half) * (2 * (size_t)TQ * LDH + (size_t)NS * STAGE);
  }
};

// 16-byte asynchronous global -> shared copy (LDGSTS); !valid zero-fills the destination without touching src
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc, bool valid) {
  const uint32_t d = (uint32_t)__cvta_generic_to_shared(smem_dst);
  const int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(gsrc), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// rows r0 .. r0+ROWS-1 (zero beyond `limit`) of an operand -> the hi / lo planes sHi / sLo (row stride LDH halves).
// Two sources: ready-made planes (Ylo != nullptr: cp.async, the caller commits / waits), or - for short sequences, where a
// tile is used by ONE CTA only and a separate split pass would cost more than it saves - the fp32 matrix itself
// (Ylo == nullptr, Yhi is a float pointer, ldp its row stride in floats): the tile is read with 128-bit loads, multiplied by
// `mul` and split on the way into shared memory, once per CTA.
template <int HD, int ROWS>
__device__ __forceinline__ void load_planes_async(const __half* __restrict__ Yhi, const __half* __restrict__ Ylo, int ldp, long long ybase,
                                                  int r0, int limit, __half* sHi, __half* sLo, float mul = 1.f) {
  constexpr int LDH = HD + 8;
  if (Ylo != nullptr) {
    constexpr int CH = HD / 8;
    for (int e = threadIdx.x; e < ROWS * CH; e += blockDim.x) {
      const int r = e / CH, d = (e % CH) * 8;
      const bool ok = r0 + r < limit;
      const long long off = ok ? ybase + (long long)(r0 + r) * ldp + d : 0;
      cp_async16(sHi + r * LDH + d, Yhi + off, ok);
      cp_async16(sLo + r * LDH + d, Ylo + off, ok);
    }
  } else {
    const float* __restrict__ Yf = reinterpret_cast<const float*>(Yhi);
    constexpr int CH = HD / 4;
    for (int e = threadIdx.x; e < ROWS * CH; e += blockDim.x) {
      const int r = e / CH, d = (e % CH) * 4;
      float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
      if (r0 + r < limit) x = *reinterpret_cast<const float4*>(Yf + ybase + (long long)(r0 + r) * ldp + d);
      uint2 h, l;
      split_f16(x.x * mul, x.y * mul, h.x, l.x);
      split_f16(x.z * mul, x.w * mul, h.y, l.y);
      *reinterpret_cast<uint2*>(sHi + r * LDH + d) = h;
      *reinterpret_cast<uint2*>(sLo + r * LDH + d) = l;
    }
  }
}

// K / V tiles stream through a ring of NS shared-memory stages (cp.async, one commit group per tile): while tile t is
// multiplied, tiles t+1 .. t+NS-1 are in flight, so the L2 latency of a tile (~1 us) is overlapped instead of paid once per
// tile.  Protocol: the caller has issued and committed tiles 0 .. NS-2 (tile 0 may share its group with the X tile); every
// iteration issues tile t+NS-1 into the stage consumed in iteration t-1, commits (an empty group when there is no tile
// left), waits until at most NS-1 groups are pending (tile t has landed) and multiplies.
template <int HD>
__device__ __forceinline__ void issue_kv_tile(const __half* __restrict__ Yhi, const __half* __restrict__ Ylo, int ldp, long long ybase,
                                              int tile, int S, __half* sKV, int NS) {
  if (tile * TKEY < S) {
    __half* st = sKV + (size_t)(tile % NS) * AttnSmem<HD>::STAGE;
    load_planes_async<HD, TKEY>(Yhi, Ylo, ldp, ybase, tile * TKEY, S, st, st + TKEY * (HD + 8));
  }
  cp_async_commit();
}

// scores[i][j] (i in the TQ-row tile, j in [0,S)) = post_scale * sum_d X[i][d] * Y[j][d] on pre-split planes.
// Warp w owns row block w % MB and the 32-key half w / MB of each key tile.
template <int HD, int MB, int NS>
__device__ __forceinline__ void tile_scores(const __half* __restrict__ Yhi, const __half* __restrict__ Ylo, int ldp, long long ybase, int S,
                                            const __half* sXh, const __half* sXl, __half* sKV, float* sP, int ldP,
                                            float post_scale, int live_rows) {
  constexpr int LDH = HD + 8;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int m0 = (warp % MB) * 16, kh = (warp / MB) * 32;
  int tile = 0;
  for (int j0 = 0; j0 < S; j0 += TKEY, ++tile) {
    issue_kv_tile<HD>(Yhi, Ylo, ldp, ybase, tile + NS - 1, S, sKV, NS);
    cp_async_wait<NS - 1>();
    __syncthreads();
    const __half* sYh = sKV + (size_t)(tile % NS) * AttnSmem<HD>::STAGE;
    const __half* sYl = sYh + TKEY * LDH;
    float acc[4][4] = {}, crs[4][4] = {};
    // live 8-key blocks of this warp's half (may be <= 0); a row block entirely past the sample's rows does no math
    const int ntiles = m0 < live_rows ? (S - j0 - kh + 7) >> 3 : 0;
    if (ntiles > 0) {
#pragma unroll
      for (int k0 = 0; k0 < HD; k0 += 16) {
        uint32_t ahi[4], alo[4];
        ldsm_x4(ahi, addr_a(sXh, LDH, m0, k0, lane));
        ldsm_x4(alo, addr_a(sXl, LDH, m0, k0, lane));
#pragma unroll
        for (int np = 0; np < 2; ++np) {                      // two pairs of 8-key tiles
          if (2 * np < ntiles) {
            uint32_t bhi[4], blo[4];
            ldsm_x4(bhi, addr_b2(sYh, LDH, kh + np * 16, k0, lane));
            ldsm_x4(blo, addr_b2(sYl, LDH, kh + np * 16, k0, lane));
            mma3(acc[2 * np], crs[2 * np], ahi, alo, bhi, blo);
            mma3(acc[2 * np + 1], crs[2 * np + 1], ahi, alo, bhi + 2, blo + 2);
          }
        }
      }
    }
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
      const int j = j0 + kh + nt * 8 + 2 * t;           // even; ldP is even
      if (j < ldP) {
        float* p0 = sP + (m0 + g) * ldP + j;
        *reinterpret_cast<float2*>(p0) = make_float2(fmaf(crs[nt][0], LO_INV, acc[nt][0]) * post_scale,
                                                     fmaf(crs[nt][1], LO_INV, acc[nt][1]) * post_scale);
        *reinterpret_cast<float2*>(p0 + 8 * ldP) = make_float2(fmaf(crs[nt][2], LO_INV, acc[nt][2]) * post_scale,
                                                               fmaf(crs[nt][3], LO_INV, acc[nt][3]) * post_scale);
      }
    }
    __syncthreads();                                    // the stage is refilled in the next iteration; the scores are visible
  }
}

// out[i][d] = sum_j P[i][j] * Y[j][d] with P as fp16 planes in the score rows (hi at halves [0, S16), lo from `lo_off` of
// each row) and Y tiles [key][d] as planes (transposed on load).  Warp w owns row block w % MB and the d half w / MB; its
// HD/16 accumulator fragments hold rows m0+g, m0+g+8 and columns d0 + 8*nt + 2t, +1.  The caller has issued the first Y
// tile into sY* with cp.async and passed a __syncthreads after the last write of the P planes.
template <int HD, int MB, int NS>
__device__ __forceinline__ void tile_pv(const __half* __restrict__ Yhi, const __half* __restrict__ Ylo, int ldp, long long ybase, int S,
                                        const __half* sP16, int ldP, int lo_off, __half* sKV, float (&out)[HD / 16][4],
                                        int live_rows) {
  constexpr int LDH = HD + 8, NT = HD / 16;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m0 = (warp % MB) * 16, d0 = (warp / MB) * (HD / 2);
  const int ldp16 = 2 * ldP;                              // halves per score row
  float crs[NT][4];
#pragma unroll
  for (int nt = 0; nt < NT; ++nt)
#pragma unroll
    for (int c = 0; c < 4; ++c) out[nt][c] = crs[nt][c] = 0.f;
  int tile = 0;
  for (int j0 = 0; j0 < S; j0 += TKEY, ++tile) {
    issue_kv_tile<HD>(Yhi, Ylo, ldp, ybase, tile + NS - 1, S, sKV, NS);
    cp_async_wait<NS - 1>();
    __syncthreads();
    const __half* sYh = sKV + (size_t)(tile % NS) * AttnSmem<HD>::STAGE;
    const __half* sYl = sYh + TKEY * LDH;
    // keys jn .. round_up(jn, 16) are zero rows of sY and finite (zero) entries of the P planes; dead row blocks skip the math
    const int jn = m0 < live_rows ? min(TKEY, S - j0) : 0;
#pragma unroll 2
    for (int kk = 0; kk < jn; kk += 16) {
      uint32_t ahi[4], alo[4];
      ldsm_x4(ahi, addr_a(sP16, ldp16, m0, j0 + kk, lane));
      ldsm_x4(alo, addr_a(sP16 + lo_off, ldp16, m0, j0 + kk, lane));
      if constexpr (NT >= 2) {
#pragma unroll
        for (int np = 0; np < NT / 2; ++np) {
          uint32_t bhi[4], blo[4];
          ldsm_x4_t(bhi, addr_bt2(sYh, LDH, kk, d0 + np * 16, lane));
          ldsm_x4_t(blo, addr_bt2(sYl, LDH, kk, d0 + np * 16, lane));
          mma3(out[2 * np], crs[2 * np], ahi, alo, bhi, blo);
          mma3(out[2 * np + 1], crs[2 * np + 1], ahi, alo, bhi + 2, blo + 2);
        }
      } else {
        uint32_t bhi[2], blo[2];
        ldsm_x2_t(bhi, addr_bt2(sYh, LDH, kk, d0, lane & 15));
        ldsm_x2_t(blo, addr_bt2(sYl, LDH, kk, d0, lane & 15));
        mma3(out[0], crs[0], ahi, alo, bhi, blo);
      }
    }
    __syncthreads();                                    // the stage is refilled in the next iteration
  }
#pragma unroll
  for (int nt = 0; nt < NT; ++nt)
#pragma unroll
    for (int c = 0; c < 4; ++c) out[nt][c] = fmaf(crs[nt][c], LO_INV, out[nt][c]);
}

// stores the P.V fragments of tile_pv: rows i0 + m0 + g (+8), columns h*HD + d0 + 8*nt + 2t
template <int HD, int MB>
__device__ __forceinline__ void store_pv(float* __restrict__ O, int ldo, long long row0, int i0, int T, int h,
                                         const float (&out)[HD / 16][4], float mul) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int m0 = (warp % MB) * 16, d0 = (warp / MB) * (HD / 2);
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    const int i = i0 + m0 + g + 8 * half;
    if (i >= T) continue;
    float* orow = O + (row0 + i) * ldo + h * HD + d0 + 2 * t;
#pragma unroll
    for (int nt = 0; nt < HD / 16; ++nt)
      *reinterpret_cast<float2*>(orow + nt * 8) = make_float2(out[nt][2 * half] * mul, out[nt][2 * half + 1] * mul);
  }
}

// One score row in registers: lane l holds the pairs (2l + 64m, 2l + 64m + 1), m < MAX_PAIRS.
template <int NP> struct RowRegs { float2 v[NP]; };

template <int HD, int TQ, int NP, int NS>
__global__ void __launch_bounds__(TQ * 4, NP <= 2 ? 3 : 1) attention_fwd_kernel(
    const __half* __restrict__ Qh, const __half* __restrict__ Ql, const __half* __restrict__ Kh, const __half* __restrict__ Kl,
    const __half* __restrict__ Vh, const __half* __restrict__ Vl, int ldp, const float* __restrict__ key_bias, float* __restrict__ A,
    int ldA, float* __restrict__ O, int ldo, int H, int T, int S, float q_mul, float post_scale, int flags, Ragged rg) {
  constexpr int LDH = AttnSmem<HD>::LDH, ATT_THREADS = TQ * 4, ATT_WARPS = TQ / 8, MB = TQ / 16;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int S_pad = score_ld(S);  // floats per score row (from the dense S, also for ragged samples)
  float* sP = reinterpret_cast<float*>(smem_raw);
  __half* sQh = reinterpret_cast<__half*>(sP + (size_t)TQ * S_pad);
  __half* sQl = sQh + TQ * LDH;
  __half* sKV = sQl + TQ * LDH;                       // NS stages of K (then V) tile planes
  const int b = blockIdx.z, h = blockIdx.y, i0 = blockIdx.x * TQ;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int Tm = T;                                   // height of the staged plane
  long long qrow0 = (long long)b * T, krow0 = (long long)b * S;
  pdl_wait();                                         // launched as a programmatic dependent (launch_pdl)
  if (rg.lens) { T = S = rg.lens[b]; qrow0 = krow0 = rg.offs[b]; }
  if (i0 >= T) {                                      // tile entirely past this sample's rows: zero its A rows
    for (int e = tid; e < TQ * ldA; e += ATT_THREADS) {
      const int i = i0 + e / ldA;
      if (i < Tm) A[(((long long)b * H + h) * Tm + i) * ldA + e % ldA] = 0.f;
    }
    return;
  }
  ATT_TRACE(0);
  load_planes_async<HD, TQ>(Qh, Ql, ldp, qrow0 * ldp + h * HD, i0, T, sQh, sQl, q_mul);     // Q tile and the first K tiles together
#pragma unroll
  for (int pt = 0; pt < NS - 1; ++pt) issue_kv_tile<HD>(Kh, Kl, ldp, krow0 * ldp + h * HD, pt, S, sKV, NS);
  ATT_TRACE(1);
  tile_scores<HD, MB, NS>(Kh, Kl, ldp, krow0 * ldp + h * HD, S, sQh, sQl, sKV, sP, S_pad, post_scale, T - i0);
  ATT_TRACE(2);
#pragma unroll
  for (int pt = 0; pt < NS - 1; ++pt) issue_kv_tile<HD>(Vh, Vl, ldp, krow0 * ldp + h * HD, pt, S, sKV, NS);   // land during the softmax
  // softmax per row (warp w owns rows w*8 .. w*8+7): the row is read once into registers, normalised there, staged to A
  // with 8-byte stores and written back as fp16 hi / lo planes for the P.V product
  const int npairs = (S + 63) >> 6;                   // pairs per lane
  const int S16 = round_up(S, 16), lo_off = plane_lo_off(S);
  // Two rows per iteration (u = 0, 1), every stage written for both: the two dependency chains (shared-memory load ->
  // max -> shuffle tree -> exp -> shuffle tree -> normalise -> split -> stores) interleave, which is what a warp with
  // 2-6 resident neighbours per scheduler needs (a one-row loop leaves every stage waiting on the one before).
  constexpr int RPW = TQ / ATT_WARPS;
  constexpr int RI = NP <= 2 ? 4 : 2;                 // rows in flight: 4 while a row is 2 registers, 2 for the long rows (32 registers each)
  static_assert(RPW % RI == 0, "rows per iteration");
  for (int rr = 0; rr < RPW; rr += RI) {
    int i[RI];
    float* row[RI];
    bool live[RI];
#pragma unroll
    for (int u = 0; u < RI; ++u) {
      const int r = warp * RPW + rr + u;
      i[u] = i0 + r;
      row[u] = sP + (size_t)r * S_pad;
      live[u] = i[u] < T;
      if (!live[u]) {                                 // dead row of a live tile: zero A row, zero P planes (they multiply V rows)
        if (i[u] < Tm) for (int j = lane; j < ldA; j += 32) A[(((long long)b * H + h) * Tm + i[u]) * ldA + j] = 0.f;
        for (int j = lane; j < S_pad; j += 32) row[u][j] = 0.f;
      }
    }
    if (!live[0]) continue;                           // rows ascend: the others are dead as well
    RowRegs<NP> x[RI];
    float mx[RI];
#pragma unroll
    for (int u = 0; u < RI; ++u) mx[u] = -CUDART_INF_F;
#pragma unroll
    for (int m = 0; m < NP; ++m) {
      if (m < npairs) {
        const int j = 2 * lane + 64 * m;
#pragma unroll
        for (int u = 0; u < RI; ++u) {
          float2 v = make_float2(-CUDART_INF_F, -CUDART_INF_F);
          if (live[u] && j < S) {                     // j even, S_pad even and > S: the pair is readable; the entry S is masked
            v = *reinterpret_cast<const float2*>(row[u] + j);
            if (key_bias) { v.x += key_bias[(long long)b * S + j]; if (j + 1 < S) v.y += key_bias[(long long)b * S + j + 1]; }
            if (j + 1 >= S) v.y = -CUDART_INF_F;
            if (flags & MMX_ATTN_CAUSAL) { if (j > i[u]) v.x = -CUDART_INF_F; if (j + 1 > i[u]) v.y = -CUDART_INF_F; }
          }
          x[u].v[m] = v;
          mx[u] = fmaxf(mx[u], fmaxf(v.x, v.y));
        }
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
      for (int u = 0; u < RI; ++u) mx[u] = fmaxf(mx[u], __shfl_xor_sync(0xffffffffu, mx[u], o));
    }
    // A key whose bias is -inf is REMOVED (exp(-inf) = 0 exactly, the same bits a -10000 mask gives); a row whose keys are
    // all removed is the softmax over an empty set: A row = 0, output 0, like the reference's empty tensors when the
    // perturbation drivers drop every box (lxmert/lxmert/perturbation.py:110-117 at step 1.0).
    float mref[RI], sum[RI];
#pragma unroll
    for (int u = 0; u < RI; ++u) { mref[u] = mx[u] == -CUDART_INF_F ? 0.f : mx[u]; sum[u] = 0.f; }
#pragma unroll
    for (int m = 0; m < NP; ++m) {
      if (m < npairs) {
#pragma unroll
        for (int u = 0; u < RI; ++u) {
          x[u].v[m].x = expf(x[u].v[m].x - mref[u]);
          x[u].v[m].y = expf(x[u].v[m].y - mref[u]);
          sum[u] += x[u].v[m].x + x[u].v[m].y;
        }
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
      for (int u = 0; u < RI; ++u) sum[u] += __shfl_xor_sync(0xffffffffu, sum[u], o);
    }
    __syncwarp();                                     // every lane has read its part of the fp32 rows before the planes overwrite them
#pragma unroll
    for (int u = 0; u < RI; ++u) {
      if (!live[u]) continue;
      float* arow = A + (((long long)b * H + h) * Tm + i[u]) * ldA;
      __half* prow = reinterpret_cast<__half*>(row[u]);
      const float inv = sum[u] > 0.f ? 1.f / sum[u] : 0.f;   // one reciprocal per row; exp(-inf) = 0 beyond S
#pragma unroll
      for (int m = 0; m < NP; ++m) {
        if (m < npairs) {
          const int j = 2 * lane + 64 * m;
          const float2 p = make_float2(x[u].v[m].x * inv, x[u].v[m].y * inv);
          if (j < ldA) *reinterpret_cast<float2*>(arow + j) = p;          // ldA % 4 == 0 and j even: the pair is inside the row
          if (j < S16) {
            uint32_t ph, pl;
            split_f16(p.x, p.y, ph, pl);
            *reinterpret_cast<uint32_t*>(prow + j) = ph;
            *reinterpret_cast<uint32_t*>(prow + lo_off + j) = pl;
          }
        }
      }
      // a ragged sample covers 64 * npairs columns only: the rest of the dense plane row is zero like everything beyond S
      for (int j = 64 * npairs + lane; j < ldA; j += 32) arow[j] = 0.f;
    }
  }
  ATT_TRACE(3);
  __syncthreads();
  ATT_TRACE(4);
  float out[HD / 16][4];
  tile_pv<HD, MB, NS>(Vh, Vl, ldp, krow0 * ldp + h * HD, S, reinterpret_cast<const __half*>(sP), S_pad, lo_off, sKV, out, T - i0);
  ATT_TRACE(5);
  store_pv<HD, MB>(O, ldo, qrow0, i0, T, h, out, 1.f);
  ATT_TRACE(6);
}

// backward, query side: dA (staged), delta, dQ
template <int HD, int TQ, int NP, int NS>
__global__ void __launch_bounds__(TQ * 4, NP <= 2 ? 3 : 1) attention_bwd_q_kernel(
    const __half* __restrict__ Gh, const __half* __restrict__ Gl, int ldg, const __half* __restrict__ Kh, const __half* __restrict__ Kl,
    const __half* __restrict__ Vh, const __half* __restrict__ Vl, int ldp, const float* __restrict__ A, float* __restrict__ dA, int ldA,
    float* __restrict__ delta, float* __restrict__ dQ, int lddq, int H, int T, int S, float scale, Ragged rg,
    const float* __restrict__ gscale) {
  constexpr int LDH = AttnSmem<HD>::LDH, ATT_THREADS = TQ * 4, ATT_WARPS = TQ / 8, MB = TQ / 16;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int S_pad = score_ld(S);
  float* sP = reinterpret_cast<float*>(smem_raw);
  __half* sXh = reinterpret_cast<__half*>(sP + (size_t)TQ * S_pad);
  __half* sXl = sXh + TQ * LDH;
  __half* sKV = sXl + TQ * LDH;                       // NS stages of V (then K) tile planes
  const int b = blockIdx.z, h = blockIdx.y, i0 = blockIdx.x * TQ;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int Tm = T;
  long long qrow0 = (long long)b * T, krow0 = (long long)b * S;
  pdl_wait();
  if (rg.lens) { T = S = rg.lens[b]; qrow0 = krow0 = rg.offs[b]; }
  if (i0 >= T) {                                      // past this sample's rows: the hooked gradient is zero there
    for (int e = tid; e < TQ * ldA; e += ATT_THREADS) {
      const int i = i0 + e / ldA;
      if (i < Tm) dA[(((long long)b * H + h) * Tm + i) * ldA + e % ldA] = 0.f;
    }
    return;
  }
  // The gradient stream of sample b may carry a power-of-two factor gscale[b] (fp16 range, see gemm_wgmma.cu); the staged
  // dA is divided by it (exact), everything that continues the backward (delta, dS, dQ) stays scaled.
  const float ginv = gscale ? 1.f / gscale[b] : 1.f;
  load_planes_async<HD, TQ>(Gh, Gl, ldg, qrow0 * ldg + h * HD, i0, T, sXh, sXl);
#pragma unroll
  for (int pt = 0; pt < NS - 1; ++pt) issue_kv_tile<HD>(Vh, Vl, ldp, krow0 * ldp + h * HD, pt, S, sKV, NS);
  tile_scores<HD, MB, NS>(Vh, Vl, ldp, krow0 * ldp + h * HD, S, sXh, sXl, sKV, sP, S_pad, 1.f, T - i0);
  if (dQ != nullptr) {                                                                    // land while dA is staged
#pragma unroll
    for (int pt = 0; pt < NS - 1; ++pt) issue_kv_tile<HD>(Kh, Kl, ldp, krow0 * ldp + h * HD, pt, S, sKV, NS);
  }
  const int npairs = (S + 63) >> 6;
  const int S16 = round_up(S, 16), lo_off = plane_lo_off(S);
  constexpr int RPW = TQ / ATT_WARPS;                 // RI rows per iteration, stage by stage (see the forward kernel)
  constexpr int RI = NP <= 2 ? 4 : 2;
  static_assert(RPW % RI == 0, "rows per iteration");
  for (int rr = 0; rr < RPW; rr += RI) {
    int i[RI];
    float* row[RI];
    bool live[RI];
    long long goff[RI];
#pragma unroll
    for (int u = 0; u < RI; ++u) {
      const int r = warp * RPW + rr + u;
      i[u] = i0 + r;
      row[u] = sP + (size_t)r * S_pad;
      live[u] = i[u] < T;
      goff[u] = (((long long)b * H + h) * Tm + i[u]) * ldA;
      if (!live[u]) {
        if (i[u] < Tm) for (int j = lane; j < ldA; j += 32) dA[goff[u] + j] = 0.f;
        if (dQ != nullptr) for (int j = lane; j < S_pad; j += 32) row[u][j] = 0.f;
      }
    }
    if (!live[0]) continue;
    RowRegs<NP> gr[RI], ar[RI];
    float dl[RI];
#pragma unroll
    for (int u = 0; u < RI; ++u) dl[u] = 0.f;
#pragma unroll
    for (int m = 0; m < NP; ++m) {
      if (m < npairs) {
        const int j = 2 * lane + 64 * m;
#pragma unroll
        for (int u = 0; u < RI; ++u) {
          float2 gv = make_float2(0.f, 0.f), av = make_float2(0.f, 0.f);
          if (live[u]) {
            if (j < S) {
              gv = *reinterpret_cast<const float2*>(row[u] + j);
              if (j + 1 >= S) gv.y = 0.f;
            }
            if (j < ldA) {
              av = *reinterpret_cast<const float2*>(A + goff[u] + j);           // pad columns of A are zero
              *reinterpret_cast<float2*>(dA + goff[u] + j) = make_float2(gv.x * ginv, gv.y * ginv);   // the hooked gradient, unmasked, in TRUE units
            }
          }
          gr[u].v[m] = gv; ar[u].v[m] = av;
          dl[u] = fmaf(gv.x, av.x, dl[u]);
          dl[u] = fmaf(gv.y, av.y, dl[u]);
        }
      }
    }
#pragma unroll
    for (int u = 0; u < RI; ++u)
      if (live[u]) for (int j = 64 * npairs + lane; j < ldA; j += 32) dA[goff[u] + j] = 0.f;   // columns a ragged sample's pairs did not reach
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
      for (int u = 0; u < RI; ++u) dl[u] += __shfl_xor_sync(0xffffffffu, dl[u], o);
    }
    if (lane == 0 && delta) {
#pragma unroll
      for (int u = 0; u < RI; ++u)
        if (live[u]) delta[((long long)b * H + h) * Tm + i[u]] = dl[u];
    }
    if (dQ != nullptr) {
      __syncwarp();                                   // the fp32 rows have been read by every lane before dS overwrites them
#pragma unroll
      for (int u = 0; u < RI; ++u) {
        if (!live[u]) continue;
        __half* prow = reinterpret_cast<__half*>(row[u]);
#pragma unroll
        for (int m = 0; m < NP; ++m) {
          if (m < npairs) {
            const int j = 2 * lane + 64 * m;
            if (j < S16) {
              uint32_t sh, sl;                                                      // dS = A (.) (dA - delta); A = 0 beyond S
              split_f16(ar[u].v[m].x * (gr[u].v[m].x - dl[u]), ar[u].v[m].y * (gr[u].v[m].y - dl[u]), sh, sl);
              *reinterpret_cast<uint32_t*>(prow + j) = sh;
              *reinterpret_cast<uint32_t*>(prow + lo_off + j) = sl;
            }
          }
        }
      }
    }
  }
  if (dQ == nullptr) return;
  __syncthreads();
  float out[HD / 16][4];
  tile_pv<HD, MB, NS>(Kh, Kl, ldp, krow0 * ldp + h * HD, S, reinterpret_cast<const __half*>(sP), S_pad, lo_off, sKV, out, T - i0);
  store_pv<HD, MB>(dQ, lddq, qrow0, i0, T, h, out, scale);
}

// backward, key side: one CTA = 64 keys of one (b,h) (a whole CLIP ViT-B/32 head); walks the query rows in tiles of 64.
//   dV[j] = sum_i A[i][j] dO[i]      dK[j] = scale * sum_i dS[i][j] Q[i],  dS = A (.) (dA - delta_i)
// Warp w owns the 16-key block w&3 and the d half w>>2 of both products.  A and dS tiles are built from the staged fp32
// planes (split on the fly: every element is used by one CTA only), dO and Q tiles arrive as pre-split planes.
constexpr int KV_KEYS = 64, KV_ROWS = 64;
template <int HD>
__global__ void __launch_bounds__(KV_THREADS) attention_bwd_kv_kernel(
    const __half* __restrict__ Gh, const __half* __restrict__ Gl, int ldg, const __half* __restrict__ Qh, const __half* __restrict__ Ql,
    int ldp, const float* __restrict__ A, const float* __restrict__ dA, int ldA, const float* __restrict__ delta, float* __restrict__ dK, int lddk,
    float* __restrict__ dV, int lddv, int H, int T, int S, float scale, Ragged rg, const float* __restrict__ gscale) {
  constexpr int LDH = HD + 8, LDK = KV_KEYS + 8, NT = HD / 16;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __half* sGh = reinterpret_cast<__half*>(smem_raw);
  __half* sGl = sGh + KV_ROWS * LDH;
  __half* sQh = sGl + KV_ROWS * LDH;
  __half* sQl = sQh + KV_ROWS * LDH;
  __half* sAh = sQl + KV_ROWS * LDH;       // [KV_ROWS][LDK]  A[i][j]
  __half* sAl = sAh + KV_ROWS * LDK;
  __half* sSh = sAl + KV_ROWS * LDK;       // [KV_ROWS][LDK]  dS[i][j]
  __half* sSl = sSh + KV_ROWS * LDK;
  const int b = blockIdx.z, h = blockIdx.y, j0 = blockIdx.x * KV_KEYS;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int m0 = (warp & 3) * 16, d0 = (warp >> 2) * (HD / 2);   // this warp's 16 keys and d half
  const int Tm = T;
  long long qrow0 = (long long)b * T, krow0 = (long long)b * S;
  pdl_wait();
  if (rg.lens) { T = S = rg.lens[b]; qrow0 = krow0 = rg.offs[b]; }
  if (j0 >= S) return;
  const float gs = gscale ? gscale[b] : 1.f;           // staged dA is in true units, delta / dO / the outputs are scaled
  float accV[NT][4] = {}, crsV[NT][4] = {}, accK[NT][4] = {}, crsK[NT][4] = {};
  const long long plane = ((long long)b * H + h) * Tm;
  for (int i0 = 0; i0 < T; i0 += KV_ROWS) {
    __syncthreads();
    load_planes_async<HD, KV_ROWS>(Gh, Gl, ldg, qrow0 * ldg + h * HD, i0, T, sGh, sGl);
    load_planes_async<HD, KV_ROWS>(Qh, Ql, ldp, qrow0 * ldp + h * HD, i0, T, sQh, sQl);
    cp_async_commit();
    // A and dS tiles: 4 keys per 128-bit load.  Staged rows are ldA (% 4 == 0) wide and zero beyond this sample's
    // keys, so a float4 that starts below ldA is entirely readable and entirely correct.
    for (int e = tid; e < KV_ROWS * (KV_KEYS / 4); e += KV_THREADS) {
      const int r = e / (KV_KEYS / 4), c = (e % (KV_KEYS / 4)) * 4;
      float4 a = make_float4(0.f, 0.f, 0.f, 0.f), ds = a;
      if (i0 + r < T && j0 + c < ldA) {
        const long long off = (plane + i0 + r) * ldA + j0 + c;
        a = *reinterpret_cast<const float4*>(A + off);
        const float4 ga = *reinterpret_cast<const float4*>(dA + off);
        const float dl = delta[plane + i0 + r];
        ds = make_float4(a.x * (ga.x * gs - dl), a.y * (ga.y * gs - dl), a.z * (ga.z * gs - dl), a.w * (ga.w * gs - dl));
      }
      uint2 ah, al, sh, sl;
      split_f16(a.x, a.y, ah.x, al.x);
      split_f16(a.z, a.w, ah.y, al.y);
      split_f16(ds.x, ds.y, sh.x, sl.x);
      split_f16(ds.z, ds.w, sh.y, sl.y);
      *reinterpret_cast<uint2*>(sAh + r * LDK + c) = ah;
      *reinterpret_cast<uint2*>(sAl + r * LDK + c) = al;
      *reinterpret_cast<uint2*>(sSh + r * LDK + c) = sh;
      *reinterpret_cast<uint2*>(sSl + r * LDK + c) = sl;
    }
    cp_async_wait_all();
    __syncthreads();
    const int in = min(KV_ROWS, T - i0);                // rows in .. round_up(in, 16) are zero-filled
    if (j0 + m0 < S) {                                  // this warp's 16 keys are live (warp-uniform)
#pragma unroll 2
      for (int kk = 0; kk < in; kk += 16) {
        uint32_t aAh[4], aAl[4], aSh[4], aSl[4];
        ldsm_x4_t(aAh, addr_at(sAh, LDK, kk, m0, lane));
        ldsm_x4_t(aAl, addr_at(sAl, LDK, kk, m0, lane));
        ldsm_x4_t(aSh, addr_at(sSh, LDK, kk, m0, lane));
        ldsm_x4_t(aSl, addr_at(sSl, LDK, kk, m0, lane));
        if constexpr (NT >= 2) {
#pragma unroll
          for (int np = 0; np < NT / 2; ++np) {
            uint32_t bh[4], bl[4];
            ldsm_x4_t(bh, addr_bt2(sGh, LDH, kk, d0 + np * 16, lane));
            ldsm_x4_t(bl, addr_bt2(sGl, LDH, kk, d0 + np * 16, lane));
            mma3(accV[2 * np], crsV[2 * np], aAh, aAl, bh, bl);
            mma3(accV[2 * np + 1], crsV[2 * np + 1], aAh, aAl, bh + 2, bl + 2);
            ldsm_x4_t(bh, addr_bt2(sQh, LDH, kk, d0 + np * 16, lane));
            ldsm_x4_t(bl, addr_bt2(sQl, LDH, kk, d0 + np * 16, lane));
            mma3(accK[2 * np], crsK[2 * np], aSh, aSl, bh, bl);
            mma3(accK[2 * np + 1], crsK[2 * np + 1], aSh, aSl, bh + 2, bl + 2);
          }
        } else {
          uint32_t bh[2], bl[2];
          ldsm_x2_t(bh, addr_bt2(sGh, LDH, kk, d0, lane & 15));
          ldsm_x2_t(bl, addr_bt2(sGl, LDH, kk, d0, lane & 15));
          mma3(accV[0], crsV[0], aAh, aAl, bh, bl);
          ldsm_x2_t(bh, addr_bt2(sQh, LDH, kk, d0, lane & 15));
          ldsm_x2_t(bl, addr_bt2(sQl, LDH, kk, d0, lane & 15));
          mma3(accK[0], crsK[0], aSh, aSl, bh, bl);
        }
      }
    }
  }
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    const int j = j0 + m0 + g + 8 * half;
    if (j >= S) continue;
    float* vrow = dV + (krow0 + j) * lddv + h * HD + d0 + 2 * t;
    float* krow = dK + (krow0 + j) * lddk + h * HD + d0 + 2 * t;
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
      *reinterpret_cast<float2*>(vrow + nt * 8) = make_float2(fmaf(crsV[nt][2 * half], LO_INV, accV[nt][2 * half]),
                                                              fmaf(crsV[nt][2 * half + 1], LO_INV, accV[nt][2 * half + 1]));
      *reinterpret_cast<float2*>(krow + nt * 8) = make_float2(fmaf(crsK[nt][2 * half], LO_INV, accK[nt][2 * half]) * scale,
                                                              fmaf(crsK[nt][2 * half + 1], LO_INV, accK[nt][2 * half + 1]) * scale);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Long rows: the shapes the single-pass kernels reject (S > 1024, or score rows of a tile beyond shared memory; DETR's
// DC5 maps have 2500 - 4200 keys).  Nothing holds a whole score row: one CTA = one (b, h, 64-query tile), 8 warps, and
// the keys stream through shared memory TWICE as 64-key tiles in one cp.async ring (pass-1 tiles, then pass-2 tiles, so
// the first pass-2 tiles land while pass 1 finishes).  Warp w computes the 16x32 block (rows (w % 4) * 16, keys
// (w / 4) * 32) of every 64x64 score tile in registers with the same fp16x3 mma.sync products as the short kernels.
//   forward   pass 1: running row max and sum of exp (per-thread online rescale, combined across the quad and the two
//                     key halves at the end; fixed order, deterministic);
//             pass 2: recompute each score tile, normalise, write the A tile (through shared memory: 256-byte row
//                     stores) and accumulate O += P.V on the probability planes.
//   backward  pass 1: dA = dO.V^T tile, staged (divided by gscale), delta = rowsum(dA (.) A) from the staged A;
//             pass 2: re-read A / dA (each thread reads back what it wrote), dS = A (.) (dA - delta), dQ += scale dS.K.
// The score tile is recomputed instead of stored, so the bound is the A / dA plane traffic (8 bytes per element written
// or read per pass), not the products.  Plane offsets are 64-bit (B*H*T*ld passes 2^31 at B = 16, S = 4200).
constexpr int LTQ = 64, LONG_THREADS = 256, LONG_MAX_S = 16384;
constexpr int LDT = TKEY + 4;     // floats per row of the fp32 tile (16-byte aligned rows)
constexpr int LDT16 = TKEY + 8;   // halves per row of a probability / dS plane tile (144 bytes: conflict-free ldmatrix)

template <int HD>
struct LongSmem {
  static constexpr int LDH = HD + 8, ST = AttnSmem<HD>::STAGE;   // one K or V tile as hi + lo planes
  // fp32 tile + row statistics, X (Q or dO) planes, P / dS planes, NS ring stages of `per_stage` tiles
  static size_t bytes(int NS, int per_stage) {
    return sizeof(float) * ((size_t)LTQ * LDT + 4 * LTQ) +
           sizeof(__half) * (2 * (size_t)LTQ * LDH + 2 * (size_t)LTQ * LDT16 + (size_t)NS * per_stage * ST);
  }
};

// Item `it` of the two-pass key stream into ring stage it % NS (stage stride `sstride` halves): it < nkt -> key tile it
// of P1; nkt <= it < nit -> key tile it - nkt of P2 (and of P3, into the second half of the stage, when P3h != nullptr).
// One commit group per item, empty past the end.
template <int HD>
__device__ __forceinline__ void issue_stream(const __half* __restrict__ P1h, const __half* __restrict__ P1l, const __half* __restrict__ P2h,
                                             const __half* __restrict__ P2l, const __half* __restrict__ P3h, const __half* __restrict__ P3l,
                                             int ldp, long long base, int it, int nkt, int nit, int S, __half* sKV, int NS, int sstride) {
  constexpr int LDH = HD + 8;
  if (it < nit) {
    __half* st = sKV + (size_t)(it % NS) * sstride;
    if (it < nkt) {
      load_planes_async<HD, TKEY>(P1h, P1l, ldp, base, it * TKEY, S, st, st + TKEY * LDH);
    } else {
      load_planes_async<HD, TKEY>(P2h, P2l, ldp, base, (it - nkt) * TKEY, S, st, st + TKEY * LDH);
      if (P3h != nullptr) {
        __half* s3 = st + AttnSmem<HD>::STAGE;
        load_planes_async<HD, TKEY>(P3h, P3l, ldp, base, (it - nkt) * TKEY, S, s3, s3 + TKEY * LDH);
      }
    }
  }
  cp_async_commit();
}

// The warp's 16x32 block of one 64x64 score tile: s[nt][c] = sum_d X[m0 + g + 8 (c >> 1)][d] * Y[kh + 8 nt + 2t + (c & 1)][d]
template <int HD>
__device__ __forceinline__ void score_block(const __half* sXh, const __half* sXl, const __half* sYh, const __half* sYl, int m0, int kh,
                                            int lane, float (&s)[4][4]) {
  constexpr int LDH = HD + 8;
  float crs[4][4];
#pragma unroll
  for (int nt = 0; nt < 4; ++nt)
#pragma unroll
    for (int c = 0; c < 4; ++c) s[nt][c] = crs[nt][c] = 0.f;
#pragma unroll
  for (int k0 = 0; k0 < HD; k0 += 16) {
    uint32_t ahi[4], alo[4];
    ldsm_x4(ahi, addr_a(sXh, LDH, m0, k0, lane));
    ldsm_x4(alo, addr_a(sXl, LDH, m0, k0, lane));
#pragma unroll
    for (int np = 0; np < 2; ++np) {
      uint32_t bhi[4], blo[4];
      ldsm_x4(bhi, addr_b2(sYh, LDH, kh + np * 16, k0, lane));
      ldsm_x4(blo, addr_b2(sYl, LDH, kh + np * 16, k0, lane));
      mma3(s[2 * np], crs[2 * np], ahi, alo, bhi, blo);
      mma3(s[2 * np + 1], crs[2 * np + 1], ahi, alo, bhi + 2, blo + 2);
    }
  }
#pragma unroll
  for (int nt = 0; nt < 4; ++nt)
#pragma unroll
    for (int c = 0; c < 4; ++c) s[nt][c] = fmaf(crs[nt][c], LO_INV, s[nt][c]);
}

// out[HD/16][4] (+ crs) += P.Y over one 64-key tile: P as planes [row][key] (LDT16), Y tile [key][d] as planes (transposed
// on load).  Warp w: rows (w % 4) * 16, d half w / 4.  Keys jn .. 63 are zero in both operands and skipped.  The main
// products of the tile are summed in their own accumulator and added to `out` once: over thousands of keys a single fp32
// accumulator would grow its rounding error with sqrt(S) relative to the (1/sqrt(S)-sized) output.
template <int HD>
__device__ __forceinline__ void pv_block(const __half* sPh, const __half* sPl, const __half* sYh, const __half* sYl, int m0, int d0,
                                         int jn, int lane, float (&out)[HD / 16][4], float (&crs)[HD / 16][4]) {
  constexpr int LDH = HD + 8, NT = HD / 16;
  float acc[NT][4];
#pragma unroll
  for (int nt = 0; nt < NT; ++nt)
#pragma unroll
    for (int c = 0; c < 4; ++c) acc[nt][c] = 0.f;
  for (int kk = 0; kk < jn; kk += 16) {
    uint32_t ahi[4], alo[4];
    ldsm_x4(ahi, addr_a(sPh, LDT16, m0, kk, lane));
    ldsm_x4(alo, addr_a(sPl, LDT16, m0, kk, lane));
    if constexpr (NT >= 2) {
#pragma unroll
      for (int np = 0; np < NT / 2; ++np) {
        uint32_t bhi[4], blo[4];
        ldsm_x4_t(bhi, addr_bt2(sYh, LDH, kk, d0 + np * 16, lane));
        ldsm_x4_t(blo, addr_bt2(sYl, LDH, kk, d0 + np * 16, lane));
        mma3(acc[2 * np], crs[2 * np], ahi, alo, bhi, blo);
        mma3(acc[2 * np + 1], crs[2 * np + 1], ahi, alo, bhi + 2, blo + 2);
      }
    } else {
      uint32_t bhi[2], blo[2];
      ldsm_x2_t(bhi, addr_bt2(sYh, LDH, kk, d0, lane & 15));
      ldsm_x2_t(blo, addr_bt2(sYl, LDH, kk, d0, lane & 15));
      mma3(acc[0], crs[0], ahi, alo, bhi, blo);
    }
  }
#pragma unroll
  for (int nt = 0; nt < NT; ++nt)
#pragma unroll
    for (int c = 0; c < 4; ++c) out[nt][c] += acc[nt][c];
}

// (m, s) <- the combination of two partial softmax statistics; -inf maxima (every key masked so far) contribute nothing
__device__ __forceinline__ void merge_stats(float& m, float& s, float m2, float s2) {
  const float M = fmaxf(m, m2), mref = M == -CUDART_INF_F ? 0.f : M;
  s = s * expf(m - mref) + s2 * expf(m2 - mref);
  m = M;
}

template <int HD, int NS>
__global__ void __launch_bounds__(LONG_THREADS, HD <= 32 ? 2 : 1) attention_fwd_long_kernel(
    const __half* __restrict__ Qh, const __half* __restrict__ Ql, const __half* __restrict__ Kh, const __half* __restrict__ Kl,
    const __half* __restrict__ Vh, const __half* __restrict__ Vl, int ldp, const float* __restrict__ key_bias, float* __restrict__ A,
    int ldA, float* __restrict__ O, int ldo, int H, int T, int S, float post_scale, int flags) {
  constexpr int LDH = HD + 8, MB = LTQ / 16, ST = AttnSmem<HD>::STAGE, NT = HD / 16;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float* sT = reinterpret_cast<float*>(smem_raw);                 // [LTQ][LDT] normalised probabilities of the tile
  float* sStat = sT + LTQ * LDT;                                  // [key half][max, sum][LTQ]
  __half* sXh = reinterpret_cast<__half*>(sStat + 4 * LTQ);
  __half* sXl = sXh + LTQ * LDH;
  __half* sPh = sXl + LTQ * LDH;                                  // [LTQ][LDT16] probability planes
  __half* sPl = sPh + LTQ * LDT16;
  __half* sKV = sPl + LTQ * LDT16;                                // NS stages of (K tile, V tile) planes
  const int b = blockIdx.z, h = blockIdx.y, i0 = blockIdx.x * LTQ;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int m0 = (warp % MB) * 16, kh = (warp / MB) * 32, d0 = (warp / MB) * (HD / 2);
  const long long kbase = (long long)b * S * ldp + h * HD, plane = ((long long)b * H + h) * T;
  const int nkt = cdiv(S, TKEY), nit = 2 * nkt;
  pdl_wait();
  load_planes_async<HD, LTQ>(Qh, Ql, ldp, (long long)b * T * ldp + h * HD, i0, T, sXh, sXl);   // shares tile 0's group
#pragma unroll
  for (int pt = 0; pt < NS - 1; ++pt) issue_stream<HD>(Kh, Kl, Kh, Kl, Vh, Vl, ldp, kbase, pt, nkt, nit, S, sKV, NS, 2 * ST);
  // score (row m0 + g + 8 (c >> 1), key j0 + kh + 8 nt + 2t + (c & 1)) with the short kernel's order: scale, bias, masks
  auto finish_scores = [&](float (&s)[4][4], int j0) {
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const int i = i0 + m0 + g + 8 * (c >> 1), j = j0 + kh + 8 * nt + 2 * t + (c & 1);
        float v = s[nt][c] * post_scale;
        if (j >= S) v = -CUDART_INF_F;
        else {
          if (key_bias) v += key_bias[(long long)b * S + j];
          if ((flags & MMX_ATTN_CAUSAL) && j > i) v = -CUDART_INF_F;
        }
        s[nt][c] = v;
      }
  };
  // ---- pass 1: row statistics (rows m0 + g and m0 + g + 8 of this thread, over its 8 keys of each tile)
  float mrun[2] = {-CUDART_INF_F, -CUDART_INF_F}, srun[2] = {0.f, 0.f};
  for (int it = 0; it < nkt; ++it) {
    issue_stream<HD>(Kh, Kl, Kh, Kl, Vh, Vl, ldp, kbase, it + NS - 1, nkt, nit, S, sKV, NS, 2 * ST);
    cp_async_wait<NS - 1>();
    __syncthreads();
    const __half* sYh = sKV + (size_t)(it % NS) * 2 * ST;
    float s[4][4];
    score_block<HD>(sXh, sXl, sYh, sYh + TKEY * LDH, m0, kh, lane, s);
    finish_scores(s, it * TKEY);
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      float tm = -CUDART_INF_F;
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) tm = fmaxf(tm, fmaxf(s[nt][2 * r], s[nt][2 * r + 1]));
      const float M = fmaxf(mrun[r], tm), mref = M == -CUDART_INF_F ? 0.f : M;
      float acc = srun[r] * expf(mrun[r] - mref);
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) acc += expf(s[nt][2 * r] - mref) + expf(s[nt][2 * r + 1] - mref);
      srun[r] = acc;
      mrun[r] = M;
    }
    __syncthreads();                                  // the stage is refilled in the next iteration
  }
  // across the quad (commutative pairwise merges: all four lanes end with the same bits), then across the key halves
#pragma unroll
  for (int o = 1; o <= 2; o <<= 1)
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const float m2 = __shfl_xor_sync(0xffffffffu, mrun[r], o), s2 = __shfl_xor_sync(0xffffffffu, srun[r], o);
      merge_stats(mrun[r], srun[r], m2, s2);
    }
  if (t == 0) {
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      sStat[(warp / MB) * 2 * LTQ + m0 + g + 8 * r] = mrun[r];
      sStat[(warp / MB) * 2 * LTQ + LTQ + m0 + g + 8 * r] = srun[r];
    }
  }
  __syncthreads();
  float mref[2], inv[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = m0 + g + 8 * r;
    float m = sStat[row], sum = sStat[LTQ + row];
    merge_stats(m, sum, sStat[2 * LTQ + row], sStat[3 * LTQ + row]);
    mref[r] = m == -CUDART_INF_F ? 0.f : m;
    inv[r] = sum > 0.f ? 1.f / sum : 0.f;            // a row whose keys are all removed: A = 0, output 0
  }
  // ---- pass 2: normalised tiles -> A (staged) and the probability planes -> O += P.V
  float out[NT][4], crs[NT][4];
#pragma unroll
  for (int nt = 0; nt < NT; ++nt)
#pragma unroll
    for (int c = 0; c < 4; ++c) out[nt][c] = crs[nt][c] = 0.f;
  for (int it = nkt; it < nit; ++it) {
    issue_stream<HD>(Kh, Kl, Kh, Kl, Vh, Vl, ldp, kbase, it + NS - 1, nkt, nit, S, sKV, NS, 2 * ST);
    cp_async_wait<NS - 1>();
    __syncthreads();
    const __half* sYh = sKV + (size_t)(it % NS) * 2 * ST;
    const int j0 = (it - nkt) * TKEY;
    float s[4][4];
    score_block<HD>(sXh, sXl, sYh, sYh + TKEY * LDH, m0, kh, lane, s);
    finish_scores(s, j0);
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const float2 p = make_float2(expf(s[nt][2 * r] - mref[r]) * inv[r], expf(s[nt][2 * r + 1] - mref[r]) * inv[r]);
        const int row = m0 + g + 8 * r, col = kh + 8 * nt + 2 * t;
        *reinterpret_cast<float2*>(sT + row * LDT + col) = p;
        uint32_t ph, pl;
        split_f16(p.x, p.y, ph, pl);
        *reinterpret_cast<uint32_t*>(sPh + row * LDT16 + col) = ph;
        *reinterpret_cast<uint32_t*>(sPl + row * LDT16 + col) = pl;
      }
    __syncthreads();
    for (int e = tid; e < LTQ * (TKEY / 4); e += LONG_THREADS) {     // 16 threads per 256-byte row segment
      const int r = e / (TKEY / 4), c = (e % (TKEY / 4)) * 4, i = i0 + r, j = j0 + c;
      if (i < T && j < ldA) *reinterpret_cast<float4*>(A + (plane + i) * ldA + j) = *reinterpret_cast<const float4*>(sT + r * LDT + c);
    }
    pv_block<HD>(sPh, sPl, sYh + ST, sYh + ST + TKEY * LDH, m0, d0, min(TKEY, S - j0), lane, out, crs);
    __syncthreads();                                  // the stage and the tiles are rewritten in the next iteration
  }
  const int jz = nkt * TKEY;                          // pad columns the tiles did not reach
  if (jz < ldA)
    for (int e = tid; e < LTQ * (ldA - jz); e += LONG_THREADS) {
      const int i = i0 + e / (ldA - jz);
      if (i < T) A[(plane + i) * ldA + jz + e % (ldA - jz)] = 0.f;
    }
#pragma unroll
  for (int nt = 0; nt < NT; ++nt)
#pragma unroll
    for (int c = 0; c < 4; ++c) out[nt][c] = fmaf(crs[nt][c], LO_INV, out[nt][c]);
  store_pv<HD, MB>(O, ldo, (long long)b * T, i0, T, h, out, 1.f);
}

template <int HD, int NS>
__global__ void __launch_bounds__(LONG_THREADS, 2) attention_bwd_q_long_kernel(
    const __half* __restrict__ Gh, const __half* __restrict__ Gl, int ldg, const __half* __restrict__ Kh, const __half* __restrict__ Kl,
    const __half* __restrict__ Vh, const __half* __restrict__ Vl, int ldp, const float* __restrict__ A, float* __restrict__ dA, int ldA,
    float* __restrict__ delta, float* __restrict__ dQ, int lddq, int H, int T, int S, float scale, const float* __restrict__ gscale) {
  constexpr int LDH = HD + 8, MB = LTQ / 16, ST = AttnSmem<HD>::STAGE, NT = HD / 16, RPW = LTQ / (LONG_THREADS / 32);
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float* sT = reinterpret_cast<float*>(smem_raw);                 // [LTQ][LDT] dA tile (scaled units)
  float* sDelta = sT + LTQ * LDT;                                 // [LTQ]
  __half* sXh = reinterpret_cast<__half*>(sDelta + 4 * LTQ);
  __half* sXl = sXh + LTQ * LDH;
  __half* sPh = sXl + LTQ * LDH;                                  // [LTQ][LDT16] dS planes
  __half* sPl = sPh + LTQ * LDT16;
  __half* sKV = sPl + LTQ * LDT16;                                // NS stages of one V (pass 1) or K (pass 2) tile
  const int b = blockIdx.z, h = blockIdx.y, i0 = blockIdx.x * LTQ;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int m0 = (warp % MB) * 16, kh = (warp / MB) * 32, d0 = (warp / MB) * (HD / 2);
  const long long kbase = (long long)b * S * ldp + h * HD, plane = ((long long)b * H + h) * T;
  const int nkt = cdiv(S, TKEY), nit = dQ != nullptr ? 2 * nkt : nkt;
  pdl_wait();
  // dA is staged in TRUE units (divided by the power-of-two gscale[b], exact); delta, dS and dQ stay scaled
  const float gs = gscale ? gscale[b] : 1.f, ginv = gscale ? 1.f / gscale[b] : 1.f;
  load_planes_async<HD, LTQ>(Gh, Gl, ldg, (long long)b * T * ldg + h * HD, i0, T, sXh, sXl);
#pragma unroll
  for (int pt = 0; pt < NS - 1; ++pt) issue_stream<HD>(Vh, Vl, Kh, Kl, nullptr, nullptr, ldp, kbase, pt, nkt, nit, S, sKV, NS, ST);
  // ---- pass 1: dA tiles -> staged dA, delta.  Warp w owns rows w * RPW .. +RPW-1, lane l the key pair (2l, 2l+1) of a tile.
  float dl[RPW];
#pragma unroll
  for (int u = 0; u < RPW; ++u) dl[u] = 0.f;
  for (int it = 0; it < nkt; ++it) {
    issue_stream<HD>(Vh, Vl, Kh, Kl, nullptr, nullptr, ldp, kbase, it + NS - 1, nkt, nit, S, sKV, NS, ST);
    cp_async_wait<NS - 1>();
    __syncthreads();
    const __half* sYh = sKV + (size_t)(it % NS) * ST;
    const int j0 = it * TKEY;
    float s[4][4];
    score_block<HD>(sXh, sXl, sYh, sYh + TKEY * LDH, m0, kh, lane, s);
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int col = kh + 8 * nt + 2 * t;
        float2 v = make_float2(s[nt][2 * r], s[nt][2 * r + 1]);
        if (j0 + col >= S) v.x = 0.f;
        if (j0 + col + 1 >= S) v.y = 0.f;
        *reinterpret_cast<float2*>(sT + (m0 + g + 8 * r) * LDT + col) = v;
      }
    __syncthreads();
    const int j = j0 + 2 * lane;
#pragma unroll
    for (int u = 0; u < RPW; ++u) {
      const int r = warp * RPW + u, i = i0 + r;
      if (i < T && j < ldA) {                         // j even, ldA % 4 == 0: the pair is inside the row
        const float2 gv = *reinterpret_cast<const float2*>(sT + r * LDT + 2 * lane);
        const long long off = (plane + i) * ldA + j;
        const float2 av = *reinterpret_cast<const float2*>(A + off);     // pad columns of A are zero
        *reinterpret_cast<float2*>(dA + off) = make_float2(gv.x * ginv, gv.y * ginv);
        dl[u] = fmaf(gv.x, av.x, dl[u]);
        dl[u] = fmaf(gv.y, av.y, dl[u]);
      }
    }
    __syncthreads();                                  // the stage and the tile are rewritten in the next iteration
  }
  const int jz = nkt * TKEY;
#pragma unroll
  for (int u = 0; u < RPW; ++u) {
    const int r = warp * RPW + u, i = i0 + r;
    if (i < T) for (int j = jz + lane; j < ldA; j += 32) dA[(plane + i) * ldA + j] = 0.f;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) dl[u] += __shfl_xor_sync(0xffffffffu, dl[u], o);
    if (lane == 0) {
      sDelta[r] = dl[u];
      if (delta && i < T) delta[plane + i] = dl[u];
    }
  }
  if (dQ == nullptr) return;
  __syncwarp();                                       // sDelta of the warp's rows is read by every lane below
  // ---- pass 2: dS = A (.) (dA - delta) planes -> dQ += dS.K
  float out[NT][4], crs[NT][4];
#pragma unroll
  for (int nt = 0; nt < NT; ++nt)
#pragma unroll
    for (int c = 0; c < 4; ++c) out[nt][c] = crs[nt][c] = 0.f;
  for (int it = nkt; it < nit; ++it) {
    issue_stream<HD>(Vh, Vl, Kh, Kl, nullptr, nullptr, ldp, kbase, it + NS - 1, nkt, nit, S, sKV, NS, ST);
    const int j0 = (it - nkt) * TKEY, j = j0 + 2 * lane;
    float2 av[RPW], gv[RPW];
#pragma unroll
    for (int u = 0; u < RPW; ++u) {                   // the same (row, pair) this thread staged in pass 1
      const int i = i0 + warp * RPW + u;
      av[u] = gv[u] = make_float2(0.f, 0.f);
      if (i < T && j < S) {
        const long long off = (plane + i) * ldA + j;
        av[u] = *reinterpret_cast<const float2*>(A + off);
        gv[u] = *reinterpret_cast<const float2*>(dA + off);
      }
    }
#pragma unroll
    for (int u = 0; u < RPW; ++u) {
      const int r = warp * RPW + u;
      const float dlr = sDelta[r];                    // written by lane 0 of this warp
      uint32_t sh, sl;
      split_f16(av[u].x * (gv[u].x * gs - dlr), av[u].y * (gv[u].y * gs - dlr), sh, sl);
      *reinterpret_cast<uint32_t*>(sPh + r * LDT16 + 2 * lane) = sh;
      *reinterpret_cast<uint32_t*>(sPl + r * LDT16 + 2 * lane) = sl;
    }
    cp_async_wait<NS - 1>();
    __syncthreads();
    const __half* sYh = sKV + (size_t)(it % NS) * ST;
    pv_block<HD>(sPh, sPl, sYh, sYh + TKEY * LDH, m0, d0, min(TKEY, S - j0), lane, out, crs);
    __syncthreads();
  }
#pragma unroll
  for (int nt = 0; nt < NT; ++nt)
#pragma unroll
    for (int c = 0; c < 4; ++c) out[nt][c] = fmaf(crs[nt][c], LO_INV, out[nt][c]);
  store_pv<HD, MB>(dQ, lddq, (long long)b * T, i0, T, h, out, scale);
}

constexpr size_t ATT_SMEM_MAX = 227 * 1024;

void attention_set_trace(long long* buf) { cudaMemcpyToSymbol(g_attn_trace, &buf, sizeof(buf)); }

// scratch planes of one call (stream-ordered allocation: cached by the pool, capturable in CUDA graphs)
struct Planes {
  __half* buf = nullptr;
  cudaStream_t st = nullptr;
  int alloc(size_t halves, cudaStream_t s) {
    st = s;
    MMX_CHECK_CUDA(cudaMallocAsync((void**)&buf, halves * sizeof(__half), s));
    return 0;
  }
  ~Planes() { if (buf) cudaFreeAsync(buf, st); }
};

static void keep_pool_cached() {
  static std::atomic<bool> done[MMX_MAX_DEVICES];
  const int dev = current_device();
  if (!done[dev].load(std::memory_order_acquire)) {     // keep stream-ordered scratch cached across synchronisation points
    cudaMemPool_t pool;
    if (cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
      unsigned long long thr = ~0ull;
      cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
    }
    done[dev].store(true, std::memory_order_release);
  }
}

// K / V ring depth that fits next to the score rows (2 .. 4)
template <int HD>
static int pick_stages(int S, int TQ) {
  for (int ns = 4; ns > 2; --ns)
    if (AttnSmem<HD>::bytes(S, TQ, ns) <= ATT_SMEM_MAX) return ns;
  return 2;
}

template <int HD, int TQ, int NP, int NS>
static int launch_fwd_tq(const __half* Qh, const __half* Ql, const __half* Kh, const __half* Kl, const __half* Vh, const __half* Vl,
                         int ldp, const float* key_bias, float* A, int ldA, float* O, int ldo, int B, int H, int T, int S,
                         float q_mul, float post_scale, int flags, Ragged rg, cudaStream_t st) {
  const size_t smem = AttnSmem<HD>::bytes(S, TQ, NS);
  MMX_CHECK_CUDA(cudaFuncSetAttribute(attention_fwd_kernel<HD, TQ, NP, NS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  dim3 grid(cdiv(T, TQ), H, B);
  MMX_CHECK_CUDA(launch_pdl(attention_fwd_kernel<HD, TQ, NP, NS>, grid, dim3(TQ * 4), smem, st, Qh, Ql, Kh, Kl, Vh, Vl, ldp, key_bias, A, ldA, O,
                            ldo, H, T, S, q_mul, post_scale, flags, rg));
  MMX_LAUNCH_CHECK();
  return 0;
}

// The single-pass kernels take a shape when a score row fits the registers of a warp (S <= 1024) and the score rows of a
// 32- or 64-query tile fit in shared memory; every other shape runs the two-pass kernels.
template <int HD>
static bool single_pass_ok(int S) {
  return S <= 64 * MAX_PAIRS && (AttnSmem<HD>::bytes(S, 64) <= ATT_SMEM_MAX || AttnSmem<HD>::bytes(S, 32) <= ATT_SMEM_MAX);
}

constexpr int LONG_NS = 3;   // ring depth of the two-pass kernels

static int check_long(int S, const Ragged& rg) {
  MMX_REQUIRE(S <= LONG_MAX_S, "attention: at most 16384 keys per row");
  MMX_REQUIRE(rg.lens == nullptr, "ragged attention: at most 1024 keys per row");
  return 0;
}

template <int HD>
static int launch_fwd_long(const __half* Qh, const __half* Ql, const __half* Kh, const __half* Kl, const __half* Vh, const __half* Vl,
                           int ldp, const float* key_bias, float* A, int ldA, float* O, int ldo, int B, int H, int T, int S,
                           float post, int flags, Ragged rg, cudaStream_t st) {
  MMX_TRY(check_long(S, rg));
  MMX_REQUIRE(Ql != nullptr, "long attention takes pre-split planes");
  const size_t smem = LongSmem<HD>::bytes(LONG_NS, 2);
  MMX_CHECK_CUDA(cudaFuncSetAttribute(attention_fwd_long_kernel<HD, LONG_NS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  dim3 grid(cdiv(T, LTQ), H, B);
  MMX_CHECK_CUDA(launch_pdl(attention_fwd_long_kernel<HD, LONG_NS>, grid, dim3(LONG_THREADS), smem, st, Qh, Ql, Kh, Kl, Vh, Vl, ldp,
                            key_bias, A, ldA, O, ldo, H, T, S, post, flags));
  MMX_LAUNCH_CHECK();
  return 0;
}

// forward on ready-made planes (row stride ldp halves; Q already carries the pre-product scale)
template <int HD>
static int launch_fwd_planes(const __half* Qh, const __half* Ql, const __half* Kh, const __half* Kl, const __half* Vh, const __half* Vl,
                             int ldp, const float* key_bias, float* A, int ldA, float* O, int ldo, int B, int H, int T, int S,
                             float q_mul, float post, int flags, Ragged rg, cudaStream_t st) {
  if (!single_pass_ok<HD>(S)) return launch_fwd_long<HD>(Qh, Ql, Kh, Kl, Vh, Vl, ldp, key_bias, A, ldA, O, ldo, B, H, T, S, post, flags, rg, st);
  const bool tq64 = AttnSmem<HD>::bytes(S, 64) <= ATT_SMEM_MAX;
#define MMX_FWD(TQ_, NP_, NS_) \
  return launch_fwd_tq<HD, TQ_, NP_, NS_>(Qh, Ql, Kh, Kl, Vh, Vl, ldp, key_bias, A, ldA, O, ldo, B, H, T, S, q_mul, post, flags, rg, st)
  if (S <= 128) MMX_FWD(64, 2, 2);
  if (tq64) {
    switch (pick_stages<HD>(S, 64)) { case 4: MMX_FWD(64, MAX_PAIRS, 4); case 3: MMX_FWD(64, MAX_PAIRS, 3); default: MMX_FWD(64, MAX_PAIRS, 2); }
  }
  switch (pick_stages<HD>(S, 32)) { case 4: MMX_FWD(32, MAX_PAIRS, 4); case 3: MMX_FWD(32, MAX_PAIRS, 3); default: MMX_FWD(32, MAX_PAIRS, 2); }
#undef MMX_FWD
}

// rows of the packed operands: B*T query rows, B*S key rows (upper bounds for ragged batches)
template <int HD>
static int launch_fwd(const float* Q, int ldq, const float* K, int ldk, const float* V, int ldv, const float* key_bias,
                      float* A, int ldA, float* O, int ldo, int B, int H, int T, int S, float scale, int flags,
                      Ragged rg, cudaStream_t st) {
  keep_pool_cached();
  const int D = H * HD;
  const long long rq = (long long)B * T, rk = (long long)B * S;
  const bool scale_scores = flags & MMX_ATTN_SCALE_SCORES;
  if (S <= 128 && ldq == ldk && ldk == ldv) {          // short sequences: the kernels split their (few) tiles themselves
    auto f = [](const float* p) { return reinterpret_cast<const __half*>(p); };
    return launch_fwd_planes<HD>(f(Q), nullptr, f(K), nullptr, f(V), nullptr, ldq, key_bias, A, ldA, O, ldo, B, H, T, S,
                                 scale_scores ? 1.f : scale, scale_scores ? scale : 1.f, flags, rg, st);
  }
  Planes pl;
  if (T == S && K == Q + D && V == Q + 2 * D && ldq == ldk && ldk == ldv) {     // packed q | k | v rows: ONE split pass, planes [rows, 3D]
    MMX_TRY(pl.alloc((size_t)2 * 3 * D * rq, st));
    __half* h3 = pl.buf; __half* l3 = h3 + rq * 3 * D;
    MMX_TRY(split_planes(Q, ldq, rq, 3 * D, scale_scores ? 1.f : scale, D, h3, l3, 3 * D, st));
    return launch_fwd_planes<HD>(h3, l3, h3 + D, l3 + D, h3 + 2 * D, l3 + 2 * D, 3 * D, key_bias, A, ldA, O, ldo, B, H, T, S, 1.f,
                                 scale_scores ? scale : 1.f, flags, rg, st);
  }
  MMX_TRY(pl.alloc((size_t)2 * D * (rq + 2 * rk), st));
  __half* Qh = pl.buf; __half* Ql = Qh + rq * D;
  __half* Kh = Ql + rq * D; __half* Kl = Kh + rk * D;
  __half* Vh = Kl + rk * D; __half* Vl = Vh + rk * D;
  MMX_TRY(split_planes(Q, ldq, rq, D, scale_scores ? 1.f : scale, D, Qh, Ql, D, st));   // the reference scales q before the product
  MMX_TRY(split_planes(K, ldk, rk, D, 1.f, 0, Kh, Kl, D, st));
  MMX_TRY(split_planes(V, ldv, rk, D, 1.f, 0, Vh, Vl, D, st));
  return launch_fwd_planes<HD>(Qh, Ql, Kh, Kl, Vh, Vl, D, key_bias, A, ldA, O, ldo, B, H, T, S, 1.f, scale_scores ? scale : 1.f, flags, rg, st);
}

template <int HD, int TQ, int NP, int NS>
static int launch_bwd_q_tq(const __half* Gh, const __half* Gl, int ldg, const __half* Kh, const __half* Kl, const __half* Vh,
                           const __half* Vl, int ldp, const float* A, float* dA, int ldA, float* delta, float* dQ, int lddq, int B, int H, int T, int S,
                           float scale, Ragged rg, const float* gscale, cudaStream_t st) {
  const size_t smem = AttnSmem<HD>::bytes(S, TQ, NS);
  MMX_CHECK_CUDA(cudaFuncSetAttribute(attention_bwd_q_kernel<HD, TQ, NP, NS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  dim3 grid(cdiv(T, TQ), H, B);
  MMX_CHECK_CUDA(launch_pdl(attention_bwd_q_kernel<HD, TQ, NP, NS>, grid, dim3(TQ * 4), smem, st, Gh, Gl, ldg, Kh, Kl, Vh, Vl, ldp, A, dA, ldA,
                            delta, dQ, lddq, H, T, S, scale, rg, gscale));
  MMX_LAUNCH_CHECK();
  return 0;
}

// backward on ready-made planes: G = dO, Q / K / V planes with row strides ldg / ldp; scale_q multiplies dQ, scale_k
// multiplies dK (1 when the Q planes already carry the pre-product scale)
template <int HD>
static int launch_bwd_planes(const __half* Gh, const __half* Gl, int ldg, const __half* Qh, const __half* Ql, const __half* Kh,
                             const __half* Kl, const __half* Vh, const __half* Vl, int ldp, const float* A, float* dA, int ldA,
                             float* delta, float* dQ, int lddq, float* dK, int lddk, float* dV, int lddv, int B, int H, int T, int S,
                             float scale_q, float scale_k, Ragged rg, const float* gscale, cudaStream_t st) {
  const bool tq64 = AttnSmem<HD>::bytes(S, 64) <= ATT_SMEM_MAX;
#define MMX_BWDQ(TQ_, NP_, NS_) \
  MMX_TRY((launch_bwd_q_tq<HD, TQ_, NP_, NS_>(Gh, Gl, ldg, Kh, Kl, Vh, Vl, ldp, A, dA, ldA, delta, dQ, lddq, B, H, T, S, scale_q, rg, gscale, st)))
  if (!single_pass_ok<HD>(S)) {
    MMX_TRY(check_long(S, rg));
    MMX_REQUIRE(Gl != nullptr, "long attention takes pre-split planes");
    const size_t smem = LongSmem<HD>::bytes(LONG_NS, 1);
    MMX_CHECK_CUDA(cudaFuncSetAttribute(attention_bwd_q_long_kernel<HD, LONG_NS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dim3 grid(cdiv(T, LTQ), H, B);
    MMX_CHECK_CUDA(launch_pdl(attention_bwd_q_long_kernel<HD, LONG_NS>, grid, dim3(LONG_THREADS), smem, st, Gh, Gl, ldg, Kh, Kl, Vh, Vl,
                              ldp, A, dA, ldA, delta, dQ, lddq, H, T, S, scale_q, gscale));
    MMX_LAUNCH_CHECK();
  } else if (S <= 128) {
    MMX_BWDQ(64, 2, 2);
  } else if (tq64) {
    switch (pick_stages<HD>(S, 64)) { case 4: MMX_BWDQ(64, MAX_PAIRS, 4); break; case 3: MMX_BWDQ(64, MAX_PAIRS, 3); break; default: MMX_BWDQ(64, MAX_PAIRS, 2); }
  } else {
    switch (pick_stages<HD>(S, 32)) { case 4: MMX_BWDQ(32, MAX_PAIRS, 4); break; case 3: MMX_BWDQ(32, MAX_PAIRS, 3); break; default: MMX_BWDQ(32, MAX_PAIRS, 2); }
  }
#undef MMX_BWDQ
  if (dQ == nullptr) return 0;
  const size_t smem2 = sizeof(__half) * (4 * KV_ROWS * (HD + 8) + 4 * KV_ROWS * (KV_KEYS + 8));
  MMX_CHECK_CUDA(cudaFuncSetAttribute(attention_bwd_kv_kernel<HD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem2));
  dim3 grid2(cdiv(S, KV_KEYS), H, B);
  MMX_CHECK_CUDA(launch_pdl(attention_bwd_kv_kernel<HD>, grid2, dim3(KV_THREADS), smem2, st, Gh, Gl, ldg, Qh, Ql, ldp, A, dA, ldA, delta, dK, lddk,
                            dV, lddv, H, T, S, scale_k, rg, gscale));
  MMX_LAUNCH_CHECK();
  return 0;
}

template <int HD>
static int launch_bwd(const float* dO, int lddo, const float* Q, int ldq, const float* K, int ldk, const float* V, int ldv,
                      const float* A, float* dA, int ldA, float* delta, float* dQ, int lddq, float* dK, int lddk, float* dV,
                      int lddv, int B, int H, int T, int S, float scale, Ragged rg, const float* gscale, cudaStream_t st) {
  keep_pool_cached();
  const int D = H * HD;
  const long long rq = (long long)B * T, rk = (long long)B * S;
  const bool full = dQ != nullptr;                   // the last relevant block stops after dA: only dO and V are needed
  if (S <= 128 && ldq == ldk && ldk == ldv) {          // short sequences: the kernels split their (few) tiles themselves
    auto f = [](const float* p) { return reinterpret_cast<const __half*>(p); };
    return launch_bwd_planes<HD>(f(dO), nullptr, lddo, f(Q), nullptr, f(K), nullptr, f(V), nullptr, ldq, A, dA, ldA, delta, dQ, lddq, dK,
                                 lddk, dV, lddv, B, H, T, S, scale, scale, rg, gscale, st);
  }
  Planes pl;
  if (T == S && K == Q + D && V == Q + 2 * D && ldq == ldk && ldk == ldv) {     // packed q | k | v rows: one split pass for them
    MMX_TRY(pl.alloc((size_t)2 * 4 * D * rq, st));
    __half* g = pl.buf; __half* gl = g + rq * D;
    __half* h3 = gl + rq * D; __half* l3 = h3 + rq * 3 * D;
    MMX_TRY(split_planes(dO, lddo, rq, D, 1.f, 0, g, gl, D, st));
    MMX_TRY(split_planes(Q, ldq, rq, 3 * D, 1.f, 0, h3, l3, 3 * D, st));
    return launch_bwd_planes<HD>(g, gl, D, h3, l3, h3 + D, l3 + D, h3 + 2 * D, l3 + 2 * D, 3 * D, A, dA, ldA, delta, dQ, lddq, dK, lddk,
                                 dV, lddv, B, H, T, S, scale, scale, rg, gscale, st);
  }
  MMX_TRY(pl.alloc((size_t)2 * D * (rq + rk + (full ? rq + rk : 0)), st));
  __half* Gh = pl.buf; __half* Gl = Gh + rq * D;
  __half* Vh = Gl + rq * D; __half* Vl = Vh + rk * D;
  __half* Kh = Vl + rk * D; __half* Kl = Kh + rk * D;
  __half* Qh = Kl + rk * D; __half* Ql = Qh + rq * D;
  MMX_TRY(split_planes(dO, lddo, rq, D, 1.f, 0, Gh, Gl, D, st));
  MMX_TRY(split_planes(V, ldv, rk, D, 1.f, 0, Vh, Vl, D, st));
  if (full) {
    MMX_TRY(split_planes(K, ldk, rk, D, 1.f, 0, Kh, Kl, D, st));
    MMX_TRY(split_planes(Q, ldq, rq, D, 1.f, 0, Qh, Ql, D, st));
  }
  return launch_bwd_planes<HD>(Gh, Gl, D, Qh, Ql, Kh, Kl, Vh, Vl, D, A, dA, ldA, delta, dQ, lddq, dK, lddk, dV, lddv, B, H, T, S, scale,
                               scale, rg, gscale, st);
}

int attention_fwd(const float* Q, int ldq, const float* K, int ldk, const float* V, int ldv, const float* key_bias, float* A,
                  int ldA, float* O, int ldo, int B, int H, int T, int S, int hd, float scale, int flags, cudaStream_t st,
                  const int* offs, const int* lens) {
  Ragged rg;
  rg.offs = offs; rg.lens = lens;
  MMX_REQUIRE(lens == nullptr || (T == S && key_bias == nullptr && offs != nullptr), "ragged attention: self-attention without key bias only");
  MMX_REQUIRE(ldA >= S && ldA % 4 == 0, "ldA must be >= S and a multiple of 4");
  MMX_REQUIRE(ldq % 4 == 0 && ldk % 4 == 0 && ldv % 4 == 0 && ldo % 4 == 0 && aligned16(Q) && aligned16(K) && aligned16(V) &&
                  aligned16(O) && aligned16(A), "attention operands must be 16-byte aligned with leading dims % 4 == 0");
  if (B == 0 || T == 0) return 0;
  switch (hd) {
    case 16: return launch_fwd<16>(Q, ldq, K, ldk, V, ldv, key_bias, A, ldA, O, ldo, B, H, T, S, scale, flags, rg, st);
    case 32: return launch_fwd<32>(Q, ldq, K, ldk, V, ldv, key_bias, A, ldA, O, ldo, B, H, T, S, scale, flags, rg, st);
    case 64: return launch_fwd<64>(Q, ldq, K, ldk, V, ldv, key_bias, A, ldA, O, ldo, B, H, T, S, scale, flags, rg, st);
    default: MMX_REQUIRE(false, "head_dim must be 16, 32 or 64");
  }
  return 0;
}

int attention_bwd(const float* dO, int lddo, const float* Q, int ldq, const float* K, int ldk, const float* V, int ldv,
                  const float* A, float* dA, int ldA, float* delta, float* dQ, int lddq, float* dK, int lddk, float* dV,
                  int lddv, int B, int H, int T, int S, int hd, float scale, int flags, cudaStream_t st, const int* offs,
                  const int* lens, const float* gscale) {
  Ragged rg;
  rg.offs = offs; rg.lens = lens;
  MMX_REQUIRE(lens == nullptr || (T == S && offs != nullptr), "ragged attention: self-attention only");
  MMX_REQUIRE(ldA >= S && ldA % 4 == 0, "ldA must be >= S and a multiple of 4");
  MMX_REQUIRE(lddo % 4 == 0 && ldq % 4 == 0 && ldk % 4 == 0 && ldv % 4 == 0 && aligned16(dO) && aligned16(Q) && aligned16(K) &&
                  aligned16(V) && aligned16(A) && aligned16(dA) && (dQ == nullptr || (lddq % 4 == 0 && lddk % 4 == 0 &&
                  lddv % 4 == 0 && aligned16(dQ) && aligned16(dK) && aligned16(dV))),
              "attention operands must be 16-byte aligned with leading dims % 4 == 0");
  MMX_REQUIRE((dQ == nullptr) == (dK == nullptr) && (dQ == nullptr) == (dV == nullptr), "dQ/dK/dV: all or none");
  MMX_REQUIRE(dQ == nullptr || delta != nullptr, "delta scratch required");
  (void)flags;  // the mask is already folded into A (masked entries are exactly 0, so dS vanishes there)
  if (B == 0 || T == 0) return 0;
  switch (hd) {
    case 16: return launch_bwd<16>(dO, lddo, Q, ldq, K, ldk, V, ldv, A, dA, ldA, delta, dQ, lddq, dK, lddk, dV, lddv, B, H, T, S, scale, rg, gscale, st);
    case 32: return launch_bwd<32>(dO, lddo, Q, ldq, K, ldk, V, ldv, A, dA, ldA, delta, dQ, lddq, dK, lddk, dV, lddv, B, H, T, S, scale, rg, gscale, st);
    case 64: return launch_bwd<64>(dO, lddo, Q, ldq, K, ldk, V, ldv, A, dA, ldA, delta, dQ, lddq, dK, lddk, dV, lddv, B, H, T, S, scale, rg, gscale, st);
    default: MMX_REQUIRE(false, "head_dim must be 16, 32 or 64");
  }
  return 0;
}

}  // namespace mmx

using namespace mmx;
extern "C" {
int mmx_attention_fwd(const float* Q, int ldq, const float* K, int ldk, const float* V, int ldv, const float* key_bias,
                      float* A, int ldA, float* O, int ldo, int B, int H, int T, int S, int hd, float scale, int flags,
                      void* stream) {
  return attention_fwd(Q, ldq, K, ldk, V, ldv, key_bias, A, ldA, O, ldo, B, H, T, S, hd, scale, flags, (cudaStream_t)stream,
                       nullptr, nullptr);
}
int mmx_attention_bwd(const float* dO, int lddo, const float* Q, int ldq, const float* K, int ldk, const float* V, int ldv,
                      const float* A, float* dA, int ldA, float* delta, float* dQ, int lddq, float* dK, int lddk, float* dV,
                      int lddv, int B, int H, int T, int S, int hd, float scale, int flags, void* stream) {
  return attention_bwd(dO, lddo, Q, ldq, K, ldk, V, ldv, A, dA, ldA, delta, dQ, lddq, dK, lddk, dV, lddv, B, H, T, S, hd, scale,
                       flags, (cudaStream_t)stream, nullptr, nullptr, nullptr);
}
int mmx_attention_bwd_scaled(const float* dO, int lddo, const float* Q, int ldq, const float* K, int ldk, const float* V,
                             int ldv, const float* A, float* dA, int ldA, float* delta, float* dQ, int lddq, float* dK,
                             int lddk, float* dV, int lddv, int B, int H, int T, int S, int hd, float scale, int flags,
                             const float* gscale, void* stream) {
  return attention_bwd(dO, lddo, Q, ldq, K, ldk, V, ldv, A, dA, ldA, delta, dQ, lddq, dK, lddk, dV, lddv, B, H, T, S, hd, scale,
                       flags, (cudaStream_t)stream, nullptr, nullptr, gscale);
}
int mmx_attention_fwd_ragged(const float* Q, int ldq, const float* K, int ldk, const float* V, int ldv, float* A, int ldA,
                             float* O, int ldo, const int* offs, const int* lens, int B, int H, int T, int hd, float scale,
                             int flags, void* stream) {
  MMX_REQUIRE(offs != nullptr && lens != nullptr, "ragged attention needs offs and lens");
  return attention_fwd(Q, ldq, K, ldk, V, ldv, nullptr, A, ldA, O, ldo, B, H, T, T, hd, scale, flags, (cudaStream_t)stream, offs,
                       lens);
}
int mmx_attention_bwd_ragged(const float* dO, int lddo, const float* Q, int ldq, const float* K, int ldk, const float* V,
                             int ldv, const float* A, float* dA, int ldA, float* delta, float* dQ, int lddq, float* dK,
                             int lddk, float* dV, int lddv, const int* offs, const int* lens, int B, int H, int T, int hd,
                             float scale, int flags, const float* gscale, void* stream) {
  MMX_REQUIRE(offs != nullptr && lens != nullptr, "ragged attention needs offs and lens");
  return attention_bwd(dO, lddo, Q, ldq, K, ldk, V, ldv, A, dA, ldA, delta, dQ, lddq, dK, lddk, dV, lddv, B, H, T, T, hd, scale,
                       flags, (cudaStream_t)stream, offs, lens, gscale);
}
}
